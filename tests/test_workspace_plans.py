"""The workspace plans of include/b2ocr.h against restatements here.

CPU: ``b2o_craft_workspace_bytes`` is the greedy liveness packing of tests/stage_refs.py's CRAFT_BUFS (largest buffer
first, ties in table order; each at the lowest offset free among the placed buffers whose lifetimes overlap its own;
256-byte rounding), and ``b2o_crnn_workspace_bytes`` keeps its pinned sizes.  GPU: after forward_until(k),
``b2o_craft_tap`` reads exactly the buffers CRAFT_BUFS holds live at step k and refuses every other one, which pins each
buffer's lifetime in the library's plan.
"""
import numpy as np
import pytest
import torch

from keras_ocr_b200 import _lib
from keras_ocr_b200 import weights as W
from tests import stage_refs as R
from tests.test_gpu_craft_stages import SIZES

CRAFT_SHAPES = SIZES + [(32, 1536, 1536), (32, 2048, 2048), (3, 97, 65), (7, 511, 257)]


def _packed_bytes(n, h, w):
    dims = R.craft_dims(h, w)
    bufs = [((n * dims[lv][0] * dims[lv][1] * c * 2 + 255) // 256 * 256, first, last)
            for lv, c, first, last in R.CRAFT_BUFS.values()]
    order = sorted(range(len(bufs)), key=lambda i: -bufs[i][0])          # stable: ties keep the table's order
    off, total = {}, 0
    for i in order:
        size, first, last = bufs[i]
        busy = sorted((off[j], off[j] + bufs[j][0]) for j in off if bufs[j][1] <= last and first <= bufs[j][2])
        at = 0
        for begin, end in busy:
            if at + size <= begin:
                break
            at = max(at, end)
        off[i] = at
        total = max(total, at + size)
    return total


@pytest.mark.parametrize("shape", CRAFT_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_craft_workspace_is_the_greedy_packing_of_craft_bufs(shape):
    assert _lib.load_library().b2o_craft_workspace_bytes(*shape) == _packed_bytes(*shape)


def test_craft_workspace_pinned_sizes():
    lib = _lib.load_library()
    assert lib.b2o_craft_workspace_bytes(32, 1536, 1536) == 21_743_271_936
    assert lib.b2o_craft_workspace_bytes(32, 2048, 2048) == 38_654_705_664


def test_crnn_workspace_pinned_sizes():
    lib = _lib.load_library()
    assert lib.b2o_crnn_workspace_bytes(1) == 10_778_112
    assert lib.b2o_crnn_workspace_bytes(2) == 21_555_456
    assert lib.b2o_crnn_workspace_bytes(257) == 2_769_833_472
    assert lib.b2o_crnn_workspace_bytes(0) == 0


@pytest.mark.gpu
def test_craft_taps_are_live_exactly_over_craft_bufs_lifetimes(cuda_device):
    n, h, w = 2, 33, 47
    ctx = _lib.Context(0)
    ctx.load_craft(W.synthetic_craft_weights(3))
    img = torch.from_numpy(np.random.default_rng(0).integers(0, 256, (n, h, w, 3), dtype=np.uint8)).cuda()
    nbytes = ctx.craft_workspace_bytes(n, h, w)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    scores = torch.empty(n * (h // 2) * (w // 2) * 2, dtype=torch.float32, device="cuda")
    out = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    for k in range(_lib.CRAFT_LAST_STEP + 1):
        ctx.craft_forward_until(img.data_ptr(), n, h, w, scores.data_ptr(), ws.data_ptr(), nbytes, k, stream)
        for name, (_lv, _c, first, last) in R.CRAFT_BUFS.items():
            if first <= k <= last:
                ctx.craft_tap(name, ws.data_ptr(), n, h, w, out.data_ptr(), out.numel(), stream)
            else:
                with pytest.raises(_lib.B2OError, match=r"\(-5\)"):
                    ctx.craft_tap(name, ws.data_ptr(), n, h, w, out.data_ptr(), out.numel(), stream)
    torch.cuda.synchronize()
