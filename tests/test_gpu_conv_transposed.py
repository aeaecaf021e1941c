"""The channels-by-pixels tensor-core instances (64-channel fp16 layers: filter bank as the wgmma A operand, pixel stage as
B, TMA-stored epilogue) against the pixels-by-channels ones they replace (B2O_TC_SWAP=0).

Both add every output's products in the same order and run the same fmaf / ReLU / fmaf and fp16 rounding, so every
output must be the same bit for bit:

1. layer by layer through ``b2o_conv_test``: the fused 2x2 pool with write_full 0 and 1, an output in a channel slice of a
   wider buffer, the 16-channel-chunk stem, a resident and a streamed filter bank, a generic 1x1 layer with a second
   affine; at sizes with partial tiles in every direction and long thin images;
2. the whole buffer is compared, so the sentinel guard channels and the region past the last pixel must stay untouched
   by both routes, and ``out`` must stay untouched where the fused pool runs with write_full = 0;
3. a batch of three equals the three images run one at a time;
4. the CRAFT score maps of the benchmark's batch (32 x 1536 x 1536).
"""
import os
import zlib

import numpy as np
import pytest
import torch

from keras_ocr_b200 import _lib
from keras_ocr_b200 import weights as W

pytestmark = pytest.mark.gpu

SENT16 = 0x7E5A                  # a NaN bit pattern
GUARD = 4096                     # elements after the last pixel of every buffer


def _stream():
    return torch.cuda.current_stream().cuda_stream


class Slab:
    """An NHWC fp16 buffer of ld channels per pixel plus GUARD elements, filled with the sentinel."""

    def __init__(self, n, h, w, ld):
        self.shape, self.ld = (n, h, w), ld
        self.raw = torch.full((n * h * w * ld + GUARD,), SENT16, dtype=torch.int16, device="cuda")
        self.data = self.raw.view(torch.float16)

    def body(self):
        return self.data[: self.raw.numel() - GUARD].view(*self.shape, self.ld)

    def ptr(self, off):
        return self.data.data_ptr() + off * 2


def _untouched(slab, off, c):
    """Channels [0, off) and [off + c, ld) of every pixel and the region past the last pixel hold the sentinel."""
    body = slab.raw[: slab.raw.numel() - GUARD].view(*slab.shape, slab.ld)
    return bool((body[..., :off] == SENT16).all() and (body[..., off + c:] == SENT16).all() and
                (slab.raw[-GUARD:] == SENT16).all())


# (name, cin, k, pool, write_full, x view (offset, extra), out view (offset, extra), second affine, relu)
LAYERS = [
    ("slice1_3_pool_wf0", 64, 3, True, 0, (0, 0), (0, 0), False, 1),
    ("slice1_3_pool_wf1", 64, 3, True, 1, (0, 0), (8, 16), False, 1),
    ("halo_into_channel_slice", 64, 3, False, 1, (72, 64), (64, 64), False, 1),
    ("stem16", 16, 3, False, 1, (0, 0), (0, 0), False, 1),
    ("upconv3_3_resident", 128, 3, False, 1, (0, 0), (0, 0), False, 1),
    ("streamed_256", 256, 3, True, 1, (0, 0), (0, 0), False, 1),
    ("upconv4_0_generic_1x1", 192, 1, False, 1, (0, 0), (0, 192), True, 0),
]
SHAPES = [(1, 32, 32), (2, 33, 47), (1, 32, 2048), (1, 2048, 40)]


def _inputs(name, n, h, w, cin, k, aff2):
    rng = np.random.default_rng(zlib.crc32(f"{name}/{n}x{h}x{w}".encode()))
    x = rng.standard_normal((n, h, w, cin)).astype(np.float16)
    wgt = (rng.standard_normal((64, k, k, cin)) * np.sqrt(2.0 / (cin * k * k))).astype(np.float32)
    s1 = (rng.uniform(0.5, 1.5, 64) * np.where(rng.random(64) < 0.2, -1.0, 1.0)).astype(np.float32)
    t1 = (rng.standard_normal(64) * 0.2).astype(np.float32)
    s2 = rng.uniform(0.5, 1.5, 64).astype(np.float32) if aff2 else None
    t2 = (rng.standard_normal(64) * 0.2).astype(np.float32) if aff2 else None
    return x, wgt, s1, t1, s2, t2


def _run(ctx, layer, x, params):
    name, cin, k, pool, write_full, (xo, xe), (oo, oe), _, relu = layer
    n, h, w = x.shape[:3]
    xs = Slab(n, h, w, cin + xo + xe)
    xs.body()[..., xo:xo + cin] = torch.from_numpy(x).cuda()
    outs = Slab(n, h, w, 64 + oo + oe)
    kw = {}
    ps = None
    if pool:
        ps = Slab(n, h // 2, w // 2, 64 + 8)
        kw.update(pool=ps.ptr(8), pool_ld=ps.ld)
    wgt, s1, t1, s2, t2 = params
    ctx.conv_test(xs.ptr(xo), n, h, w, cin, xs.ld, wgt, 64, k, 1, s1, t1, relu, s2, t2, outs.ptr(oo), outs.ld,
                  _lib.CONV_AUTO, _stream(), write_full=write_full, **kw)
    torch.cuda.synchronize()
    return outs, ps


def _make_ctx(swap):
    old = os.environ.get("B2O_TC_SWAP")
    os.environ["B2O_TC_SWAP"] = "1" if swap else "0"
    try:
        return _lib.Context(0)
    finally:
        if old is None:
            del os.environ["B2O_TC_SWAP"]
        else:
            os.environ["B2O_TC_SWAP"] = old


@pytest.fixture(scope="module")
def ctxs(cuda_device):
    made = {"swap": _make_ctx(True), "noswap": _make_ctx(False)}
    yield made
    for c in made.values():
        c.close()


@pytest.mark.parametrize("shape", SHAPES, ids=[f"{n}x{h}x{w}" for n, h, w in SHAPES])
@pytest.mark.parametrize("layer", LAYERS, ids=[lay[0] for lay in LAYERS])
def test_channels_by_pixels_bit_identical(ctxs, layer, shape):
    name, cin, k, pool, write_full, _, (oo, _), aff2, _ = layer
    x, *params = _inputs(name, *shape, cin, k, aff2)
    a_out, a_pool = _run(ctxs["swap"], layer, x, params)
    b_out, b_pool = _run(ctxs["noswap"], layer, x, params)
    assert torch.equal(a_out.raw, b_out.raw), f"{name} {shape}: out differs (or a store outside the view)"
    if write_full:
        assert _untouched(a_out, oo, 64), f"{name} {shape}: store outside the output slice"
        assert not (a_out.body()[..., oo:oo + 64].view(torch.int16) == SENT16).any(), f"{name} {shape}: pixel unwritten"
    else:
        assert _untouched(a_out, 0, 0), f"{name} {shape}: out written with write_full = 0"
    if pool:
        assert torch.equal(a_pool.raw, b_pool.raw), f"{name} {shape}: pooled output differs"
        assert _untouched(a_pool, 8, 64), f"{name} {shape}: store outside the pooled view"
        assert not (a_pool.body()[..., 8:72].view(torch.int16) == SENT16).any(), f"{name} {shape}: pooled pixel unwritten"


@pytest.mark.parametrize("layer", [LAYERS[0], LAYERS[2], LAYERS[6]], ids=[LAYERS[i][0] for i in (0, 2, 6)])
def test_channels_by_pixels_batch_independent(ctxs, layer):
    """An image gives the same bits alone and as one of a batch of three."""
    name, cin, k, pool, _, _, (oo, _), aff2, _ = layer
    x, *params = _inputs(name, 3, 33, 47, cin, k, aff2)
    full_out, full_pool = _run(ctxs["swap"], layer, x, params)
    bits = lambda slab, i: slab.body()[i].view(torch.int16)       # noqa: E731 (the sentinel is a NaN)
    for i in range(3):
        one_out, one_pool = _run(ctxs["swap"], layer, x[i:i + 1], params)
        assert torch.equal(bits(one_out, 0), bits(full_out, i)), (name, i)
        if pool:
            assert torch.equal(bits(one_pool, 0), bits(full_pool, i)), (name, i)


def test_craft_scores_at_benchmark_batch(cuda_device, monkeypatch):
    """The CRAFT score maps of a 32 x 1536 x 1536 batch (bench.py's detector input) are the same bits either way."""
    from keras_ocr_b200.detection import Detector
    cw = W.synthetic_craft_weights(3, textlike=True)
    gen = torch.Generator(device=cuda_device).manual_seed(31)
    img = torch.randint(0, 256, (32, 1536, 1536, 3), dtype=torch.uint8, device=cuda_device, generator=gen)
    scores = []
    for swap in ("1", "0"):                                   # one detector's workspace at a time
        monkeypatch.setenv("B2O_TC_SWAP", swap)
        det = Detector(weights=cw)
        scores.append(det.predict_device(img).clone())
        del det
        torch.cuda.empty_cache()
    a, b = scores
    assert torch.equal(a[0], b[0]) and torch.equal(a[31], b[31])
    assert torch.equal(a, b)
