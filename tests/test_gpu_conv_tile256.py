"""The channels-by-pixels body on 16 x 16-pixel tiles (streamed 128-channel 3x3 layers: one filter stage serves 256
pixels, both consumer warpgroups read every stage) against the pixels-by-channels body on 8 x 16 tiles it replaces
(B2O_TC_SWAP=0).

Both add every output's products in the same order and run the same fmaf / ReLU / fmaf and fp16 rounding, so:

1. through ``b2o_conv_test``, every output and fused-pool buffer is the same bit for bit, whole buffers with sentinel
   guards compared: 1, 2 and 4 n-tiles, the fused pool with write_full 0 and 1 and odd pooled sizes, a second affine,
   relu = 0, input and output in channel slices of wider buffers; on one tile, maps with partial right and bottom
   tiles, the recognizer's 200 x 31 and 100 x 15 maps, and a width the selection turns down;
2. ``b2o_tc_tile256_launches`` shows that the body ran for every shape that claims it, and for no other;
3. the outputs lie within the fp64 bound of ``tests/stage_refs.py``;
4. a one-tile image gives the same bits alone and in batches around the SM count, at CTA positions 0, 1 and 2;
5. the profiler sees only the ``conv_tc_kernel<128, 64, 1, false, false>`` instance.
"""
import re
import zlib

import numpy as np
import pytest
import torch

from keras_ocr_b200 import _lib
from tests import stage_refs as R
from tests import test_conv_plans as P
from tests.test_gpu_conv_transposed import SENT16, Slab, _make_ctx, _untouched

pytestmark = pytest.mark.gpu


def _stream():
    return torch.cuda.current_stream().cuda_stream


# (name, cin, cout, pool, write_full, x view (offset, extra), out view (offset, extra), second affine, relu)
LAYERS = [
    ("c128_128", 128, 128, False, 1, (0, 0), (0, 0), False, 1),
    ("c128_256_pool_wf1_slice", 128, 256, True, 1, (0, 0), (8, 16), False, 1),
    ("c256_512_pool_wf0", 256, 512, True, 0, (0, 0), (0, 0), False, 1),
    ("c128_128_aff2_relu0_slices", 128, 128, False, 1, (64, 64), (128, 64), True, 0),
    ("c512_512_relu0", 512, 512, False, 1, (0, 0), (0, 0), False, 0),
]
# (n, h, w): one tile, partial right and bottom tiles, the CRNN's maps (100 x 15 takes the halo tiles only with the
# fused pool), and widths whose 16-wide tiles cover more columns than the 8-wide ones (40, 24: not selected)
SHAPES = [(1, 16, 16), (2, 31, 47), (1, 200, 31), (2, 100, 15), (1, 32, 40), (1, 17, 24)]


def _selected(cin, cout, shape, pool):
    """The plan's choice of the 16 x 16 body for this layer and shape, as tests/test_conv_plans.py restates it (and
    checks the restatement against the library's plan)."""
    return P.restate(*shape, cin, cout, 3, pool=pool)["body"] == P.TILE256


def _inputs(name, n, h, w, cin, cout, aff2):
    rng = np.random.default_rng(zlib.crc32(f"tile256/{name}/{n}x{h}x{w}".encode()))
    x = rng.standard_normal((n, h, w, cin)).astype(np.float16)
    wgt = (rng.standard_normal((cout, 3, 3, cin)) * np.sqrt(2.0 / (cin * 9))).astype(np.float32)
    s1 = (rng.uniform(0.5, 1.5, cout) * np.where(rng.random(cout) < 0.2, -1.0, 1.0)).astype(np.float32)
    t1 = (rng.standard_normal(cout) * 0.2).astype(np.float32)
    s2 = rng.uniform(0.5, 1.5, cout).astype(np.float32) if aff2 else None
    t2 = (rng.standard_normal(cout) * 0.2).astype(np.float32) if aff2 else None
    return x, wgt, s1, t1, s2, t2


def _run(ctx, layer, x, params):
    name, cin, cout, pool, write_full, (xo, xe), (oo, oe), _, relu = layer
    n, h, w = x.shape[:3]
    xs = Slab(n, h, w, cin + xo + xe)
    xs.body()[..., xo:xo + cin] = torch.from_numpy(x).cuda()
    outs = Slab(n, h, w, cout + oo + oe)
    kw = {}
    ps = None
    if pool:
        ps = Slab(n, h // 2, w // 2, cout + 8)
        kw.update(pool=ps.ptr(8), pool_ld=ps.ld)
    wgt, s1, t1, s2, t2 = params
    before = ctx.tile256_launches()
    ctx.conv_test(xs.ptr(xo), n, h, w, cin, xs.ld, wgt, cout, 3, 1, s1, t1, relu, s2, t2, outs.ptr(oo), outs.ld,
                  _lib.CONV_AUTO, _stream(), write_full=write_full, **kw)
    torch.cuda.synchronize()
    return outs, ps, ctx.tile256_launches() - before


@pytest.fixture(scope="module")
def ctxs(cuda_device):
    made = {"swap": _make_ctx(True), "noswap": _make_ctx(False)}
    yield made
    for c in made.values():
        c.close()


@pytest.mark.parametrize("shape", SHAPES, ids=[f"{n}x{h}x{w}" for n, h, w in SHAPES])
@pytest.mark.parametrize("layer", LAYERS, ids=[lay[0] for lay in LAYERS])
def test_tile256_bit_identical(ctxs, layer, shape):
    name, cin, cout, pool, write_full, _, (oo, _), aff2, relu = layer
    x, *params = _inputs(name, *shape, cin, cout, aff2)
    a_out, a_pool, a_ran = _run(ctxs["swap"], layer, x, params)
    b_out, b_pool, b_ran = _run(ctxs["noswap"], layer, x, params)
    assert a_ran == (1 if _selected(cin, cout, shape, pool) else 0), f"{name} {shape}: 16 x 16 body launches {a_ran}"
    assert b_ran == 0, "B2O_TC_SWAP=0 ran the 16 x 16 body"
    assert torch.equal(a_out.raw, b_out.raw), f"{name} {shape}: out differs (or a store outside the view)"
    if write_full:
        assert _untouched(a_out, oo, cout), f"{name} {shape}: store outside the output slice"
        assert not (a_out.body()[..., oo:oo + cout].view(torch.int16) == SENT16).any(), f"{name} {shape}: pixel unwritten"
    else:
        assert _untouched(a_out, 0, 0), f"{name} {shape}: out written with write_full = 0"
    if pool:
        assert torch.equal(a_pool.raw, b_pool.raw), f"{name} {shape}: pooled output differs"
        assert _untouched(a_pool, 8, cout), f"{name} {shape}: store outside the pooled view"
        assert not (a_pool.body()[..., 8:8 + cout].view(torch.int16) == SENT16).any(), f"{name} {shape}: pooled pixel unwritten"
    if shape == (2, 31, 47):                                  # against fp64 (bounded CPU time)
        wgt, s1, t1, s2, t2 = params
        y, e = R.conv_ref(x, wgt, 3, 1, s1, t1, relu, s2, t2)
        y, e = np.asarray(y), np.asarray(e)
        if write_full:
            got = a_out.body()[..., oo:oo + cout].float().cpu().numpy().astype(np.float64)
            assert (np.abs(got - y) <= e).all(), f"{name}: max excess {np.max(np.abs(got - y) - e)}"
        if pool:
            py, pe = (np.asarray(v) for v in R.pool_ref(y, e))
            got = a_pool.body()[..., 8:8 + cout].float().cpu().numpy().astype(np.float64)
            assert (np.abs(got - py) <= pe).all(), f"{name}: pooled max excess {np.max(np.abs(got - py) - pe)}"


def test_tile256_batch_and_position_independent(ctxs):
    """A one-tile (16 x 16) image gives the same bits alone and in batches of 1, SM - 1, SM, SM + 1 and 2 SM + 1, at
    batch positions 0, 1 and 2 (so on the CTAs 0, 1 and 2 of the persistent grid)."""
    ctx = ctxs["swap"]
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    layer = ("c128_128_pool", 128, 128, True, 1, (0, 0), (0, 0), False, 1)     # one n-tile: one CTA per image
    name, cin, cout = layer[:3]
    x1, *params = _inputs(name, 1, 16, 16, cin, cout, False)
    alone_out, alone_pool, ran = _run(ctx, layer, x1, params)
    assert ran == 1
    bits = lambda slab, i: slab.body()[i].view(torch.int16)       # noqa: E731 (the sentinel is a NaN)
    rng = np.random.default_rng(7)
    for b in (1, sm - 1, sm, sm + 1, 2 * sm + 1):
        for pos in (0, 1, 2):
            if pos >= b:
                continue
            xb = rng.standard_normal((b, 16, 16, cin)).astype(np.float16)
            xb[pos] = x1[0]
            out, pool, ran = _run(ctx, layer, xb, params)
            assert ran == 1
            assert torch.equal(bits(out, pos), bits(alone_out, 0)), (b, pos)
            assert torch.equal(bits(pool, pos), bits(alone_pool, 0)), (b, pos)


def test_tile256_runs_in_the_streamed_128_instance(ctxs):
    """The 16 x 16 body is a second body inside conv_tc_kernel<128, 64, 1, false, false>: no other instance runs."""
    from torch.profiler import ProfilerActivity, profile
    ctx = ctxs["swap"]
    layer = LAYERS[1]
    name, cin, cout = layer[:3]
    x, *params = _inputs(name, 2, 31, 47, cin, cout, False)
    _run(ctx, layer, x, params)                                # warm-up (module load)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _, _, ran = _run(ctx, layer, x, params)
    assert ran == 1
    names = {e.name for e in prof.events() if "conv_tc_kernel" in e.name}
    instances = {re.search(r"conv_tc_kernel<([^>]*)>", n).group(1).replace(" ", "") for n in names}
    assert instances == {"128,64,1,false,false"}, names
