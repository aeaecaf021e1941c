"""Paired n-tiles (``b2o_conv_plan.coop_n``): on generic 128-channel tiles of layers with cout % 256 == 0, both consumer
warpgroups share every activation box, warpgroup wg computing n-tile 2j + wg of a unit.

The reference is the ping-pong schedule the library runs for a 128-channel layer: the same layer split into cout / 128
launches of 128 output channels, each writing its channel slice of the same output.  That is the same box, the same
chunks, the same MMAs and the same epilogue per n-tile, so the outputs must be equal bit for bit:

1. whole buffers with sentinel guards, over 1x1 and 3x3 layers, dilation 6, cout 256, 512 and 1024, the recognizer's
   50 x 7 and 100 x 15 maps at odd batches, the bench's 96 x 96 map, a second affine, relu = 0, fp32 output and channel
   slices of wider input and output buffers; fewer units than SMs and an odd number of units per CTA;
2. a crop alone and the same crop at batch positions 0, 1 and 2 of batches SM - 1, SM + 1 and 300;
3. ``b2o_tc_coop_n_launches`` shows that pairing ran wherever the plan says so, and never in the reference;
4. only the ``conv_tc_kernel<128, 64, 0, false, false>`` instance runs.

The CPU part checks the plan's rule for the flag over every launch of both forwards, and that the fields
tests/test_conv_plans.py restates do not change with it.
"""
import re
import zlib

import numpy as np
import pytest
import torch

from keras_ocr_b200 import _lib
from tests import test_conv_plans as P

GUARD = 4096                          # elements after the last pixel of every buffer
SENT = {torch.float16: 0x7E5A, torch.float32: 0x7FC05A5A}    # NaN bit patterns


def coop_rule(plan, cout, up_add=False, tail=False):
    """The plan's flag as restated: generic tiles, 64-channel chunks, 128-channel n-tiles, an even number of them, no
    CTA pair, upsample-add or tail."""
    return int(plan["mode"] == 0 and plan["kch"] == 64 and plan["block_n"] == 128 and cout % 256 == 0 and
               not plan["pair"] and not up_add and not tail)


# ------------------------------------------------------------------------------------------------ CPU: the plans
@pytest.mark.parametrize("shape", P.FORWARD_SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_craft_plans_pair_by_the_rule(shape):
    for engine in (P.AUTO, P.GENERIC):
        for b in P.BATCHES:
            for lc in P.craft_launches(b, *shape, engine):
                got = P._plan(lc, engine, 1)
                assert got["coop_n"] == coop_rule(got, lc.cout, lc.up_add, lc.tail), (lc, got)
                P._check(lc, engine, 1)             # the restated fields and invariants hold with the flag


def test_crnn_plans_pair_by_the_rule():
    for engine in (P.AUTO, P.GENERIC):
        for b in P.BATCHES:
            for lc in P.crnn_launches(b, engine):
                got = P._plan(lc, engine, 1)
                assert got["coop_n"] == coop_rule(got, lc.cout, lc.up_add, lc.tail), (lc, got)
                P._check(lc, engine, 1)


def test_bench_layers_that_pair():
    """The layers of the bench's step that run paired n-tiles (the detector at 1536 x 1536, the recognizer's crops;
    without the opt-in commuted decoder halves ".y" / ".s")."""
    paired = {lc.layer for lc in P.craft_launches(32, *P.BENCH, P.AUTO) + P.crnn_launches(1028, P.AUTO)
              if P._plan(lc, P.AUTO, 1)["coop_n"] and not lc.layer.endswith((".y", ".s"))}
    assert paired == {"basenet.slice5.1", "basenet.slice5.2", "upconv1.conv.0", "upconv2.conv.0", "conv_4", "conv_6",
                      "conv_7", "stn.conv_a_gemm", "lstm_in_1", "lstm_in_2"}, paired


# ------------------------------------------------------------------------------------------------ GPU: the outputs
class Buf:
    """An NHWC buffer of ld channels per pixel plus GUARD elements, filled with the sentinel."""

    def __init__(self, n, h, w, ld, dtype=torch.float16):
        self.shape, self.ld, self.dtype = (n, h, w), ld, dtype
        itype = torch.int16 if dtype == torch.float16 else torch.int32
        self.raw = torch.full((n * h * w * ld + GUARD,), SENT[dtype], dtype=itype, device="cuda")
        self.data = self.raw.view(dtype)

    def body(self):
        return self.data[: self.raw.numel() - GUARD].view(*self.shape, self.ld)

    def ptr(self, off):
        return self.data.data_ptr() + off * self.data.element_size()

    def untouched(self, off, c):
        """Channels [0, off) and [off + c, ld) of every pixel and the guard hold the sentinel, and every pixel of the
        view was written."""
        body = self.raw[: self.raw.numel() - GUARD].view(*self.shape, self.ld)
        return bool((body[..., :off] == SENT[self.dtype]).all() and (body[..., off + c:] == SENT[self.dtype]).all() and
                    (self.raw[-GUARD:] == SENT[self.dtype]).all() and not (body[..., off:off + c] == SENT[self.dtype]).any())


def _stream():
    return torch.cuda.current_stream().cuda_stream


# (name, cin, cout, k, dilation, x view (offset, extra), out view (offset, extra), second affine, relu, fp32 out)
LAYERS = {
    "slice5_2_1x1": (1024, 1024, 1, 1, (0, 0), (0, 0), False, 1, False),
    "upconv1_0_1x1": (1536, 512, 1, 1, (0, 0), (0, 0), False, 1, False),
    "slice5_1_dil6": (512, 1024, 3, 6, (0, 0), (0, 0), False, 1, False),
    "conv_4": (256, 256, 3, 1, (0, 0), (0, 0), True, 1, False),
    "conv_6": (512, 512, 3, 1, (0, 0), (0, 0), True, 1, False),
    "c256_512_1x1_slices_relu0": (256, 512, 1, 1, (64, 64), (128, 64), False, 0, False),
    "c256_256_3x3_aff2_relu0": (256, 256, 3, 1, (0, 0), (0, 0), True, 0, False),
    "lstm_in_fp32": (128, 1024, 1, 1, (0, 0), (0, 0), False, 1, True),
    "c512_256_fp32_slices": (512, 256, 1, 1, (64, 0), (32, 32), False, 0, True),
    "flat_256": (256, 256, 1, 1, (0, 0), (0, 0), False, 1, False),
}


def _inputs(name, n, h, w, cin, cout, k, aff2):
    rng = np.random.default_rng(zlib.crc32(f"coop_n/{name}/{n}x{h}x{w}".encode()))
    x = rng.standard_normal((n, h, w, cin)).astype(np.float16)
    wgt = (rng.standard_normal((cout, k, k, cin)) * np.sqrt(2.0 / (cin * k * k))).astype(np.float32)
    s1 = (rng.uniform(0.5, 1.5, cout) * np.where(rng.random(cout) < 0.2, -1.0, 1.0)).astype(np.float32)
    t1 = (rng.standard_normal(cout) * 0.2).astype(np.float32)
    s2 = rng.uniform(0.5, 1.5, cout).astype(np.float32) if aff2 else None
    t2 = (rng.standard_normal(cout) * 0.2).astype(np.float32) if aff2 else None
    return x, (wgt, s1, t1, s2, t2)


def _run(ctx, layer, x, params, split):
    """The layer over x as one launch (split = False) or as cout / 128 launches of 128 channels each; returns the output
    buffer and the number of launches that ran paired n-tiles."""
    cin, cout, k, dil, (xo, xe), (oo, oe), _, relu, f32 = layer
    n, h, w = x.shape[:3]
    xs = Buf(n, h, w, cin + xo + xe)
    xs.body()[..., xo:xo + cin] = torch.from_numpy(x).cuda()
    out = Buf(n, h, w, cout + oo + oe, torch.float32 if f32 else torch.float16)
    wgt, s1, t1, s2, t2 = params
    before = ctx.coop_n_launches()
    for c0 in range(0, cout, 128) if split else [0]:
        c1 = c0 + 128 if split else cout
        part = lambda a: None if a is None else np.ascontiguousarray(a[c0:c1])      # noqa: E731
        ctx.conv_test(xs.ptr(xo), n, h, w, cin, xs.ld, part(wgt), c1 - c0, k, dil, part(s1), part(t1), relu, part(s2),
                      part(t2), out.ptr(oo + c0), out.ld, _lib.CONV_AUTO, _stream(), out_f32=f32)
    torch.cuda.synchronize()
    return out, ctx.coop_n_launches() - before


@pytest.fixture(scope="module")
def ctx(cuda_device):
    c = _lib.Context(0)
    yield c
    c.close()


def _check_layer(ctx, name, shape):
    layer = LAYERS[name]
    cin, cout, k, dil, _, (oo, _), aff2, _, f32 = layer
    x, params = _inputs(name, *shape, cin, cout, k, aff2)
    plan = _lib.conv_plan(*shape, cin, cout, k, dil, out_f32=f32, sm_count=torch.cuda.get_device_properties(0).multi_processor_count)
    want = coop_rule(plan, cout)
    assert plan["coop_n"] == want, (name, shape, plan)
    got, ran = _run(ctx, layer, x, params, split=False)
    ref, ref_ran = _run(ctx, layer, x, params, split=True)
    assert ran == want, f"{name} {shape}: paired launches {ran}, plan {want}"
    assert ref_ran == 0, "a 128-channel launch ran paired n-tiles"
    assert torch.equal(got.raw, ref.raw), f"{name} {shape}: differs from the 128-channel launches"
    assert got.untouched(oo, cout), f"{name} {shape}: a store outside the view, or a pixel unwritten"
    return plan, got


# (layer, (n, h, w)): the bench's 96 x 96 map, the CRNN's maps at odd batches, small and odd maps
CASES = [
    ("slice5_2_1x1", (1, 96, 96)), ("upconv1_0_1x1", (1, 96, 96)), ("slice5_1_dil6", (1, 96, 96)),
    ("conv_4", (5, 100, 15)), ("conv_6", (37, 50, 7)), ("conv_6", (1, 50, 7)),
    ("c256_512_1x1_slices_relu0", (3, 50, 7)), ("c256_256_3x3_aff2_relu0", (7, 100, 15)),
    ("lstm_in_fp32", (1, 1, 50 * 13)), ("c512_256_fp32_slices", (3, 17, 23)),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[f"{c[0]}-{'x'.join(map(str, c[1]))}" for c in CASES])
def test_coop_n_bit_identical(ctx, case):
    _check_layer(ctx, *case)


@pytest.mark.gpu
def test_coop_n_fewer_units_than_sms(ctx):
    """One pixel tile of a 512-channel layer: 2 units, the other CTAs leave at once."""
    plan, _ = _check_layer(ctx, "slice5_1_dil6", (1, 8, 16))
    assert plan["coop_n"] and plan["tiles"] // 2 < plan["grid"], plan


@pytest.mark.gpu
def test_coop_n_odd_units_per_cta(ctx):
    """A flat map of 3 SM units less half a tile: every CTA walks 3 units, the last one partial."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    plan, _ = _check_layer(ctx, "flat_256", (1, 1, 128 * 3 * sm - 64))
    assert plan["coop_n"] and plan["tiles"] == 2 * 3 * sm and plan["grid"] == sm, plan


@pytest.mark.gpu
def test_coop_n_batch_and_position_independent(ctx):
    """A 50 x 7 crop of conv_6 gives the same bits alone and at batch positions 0, 1 and 2 of batches SM - 1, SM + 1
    and 300, and each batch equals its 128-channel launches."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    name = "conv_6"
    _, alone = _check_layer(ctx, name, (1, 50, 7))
    cin, cout, k, _, _, _, aff2, _, _ = LAYERS[name]
    x1, params = _inputs(name, 1, 50, 7, cin, cout, k, aff2)
    rng = np.random.default_rng(11)
    for b in (1, sm - 1, sm + 1, 300):
        xb = rng.standard_normal((b, 50, 7, cin)).astype(np.float16)
        for pos in (0, 1, 2):
            if pos < b:
                xb[pos] = x1[0]
        got, ran = _run(ctx, LAYERS[name], xb, params, split=False)
        assert ran == 1
        if b > 1:
            ref, _ = _run(ctx, LAYERS[name], xb, params, split=True)
            assert torch.equal(got.raw, ref.raw), b
        for pos in range(min(b, 3)):
            assert torch.equal(got.body()[pos].view(torch.int16), alone.body()[0].view(torch.int16)), (b, pos)


@pytest.mark.gpu
def test_coop_n_runs_in_the_generic_128_instance(ctx):
    """Paired n-tiles are a second body inside conv_tc_kernel<128, 64, 0, false, false>: no other instance runs."""
    from torch.profiler import ProfilerActivity, profile
    name, shape = "conv_6", (3, 50, 7)
    cin, cout, k, _, _, _, aff2, _, _ = LAYERS[name]
    x, params = _inputs(name, *shape, cin, cout, k, aff2)
    _run(ctx, LAYERS[name], x, params, split=False)                  # warm-up (module load)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _, ran = _run(ctx, LAYERS[name], x, params, split=False)
    assert ran == 1
    names = {e.name for e in prof.events() if "conv_tc_kernel" in e.name}
    instances = {re.search(r"conv_tc_kernel<([^>]*)>", n).group(1).replace(" ", "") for n in names}
    assert instances == {"128,64,0,false,false"}, names
