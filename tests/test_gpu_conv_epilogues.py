"""Every epilogue feature of the convolution engines, one layer at a time, against an fp64 CPU reference.

Each case runs ``b2o_conv_test`` (routed like the product routes the layer) and checks, for every engine that supports
it (B2O_CONV_AUTO = the product path, TC_GENERIC, SIMT):

1. **values**: ``|dev - ref| <= bound`` element by element, where ``ref`` is the fp64 layer evaluated on the same
   fp16-rounded input, weights and low-resolution ``up`` tensor, and ``bound`` is derived from the arithmetic
   (tests/stage_refs.py): ``GAMMA(K) * sum|x*w| * |s1| (* |s2|)`` for the fp32 accumulation of K = taps * cin terms,
   ``2^-24`` per fmaf of the epilogue, ``2^-11 * |y|`` for the final fp16 rounding; a pooled output takes the largest of
   its window's four bounds; the CRAFT tail propagates the bound through |w6| and |w8|.  The worst ratio of error to
   bound is printed per case.  Measured on an H100 80GB HBM3 (700 W), every engine: 0.91 for fp16 outputs (the half-ulp
   rounding term dominates and is tight by construction), 0.55 for pooled outputs, 0.105 for the tail's scores against
   the fp64 chain and 0.0065 against the tail of the device's own 16-channel map.
2. **nothing written outside the output**: every buffer starts as a NaN sentinel bit pattern; output and pool views sit
   in a wider buffer with guard channels on both sides, and every buffer has a guard region after its last pixel.  The
   guards must be unchanged bit for bit, and ``out`` must be untouched where the fused pool runs with write_full = 0.
3. **bit identity across routes**: the fused pool equals the 2x2 max of the same run's full fp16 output; the fused CRAFT
   tail equals the separate ``head_tail_kernel`` route (B2O_FUSED_TAIL=0); CTA pairs (B2O_TC_PAIR=1, 2) and the
   epilogue constants in shared memory (B2O_TC_AFF=smem) equal the default, including an odd number of tile columns.
"""
import os
import zlib

import numpy as np
import pytest
import torch

from keras_ocr_b200 import _lib
from tests import stage_refs as R

pytestmark = pytest.mark.gpu

SENT16 = 0x7E5A                  # a NaN: any read of it into a result shows up in the value check
SENT32 = 0x7FA5A5A5
GUARD = 4096                     # elements after the last pixel of every buffer
ENGINES = {"auto": _lib.CONV_AUTO, "tc_generic": _lib.CONV_TC_GENERIC, "simt": _lib.CONV_SIMT}


def _stream():
    return torch.cuda.current_stream().cuda_stream


class Slab:
    """An NHWC buffer of ld channels per pixel plus GUARD elements, filled with the sentinel; a view is (offset, c)."""

    def __init__(self, n, h, w, ld, f32=False):
        self.shape, self.ld, self.f32 = (n, h, w), ld, f32
        it = torch.int32 if f32 else torch.int16
        self.raw = torch.full((n * h * w * ld + GUARD,), SENT32 if f32 else SENT16, dtype=it, device="cuda")
        self.data = self.raw.view(torch.float32 if f32 else torch.float16)

    def body(self):
        return self.data[: self.raw.numel() - GUARD].view(*self.shape, self.ld)

    def ptr(self, off):
        return self.data.data_ptr() + off * self.data.element_size()

    def bits(self):
        return self.raw.cpu().numpy()


def _guards_intact(slab, off, c):
    """Guard channels [0, off) and [off + c, ld) of every pixel and the region after the last pixel: sentinel."""
    bits = slab.bits()
    body = bits[: bits.size - GUARD].reshape(*slab.shape, slab.ld)
    sent = SENT32 if slab.f32 else SENT16
    sent = np.array(sent, bits.dtype)
    return bool((body[..., :off] == sent).all() and (body[..., off + c:] == sent).all() and (bits[-GUARD:] == sent).all())


def _input_unchanged(slab, off, values):
    fresh = Slab(*slab.shape, slab.ld)
    fresh.body()[..., off:off + values.shape[-1]] = torch.from_numpy(values).cuda()
    return bool(np.array_equal(slab.bits(), fresh.bits()))


def _case(name, n, h, w, cin, cout, k=3, dil=1, relu=1, aff2=False, pool=False, write_full=1, x=(0, 0), out=(8, 16),
          pool_view=(8, 16), out_f32=False, up=None, tail=False, engines=("auto", "tc_generic", "simt"), zero_cols=0):
    """x / out / pool_view = (channel offset, extra channels): the view sits at that offset of a buffer of
    c + extra channels.  up = (offset, extra) of the low-resolution tensor's buffer, or None."""
    return dict(name=name, n=n, h=h, w=w, cin=cin, cout=cout, k=k, dil=dil, relu=relu, aff2=aff2, pool=pool,
                write_full=write_full, x=x, out=out, pool_view=pool_view, out_f32=out_f32, up=up, tail=tail,
                engines=engines, zero_cols=zero_cols)


CASES = [
    # ---- fused 2x2 max-pool (halo tiles): resident and streamed filter banks, odd / even sizes, N = 1 and 3
    _case("pool_resident_16x16", 1, 16, 16, 64, 64, pool=True, write_full=0),
    _case("pool_resident_wf1_n3_17x23", 3, 17, 23, 64, 64, pool=True, write_full=1),
    _case("pool_small_9x5", 1, 9, 5, 64, 64, pool=True, write_full=0),
    _case("pool_small_n3_7x6", 3, 7, 6, 64, 64, pool=True, write_full=1),
    _case("pool_streamed_24x40", 1, 24, 40, 128, 128, pool=True, write_full=0),
    _case("pool_streamed_n3_17x15", 3, 17, 15, 128, 128, pool=True, write_full=1),
    _case("pool_odd_tile_columns_16x200", 1, 16, 200, 64, 64, pool=True, write_full=0),
    _case("crnn_conv_3_200x31", 1, 200, 31, 128, 256, aff2=True, pool=True, write_full=0),
    _case("crnn_conv_5_n3_100x15", 3, 100, 15, 256, 512, aff2=True, pool=True, write_full=0),
    # slice1.10: full output into the s1 slice of cat4 (ld 192, offset 64) + pooled p2
    _case("slice1_10_s1_and_p2", 1, 24, 40, 128, 128, pool=True, write_full=1, out=(64, 0)),
    # slice3.20 / slice4.30: input read from a concat slice, pooled output
    _case("slice3_20_in_cat3", 2, 12, 20, 256, 256, pool=True, write_full=0, x=(128, 0)),
    _case("slice4_30_in_cat2_odd", 1, 11, 13, 512, 512, pool=True, write_full=0, x=(256, 0)),
    # ---- channel slices: offsets that are multiples of 8 but not of 64, then the CRAFT concat slices
    _case("slice_ld200_off72", 2, 20, 24, 64, 64, x=(72, 64), out=(72, 64)),
    _case("slice2_17_cat3", 2, 12, 20, 256, 256, out=(128, 0)),
    _case("slice3_27_cat2", 1, 10, 14, 512, 512, out=(256, 0)),
    _case("slice4_37_cat1", 1, 6, 10, 512, 512, relu=0, out=(1024, 0)),
    _case("slice5_2_cat1", 1, 6, 10, 1024, 1024, k=1, relu=0, out=(0, 512)),
    _case("dilated_slice5_1", 1, 9, 13, 512, 1024, dil=6, relu=0),
    # ---- fp32 output: lstm_in_1 / lstm_in_2 over B * 50 rows, and one 3x3 layer
    _case("lstm_in_b1", 1, 1, 50, 128, 1024, k=1, relu=0, out=(4, 8), out_f32=True),
    _case("lstm_in_b9", 1, 1, 450, 128, 1024, k=1, relu=0, out=(4, 8), out_f32=True),
    _case("lstm_in_b257", 1, 1, 12850, 128, 1024, k=1, relu=0, out=(4, 8), out_f32=True),
    _case("f32_3x3", 2, 10, 12, 64, 64, out=(4, 8), out_f32=True, aff2=True),
    # ---- fused CRAFT tail on conv_cls.4 (32 -> 16, 3x3)
    _case("tail_n2_33x29", 2, 33, 29, 32, 16, tail=True),
    _case("tail_n2_17x9", 2, 17, 9, 32, 16, tail=True),
    # ---- upsample-add (commuted decoder upsampling): 64 / 128 channels, 1 x k and k x 1 low resolution, slices
    _case("upadd_64_low1x7_skip_in_cat4", 2, 2, 14, 128, 64, k=1, x=(64, 0), up=(0, 0), engines=("auto", "tc_generic")),
    _case("upadd_128_low6x1_skip_in_cat3", 1, 12, 2, 256, 128, k=1, x=(128, 0), up=(0, 0), engines=("auto", "tc_generic")),
    _case("upadd_64_up_in_slice_10x12", 2, 10, 12, 64, 64, k=1, up=(8, 16), engines=("auto", "tc_generic")),
    # ---- very long K / rows-as-width views
    _case("stn_dense_a_b1", 1, 1, 1, 11200, 64, k=1),
    _case("stn_dense_a_b300", 1, 1, 300, 11200, 64, k=1),
    _case("fc_9_b7", 1, 1, 350, 3584, 128, k=1),
    _case("stn_conv_a_gemm_b2", 2, 50, 7, 512, 512, k=1, relu=0, zero_cols=112),
]
CASE_IDS = [c["name"] for c in CASES]


def _inputs(case):
    rng = np.random.default_rng(zlib.crc32(case["name"].encode()))
    n, h, w, cin, cout, k = (case[q] for q in ("n", "h", "w", "cin", "cout", "k"))
    x = rng.standard_normal((n, h, w, cin)).astype(np.float16)
    wgt = (rng.standard_normal((cout, k, k, cin)) * np.sqrt(2.0 / (cin * k * k))).astype(np.float32)
    if case["zero_cols"]:
        wgt[cout - case["zero_cols"]:] = 0.0                     # the padding columns of stn.conv_a_gemm
    sign = lambda m: np.where(rng.random(m) < 0.2, -1.0, 1.0)   # noqa: E731
    s1 = (rng.uniform(0.5, 1.5, cout) * sign(cout)).astype(np.float32)
    t1 = (rng.standard_normal(cout) * 0.2).astype(np.float32)
    s2 = (rng.uniform(0.5, 1.5, cout) * sign(cout)).astype(np.float32) if case["aff2"] else None
    t2 = (rng.standard_normal(cout) * 0.2).astype(np.float32) if case["aff2"] else None
    up = rng.standard_normal((n, h // 2, w // 2, cout)).astype(np.float16) if case["up"] is not None else None
    tail = None
    if case["tail"]:
        tail = ((rng.standard_normal((16, 16)) * 0.35).astype(np.float32), (rng.standard_normal(16) * 0.1).astype(np.float32),
                (rng.standard_normal((16, 2)) * 0.3).astype(np.float32), np.array([0.5, -0.5], np.float32))
    return dict(x=x, wgt=wgt, s1=s1, t1=t1, s2=s2, t2=t2, up=up, tail=tail)


_REFS = {}


def _reference(case, d):
    if case["name"] not in _REFS:
        y, e = R.conv_ref(d["x"], d["wgt"], case["k"], case["dil"], d["s1"], d["t1"], case["relu"], d["s2"], d["t2"],
                          up=d["up"], out_f32=case["out_f32"])
        ref = {"out": (y, e)}
        if case["pool"]:
            ref["pool"] = R.pool_ref(y, e)
        if case["tail"]:
            ref["scores"] = R.tail_ref(y, *d["tail"], x_err=e)
        _REFS[case["name"]] = ref
    return _REFS[case["name"]]


def _run(ctx, case, d, engine, write_full=None):
    """One b2o_conv_test call on fresh sentinel buffers; returns the slabs."""
    n, h, w, cin, cout = (case[q] for q in ("n", "h", "w", "cin", "cout"))
    xo, xe = case["x"]
    xs = Slab(n, h, w, cin + xo + xe)
    xs.body()[..., xo:xo + cin] = torch.from_numpy(d["x"]).cuda()
    oo, oe = case["out"]
    outs = Slab(n, h, w, cout + oo + oe, f32=case["out_f32"])
    s = dict(x=xs, out=outs)
    kw = {}
    if case["pool"]:
        po, pe = case["pool_view"]
        s["pool"] = Slab(n, h // 2, w // 2, cout + po + pe)
        kw.update(pool=s["pool"].ptr(po), pool_ld=s["pool"].ld)
    if d["up"] is not None:
        uo, ue = case["up"]
        s["up"] = Slab(n, h // 2, w // 2, cout + uo + ue)
        s["up"].body()[..., uo:uo + cout] = torch.from_numpy(d["up"]).cuda()
        kw.update(up=s["up"].ptr(uo), up_ld=s["up"].ld)
    if d["tail"] is not None:
        s["scores"] = Slab(n, h, w, 2, f32=True)
        kw.update(tail=d["tail"], scores=s["scores"].ptr(0))
    wf = case["write_full"] if write_full is None else write_full
    ctx.conv_test(xs.ptr(xo), n, h, w, cin, xs.ld, d["wgt"], cout, case["k"], case["dil"], d["s1"], d["t1"], case["relu"],
                  d["s2"], d["t2"], outs.ptr(oo), outs.ld, engine, _stream(), out_f32=case["out_f32"], write_full=wf, **kw)
    torch.cuda.synchronize()
    return s


def _view(slab, off, c):
    return slab.body()[..., off:off + c].double().cpu().numpy()


def _check_values(tag, dev, ref):
    val, bound = ref
    assert np.isfinite(dev).all(), f"{tag}: unwritten (sentinel) or non-finite output"
    ratio = np.abs(dev - val) / bound
    worst = float(ratio.max())
    print(f"{tag}: worst error / bound = {worst:.3g}")
    assert worst <= 1.0, (tag, worst, np.unravel_index(int(ratio.argmax()), ratio.shape))
    return worst


def _out_is_written(case, engine):
    """The fused pool with write_full = 0 skips `out` (product path only); the tail fused into conv_cls.4's epilogue
    never writes the 16-channel map."""
    if case["pool"] and not case["write_full"] and engine == "auto":
        return False
    if case["tail"] and engine == "auto":
        return False
    return True


@pytest.fixture(scope="module")
def ctx(cuda_device):
    c = _lib.Context(0)
    yield c
    c.close()


@pytest.mark.parametrize("engine", list(ENGINES))
@pytest.mark.parametrize("case", CASES, ids=CASE_IDS)
def test_conv_epilogue_vs_fp64(ctx, case, engine):
    """Values within the per-element bound, guards untouched, fused pool == max-pool of the same run's output."""
    if engine not in case["engines"]:
        pytest.skip(f"{case['name']} is not run by the {engine} engine")
    d = _inputs(case)
    ref = _reference(case, d)
    s = _run(ctx, case, d, ENGINES[engine])
    cout, (oo, _), tag = case["cout"], case["out"], f"{case['name']}[{engine}]"
    assert _guards_intact(s["out"], oo, cout), f"{tag}: store outside the output slice"
    assert _input_unchanged(s["x"], case["x"][0], d["x"]), f"{tag}: input buffer modified"
    if case["up"] is not None:
        assert _input_unchanged(s["up"], case["up"][0], d["up"]), f"{tag}: low-resolution buffer modified"
    written = _out_is_written(case, engine)
    if written:
        _check_values(tag + " out", _view(s["out"], oo, cout), ref["out"])
    else:
        assert _guards_intact(s["out"], 0, 0), f"{tag}: out written although the route skips it"
    if case["pool"]:
        po = case["pool_view"][0]
        assert _guards_intact(s["pool"], po, cout), f"{tag}: store outside the pool slice / past PH, PW"
        pooled = _view(s["pool"], po, cout)
        _check_values(tag + " pool", pooled, ref["pool"])
        full = s["out"] if written else _run(ctx, case, d, ENGINES[engine], write_full=1)["out"]
        own = R.maxpool2_exact(full.body()[..., oo:oo + cout].cpu().numpy())
        assert np.array_equal(s["pool"].body()[..., po:po + cout].cpu().numpy().view(np.int16), own.view(np.int16)), \
            f"{tag}: fused pool != max-pool of the full output"
    if case["tail"]:
        assert _guards_intact(s["scores"], 0, 2), f"{tag}: store past the score map"
        scores = s["scores"].body().double().cpu().numpy()
        _check_values(tag + " scores", scores, ref["scores"])
        if written:                                            # head_tail_kernel route: also against its own input map
            own = R.tail_ref(_view(s["out"], oo, cout), *d["tail"])
            _check_values(tag + " scores(own map)", scores, own)


# ------------------------------------------------------------------------------ bit identity across switches
VARIANT_CASES = [c for c in CASES if c["name"] in (
    "pool_resident_wf1_n3_17x23", "pool_streamed_24x40", "pool_odd_tile_columns_16x200", "crnn_conv_3_200x31",
    "slice1_10_s1_and_p2", "slice4_30_in_cat2_odd", "slice_ld200_off72", "slice5_2_cat1", "dilated_slice5_1",
    "lstm_in_b9", "tail_n2_33x29", "tail_n2_17x9", "upadd_64_low1x7_skip_in_cat4", "stn_conv_a_gemm_b2", "fc_9_b7")]


@pytest.fixture(scope="module")
def variant_ctx(cuda_device):
    """One context per creation-time switch (each is read by b2o_create)."""
    made = {}
    for key, val in (("B2O_TC_PAIR", "1"), ("B2O_TC_PAIR", "2"), ("B2O_TC_AFF", "smem"), ("B2O_FUSED_TAIL", "0")):
        old = os.environ.get(key)
        os.environ[key] = val
        try:
            made[f"{key}={val}"] = _lib.Context(0)
        finally:
            if old is None:
                del os.environ[key]
            else:
                os.environ[key] = old
    yield made
    for c in made.values():
        c.close()


@pytest.mark.parametrize("switch", ["B2O_TC_PAIR=1", "B2O_TC_PAIR=2", "B2O_TC_AFF=smem", "B2O_FUSED_TAIL=0"])
@pytest.mark.parametrize("case", VARIANT_CASES, ids=[c["name"] for c in VARIANT_CASES])
def test_conv_epilogue_switches_bit_identical(ctx, variant_ctx, case, switch):
    """The default context and one with the switch give the same bits in every output (B2O_FUSED_TAIL=0: the tail as
    the separate head_tail_kernel over the same conv_cls.4 output)."""
    d = _inputs(case)
    a = _run(ctx, case, d, _lib.CONV_AUTO)
    b = _run(variant_ctx[switch], case, d, _lib.CONV_AUTO)
    for key in ("pool", "scores"):
        if key in a:
            assert np.array_equal(a[key].bits(), b[key].bits()), (case["name"], switch, key)
    if _out_is_written(case, "auto"):
        assert np.array_equal(a["out"].bits(), b["out"].bits()), (case["name"], switch, "out")


# ------------------------------------------------------------------------------ host-side rejections
def test_upsample_add_rejections_are_errors(ctx):
    """conv_tc_run refuses every upsample-add it has no kernel for before anything is launched; each comes back as
    B2OError and leaves every buffer as it was."""
    base = _case("reject", 1, 8, 10, 64, 64, k=1, up=(0, 0), engines=("auto",))

    def attempt(engine=_lib.CONV_AUTO, up_shift=0, up_extra=0, **over):
        case = dict(base, **over)
        d = _inputs(case)
        n, h, w, cin, cout, k = (case[q] for q in ("n", "h", "w", "cin", "cout", "k"))
        xs, outs = Slab(n, h, w, cin), Slab(n, h, w, cout, f32=case["out_f32"])
        ups = Slab(n, max(h // 2, 1), max(w // 2, 1), cout + up_extra + 8)
        kw = dict(up=ups.ptr(up_shift), up_ld=cout + up_extra)
        if case["pool"]:
            ps = Slab(n, h // 2, w // 2, cout)
            kw.update(pool=ps.ptr(0), pool_ld=cout)
        if case["tail"]:
            sc = Slab(n, h, w, 2, f32=True)
            kw.update(tail=d["tail"], scores=sc.ptr(0))
        before = outs.bits()
        with pytest.raises(_lib.B2OError):
            ctx.conv_test(xs.ptr(0), n, h, w, cin, cin, d["wgt"], cout, k, 1, d["s1"], d["t1"], 1, None, None,
                          outs.ptr(0), cout, engine, _stream(), out_f32=case["out_f32"], **kw)
        torch.cuda.synchronize()
        assert np.array_equal(outs.bits(), before)

    attempt(k=3)                                  # not a 1x1 layer
    attempt(cin=32)                               # 32-channel K chunks
    attempt(cout=32)                              # N tile below 64
    attempt(out_f32=True)                         # fp32 output
    attempt(pool=True)                            # with a fused pool
    attempt(cout=16, cin=32, tail=True)          # with the fused tail
    attempt(h=9)                                  # odd height: the low-resolution map is not exactly half
    attempt(w=11)                                 # odd width
    attempt(up_extra=4)                           # low-resolution channel stride not a multiple of 8
    attempt(up_shift=4)                           # low-resolution tensor not 16-byte aligned
    attempt(engine=_lib.CONV_SIMT)                # the SIMT engine has no upsample-add
