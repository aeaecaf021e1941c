"""The CRAFT forward measured stage by stage: ``b2o_craft_forward_until`` stops after each step k, ``b2o_craft_tap`` reads
every buffer live at k, and each step's output is compared with an fp64 reference of that step alone, computed from the
device's OWN inputs (tests/stage_refs.py: CRAFT_STEPS restates the step table, CRAFT_BUFS plan_craft's lifetimes).  The
BN layers are folded here, in fp64, from the raw ``.pth``-named weights, never read back from the device.

Per step (the worst error / bound ratio of every stage is printed):

* normalize16: the fp16 channels 0..2 are exactly fp16(compute_input) with numpy float32 semantics; channels 3..15 are 0.
* stem (tensor-core stem16 / SIMT stem_rgb_kernel): the conv bound on the exact operand (the fp16 x16 tap; the fp32
  normalisation for the SIMT stem, whose 3-channel weights build_layer keeps in fp32), and again against the fp64
  normalisation with the fp32 / fp16 rounding of the input propagated as ``x_err``.
* every convolution: ``stage_refs.conv_ref``; a pooled output within the largest of its window's bounds, and bit equal to
  the 2x2 max of the full output where the engine writes it.
* maxpool3s1: bit exact.  upsample (upsample_kernel / upsample2x_kernel): float32 coordinates as the kernel forms them,
  blend in fp64, one fp16 half-ulp plus 4 * 2^-24 * sum|w * v| (the difference from fp64-coordinate F.interpolate is
  printed); commuted levels (B2O_UPCONV_COMMUTE=1): the low-resolution half z and the upsample-add convolution.
* conv_cls.4 + tail: the scores against the tail of the conv_cls.4 reference (fused tail), or the separate head tail
  against the device's own h3.

Besides the values: a buffer's written channels are bit-identical at every step of its lifetime after the one that
writes them (a buffer that shares memory with another one would be overwritten), hold no sentinel, the guard after the
workspace and around the scores is never touched, forward_until(30) is b2o_craft_forward bit for bit, and taps outside a
lifetime are refused.  The bench shape (32, 1536, 1536) runs on images 0 and 31, on row bands at the top and bottom of
every level (the conv references on those bands, their halo rows discarded).

Measured on an H100 80GB HBM3 (400 W power limit), worst error / bound over every size and engine: normalize16,
maxpool3s1 and every pool against the max of its full map exact; stem16 0.96 (0.955 against the fp64 normalisation),
stem_rgb 0.985 (0.985); encoder convs 0.87 (slice1.3) down to 0.09 (slice4.34), slice4.37 0.11, slice5.1 0.13, slice5.2
0.43; pooled outputs at most 0.87; decoder convs 0.12 to 0.95, the commuted low-resolution halves 0.96; head convs 0.85;
upsample and upsample2x 1.0 (a blend landing exactly on an fp16 midpoint rounds by exactly the half-ulp term, with
device - F.interpolate at most 0.0039); scores 0.086 against the tail of the conv_cls.4 reference (fused tail) and
0.0052 against the device's own h3 (head_tail_kernel).  CRNN backbone: conv_1 0.98, conv_2 0.71, conv_3 0.76 (pool
0.58), conv_4 .. conv_7 at most 0.21.
The per-element bound of a deep layer is sized for the worst case of a K = 4608 fp32 accumulation, several times the
realised error, so a constant shift of a whole channel by less than that (a BN shift folded 1 % off) fits under it.
Every convolution output (stems, encoder, decoder, commuted halves, head; the CRNN convs) is therefore also checked
per channel for a systematic error: the signed mean of device - reference over the channel's distinct values must stay
within (mean bound + 1.75 fp16 ulp) / sqrt(N) + 2^-16 mean |reference| (``_mean_check``).  Measured worst |mean| /
allowance: 0.70 (upconv4.conv.0), 0.35 or less in every other layer, 0.08 for slice4.37; slice4.37's folded BN shift
scaled by 1.01 gives 1.00 to 1.17 at 2 x 144 x 200, 2 x 160 x 224, 1 x 32 x 2048 and 1 x 2048 x 40, and 1.55 at the
bench shape, on every engine.
"""
import os

import numpy as np
import pytest
import torch

from keras_ocr_b200 import _lib
from keras_ocr_b200 import weights as W
from tests import stage_refs as R

pytestmark = pytest.mark.gpu

SENT16 = 0x7E5A                  # fp16 NaN: the workspace and every tap start as this bit pattern
SENT32 = 0x7FA5A5A5              # fp32 NaN for the scores
GUARD = 1 << 16                  # bytes after the workspace
SGUARD = 4096                    # floats before and after the scores
BAND, GAP = 8, 8                 # bench shape: rows per band at every level, NaN rows between the top and bottom band
LAST = _lib.CRAFT_LAST_STEP
CONFIGS = {"auto": (_lib.CONV_AUTO, False), "tc_generic": (_lib.CONV_TC_GENERIC, False), "simt": (_lib.CONV_SIMT, False),
           "auto_commute": (_lib.CONV_AUTO, True)}
SIZES = [(1, 32, 32), (2, 33, 47), (2, 144, 200), (2, 160, 224), (1, 32, 2048), (1, 2048, 40)]
WORST = {}                       # (stage) -> worst ratio over every case, printed by the last test


def _stream():
    return torch.cuda.current_stream().cuda_stream


class Band:
    """Rows ``rows`` (real row index, -1 for a NaN gap row) of an (n, H, W, C) map: data (n, len(rows), W, C)."""

    def __init__(self, data, rows):
        self.data, self.rows = data, np.asarray(rows)


def _band_rows(h, banded):
    if not banded or h < 2 * BAND + GAP:
        return np.arange(h)
    return np.concatenate([np.arange(BAND), np.full(GAP, -1), np.arange(h - BAND, h)])


def _select(t, images, rows):
    """Device tensor (n, H, ...) -> float32 host numpy of the selected images and rows, gap rows NaN (int16 bit
    patterns are exact in float32)."""
    idx = torch.as_tensor(np.maximum(rows, 0), device=t.device)
    out = t[torch.as_tensor(images, device=t.device)][:, idx].cpu().numpy().astype(np.float32)
    out[:, rows < 0] = np.nan
    return out


def _pooled_rows(rows):
    """Row map of a 2x2 pool of a band: pair (2r, 2r + 1) -> r, anything else a gap."""
    m = len(rows) // 2
    a, b = rows[0:2 * m:2], rows[1:2 * m:2]
    return np.where((a >= 0) & (a % 2 == 0) & (b == a + 1), a // 2, -1)


def _pool(val, bound, rows):
    pv, pb = R.pool_ref(val, bound)
    pr = _pooled_rows(rows)
    pv[:, pr < 0] = np.nan
    return pv, pb, pr


MEAN_MIN = 64                    # distinct values a channel needs before its mean error is judged


def _mean_check(tag, d, v, bound, fin):
    """Per output channel, the signed mean of device - reference over the channel's distinct nonzero reference values
    (a flat image region repeats one value, and with it one rounding error, over many pixels: it counts once).  The
    output rounding and the fp32 accumulation errors have no common sign across distinct values, so their mean shrinks
    like 1 / sqrt(N); a misfolded or shifted epilogue constant moves every element of the channel the same way and
    does not.  Allowed: (mean bound + 1.75 mean fp16 ulp) / sqrt(N) -- the ulp term is six standard deviations of the
    mean of N independent round-to-nearest errors -- plus 2^-16 mean |reference| for the tensor cores' truncating
    adds.  Returns the worst ratio of |mean error| to that allowance over the channels with at least MEAN_MIN values."""
    c = v.shape[-1]
    dd, vv, bb, ff = (a.reshape(-1, c) for a in (d, np.where(fin, v, 0.0), bound, fin))
    worst = 0.0
    for ch in range(c):
        keep = ff[:, ch] & (vv[:, ch] != 0)
        vals, first = np.unique(vv[keep, ch], return_index=True)
        if vals.size < MEAN_MIN:
            continue
        idx = np.nonzero(keep)[0][first]
        err = float(np.mean(dd[idx, ch] - vv[idx, ch]))
        allowed = (np.mean(bb[idx, ch]) + 1.75 * np.mean(R.ulp16(vv[idx, ch]))) / np.sqrt(idx.size) \
            + 2.0 ** -16 * np.mean(np.abs(vv[idx, ch]))
        r = abs(err) / allowed
        assert r <= 1.0, (tag, "systematic error in channel", ch, err, allowed)
        worst = max(worst, r)
    return worst


def _check(tag, dev, val, bound, rows, h, exact=False, mean=False):
    """dev (a Band, float64) against (val, bound) on rows ``rows``; compared where val is finite.  Rows 0 and h - 1 of
    the level must be among the compared rows.  mean: also the per-channel systematic error (``_mean_check``).
    Returns the worst ratio (0 for an exact check)."""
    pos = {int(r): i for i, r in enumerate(dev.rows) if r >= 0}
    keep = [(i, pos[int(r)]) for i, r in enumerate(rows) if r >= 0 and int(r) in pos]
    ri, di = np.array([k[0] for k in keep]), np.array([k[1] for k in keep])
    v, d = val[:, ri], dev.data[:, di]
    fin = np.isfinite(v)
    full_rows = set(int(rows[i]) for j, i in enumerate(ri) if fin[:, j].all())
    assert {0, h - 1} <= full_rows, (tag, "first / last row not compared")
    assert np.isfinite(d[fin]).all(), (tag, "NaN (sentinel or stale) where the stage writes")
    if exact:
        assert np.array_equal(d[fin], v[fin]), tag
        r = 0.0
    else:
        err, b = np.abs(d[fin] - v[fin]), bound[:, ri][fin]
        ratio = np.divide(err, b, out=np.where(err > 0, np.inf, 0.0), where=b > 0)     # a zero bound allows no error
        r = float(ratio.max())
        if r > 1.0:
            where = np.argwhere(fin)[int(ratio.argmax())]
            print(f"{tag}: FAIL at (image, band row, col, channel) {tuple(where)}: device {d[fin][ratio.argmax()]}, "
                  f"reference {v[fin][ratio.argmax()]}, bound {b[ratio.argmax()]}, {int((ratio > 1).sum())} elements out")
        assert r <= 1.0, (tag, r)
    print(f"{tag}: worst error / bound = {r:.3g}")
    key = tag.split(" ")[-1]
    WORST[key] = max(WORST.get(key, 0.0), r)
    if mean:
        m = _mean_check(tag, d, v, bound[:, ri], fin)
        print(f"{tag}: worst per-channel mean error / allowance = {m:.3g}")
        WORST[key + " mean"] = max(WORST.get(key + " mean", 0.0), m)
    return r


class Forward:
    """One context, one input batch: runs forward_until(k) on a sentinel-filled workspace and taps its buffers."""

    def __init__(self, ctx, img, banded=False):
        self.ctx, self.img_host = ctx, img
        self.n, self.h, self.w = img.shape[:3]
        self.img = torch.from_numpy(img).cuda()
        self.dims = R.craft_dims(self.h, self.w)
        self.nbytes = ctx.craft_workspace_bytes(self.n, self.h, self.w)
        self.ws = torch.empty(self.nbytes + GUARD, dtype=torch.uint8, device="cuda")
        h2, w2 = self.dims[2]
        self.n_scores = self.n * h2 * w2 * 2
        self.scores = torch.empty(self.n_scores + 2 * SGUARD, dtype=torch.float32, device="cuda")
        big = max(self.n * self.dims[lv][0] * self.dims[lv][1] * c * 2 for lv, c, _f, _l in R.CRAFT_BUFS.values())
        self.scratch = torch.empty(big, dtype=torch.uint8, device="cuda")
        self.images = [0, self.n - 1] if banded else list(range(self.n))
        self.rows = {lv: _band_rows(self.dims[lv][0], banded) for lv in self.dims}

    def run(self, k):
        self.ws.view(torch.int16).fill_(SENT16)
        self.scores.view(torch.int32).fill_(SENT32)
        self.ctx.craft_forward_until(self.img.data_ptr(), self.n, self.h, self.w, self.scores[SGUARD:].data_ptr(),
                                     self.ws.data_ptr(), self.nbytes, k, _stream())
        torch.cuda.synchronize()
        assert bool((self.ws[self.nbytes:].view(torch.int16) == SENT16).all()), "write past the workspace"
        g = self.scores.view(torch.int32)
        assert bool((g[:SGUARD] == SENT32).all() and (g[SGUARD + self.n_scores:] == SENT32).all()), "write around scores"

    def tap(self, name):
        lv, c, _f, _l = R.CRAFT_BUFS[name]
        hh, ww = self.dims[lv]
        nbytes = self.n * hh * ww * c * 2
        self.ctx.craft_tap(name, self.ws.data_ptr(), self.n, self.h, self.w, self.scratch.data_ptr(), self.scratch.numel(),
                           _stream())
        return _select(self.scratch[:nbytes].view(torch.int16).view(self.n, hh, ww, c), self.images, self.rows[lv])

    def scores_band(self):
        h2, w2 = self.dims[2]
        t = self.scores[SGUARD:SGUARD + self.n_scores].view(self.n, h2, w2, 2)
        return Band(_select(t, self.images, self.rows[2]), self.rows[2])

    def scores_untouched(self):
        return bool((self.scores.view(torch.int32)[SGUARD:SGUARD + self.n_scores] == SENT32).all())


def _as_half(bits):
    """int16 bit patterns held in float32 (gap rows NaN) -> fp16 values as float64 (gap rows NaN)."""
    gap = np.isnan(bits)
    h = np.where(gap, 0, bits).astype(np.int16).view(np.float16).astype(np.float64)
    h[gap] = np.nan
    return h


def _commuted(engine, commute, dims, st):
    lv_src, lv_skip = R.CRAFT_BUFS[st.get("y", st["src"])[0]][0], R.CRAFT_BUFS[st["skip"][0]][0]
    (sh, sw), (kh, kw) = dims[lv_src], dims[lv_skip]
    return engine == _lib.CONV_AUTO and commute and kh == 2 * sh and kw == 2 * sw


def _written(st, engine, commute, dims):
    """Slices (buf, c0, c1) step ``st`` writes on this path."""
    kind = st["kind"]
    if kind == "normalize":
        return [st["out"]] if engine != _lib.CONV_SIMT else []
    if kind == "tail":
        return []
    if kind == "up":
        return [st["z"] if _commuted(engine, commute, dims, st) else st["out"]]
    if st["step"] == 29 and engine == _lib.CONV_AUTO:
        return []                                                               # the fused tail stores only the scores
    out = [st["out"]]
    if st.get("pool"):
        out = ([st["out"]] if st["full"] or engine != _lib.CONV_AUTO else []) + [st["pool"]]
    return out


def _live(k):
    return [name for name, (_lv, _c, first, last) in R.CRAFT_BUFS.items() if first <= k <= last]


def _stage(f, w, st, taps, engine, commute, tag):
    """Check step ``st`` from the taps of the same forward (taps: name -> int16 bits held in float32)."""
    kind, dims, rows = st["kind"], f.dims, f.rows

    def get(s):
        lv = R.CRAFT_BUFS[s[0]][0]
        return Band(_as_half(taps[s[0]][..., s[1]:s[2]]), rows[lv])

    def lvl(s):
        return R.CRAFT_BUFS[s[0]][0]

    out = []
    if kind in ("normalize", "stem"):
        img = np.asarray(f.img_host[f.images], np.float64)[:, np.maximum(rows[1], 0)]
        img[:, rows[1] < 0] = np.nan
        x32, x64 = R.compute_input_f32(img), (img - R.CRAFT_MEAN) / R.CRAFT_STD
    if kind == "normalize":
        if engine == _lib.CONV_SIMT:
            return out                                                           # the SIMT stem normalises itself
        dev = get(st["out"])
        want = Band(np.concatenate([R.f16(x32), np.zeros(x32.shape[:3] + (13,))], -1), rows[1])
        out.append(_check(f"{tag} normalize16", dev, want.data, None, rows[1], dims[1][0], exact=True))
        return out
    if kind == "stem":
        dev = get(st["out"])
        if engine == _lib.CONV_SIMT:
            val, bnd = R.craft_layer_ref(w, "basenet.slice1.0", x32.astype(np.float32).astype(np.float64), round_w=False)
            out.append(_check(f"{tag} stem_rgb", dev, val, bnd, rows[1], dims[1][0], mean=True))
            val, bnd = R.craft_layer_ref(w, "basenet.slice1.0", x64, round_w=False, x_err=np.abs(x32 - x64))
            out.append(_check(f"{tag} stem_rgb_vs_fp64_input", dev, val, bnd, rows[1], dims[1][0]))
        else:
            x16 = get(st["src"])
            val, bnd = R.craft_layer_ref(w, "basenet.slice1.0", x16.data, stem16=True)
            out.append(_check(f"{tag} stem16", dev, val, bnd, rows[1], dims[1][0], mean=True))
            err = np.concatenate([np.abs(R.f16(x32) - x64), np.zeros(x64.shape[:3] + (13,))], -1)
            x64p = np.concatenate([x64, np.zeros(x64.shape[:3] + (13,))], -1)
            val, bnd = R.craft_layer_ref(w, "basenet.slice1.0", x64p, x_err=err, stem16=True)
            out.append(_check(f"{tag} stem16_vs_fp64_input", dev, val, bnd, rows[1], dims[1][0]))
        return out
    if kind == "maxpool3":
        src = get(st["src"])
        out.append(_check(f"{tag} maxpool3s1", get(st["out"]), R.maxpool3s1_exact(src.data), None, src.rows,
                          dims[16][0], exact=True))
        return out
    if kind == "up":
        src = get(st["src"])
        lo, ls = lvl(st["out"]), lvl(st["src"])
        if _commuted(engine, commute, dims, st):
            cy = st["out"][2] - st["out"][1]
            val, bnd = R.craft_layer_ref(w, st["layer"], src.data, cols=(0, cy))
            out.append(_check(f"{tag} upconv_low_half", get(st["z"]), val, bnd, src.rows, dims[ls][0], mean=True))
            return out
        oh, ow = dims[lo]
        val, bnd = R.upsample_ref(src.data, src.rows, dims[ls][0], np.maximum(rows[lo], 0), oh, ow)
        val[:, rows[lo] < 0] = np.nan
        kname = "upsample2x" if (oh, ow) == (2 * dims[ls][0], 2 * dims[ls][1]) else "upsample"
        out.append(_check(f"{tag} {kname}", get(st["out"]), val, bnd, rows[lo], oh))
        if not (rows[ls] < 0).any():
            ref = R._nhwc(R.upsample_like(R._nchw(src.data), oh, ow))
            print(f"{tag} {kname}: max |device - F.interpolate (fp64 coordinates)| = "
                  f"{np.abs(get(st['out']).data - ref).max():.3g}")
        return out
    if kind == "tail":
        if engine == _lib.CONV_AUTO:
            return out
        h3 = get(st["src"])
        val, bnd = R.craft_tail_ref(w, h3.data)
        out.append(_check(f"{tag} head_tail", f.scores_band(), val, bnd, rows[2], dims[2][0]))
        return out
    # convolutions
    if kind == "upconv" and _commuted(engine, commute, dims, st):
        skip, z = get(st["skip"]), get(st["z"])
        cy = st["skip"][1]
        val, bnd = R.craft_layer_ref(w, st["layer"], skip.data, cols=(cy, R.CRAFT_LAYERS[st["layer"]][0]), up=z.data)
        src = skip
    else:
        src = get(st["src"])
        val, bnd = R.craft_layer_ref(w, st["layer"], src.data)
    lo = lvl(st["out"])
    name = st["layer"]
    if st["step"] == 29 and engine == _lib.CONV_AUTO:               # fused tail: scores from the conv_cls.4 reference
        sv, sb = R.craft_tail_ref(w, val, x_err=bnd)
        out.append(_check(f"{tag} conv_cls.4+fused_tail", f.scores_band(), sv, sb, src.rows, dims[2][0]))
        return out
    if st["out"] in _written(st, engine, commute, dims):
        out.append(_check(f"{tag} {name}", get(st["out"]), val, bnd, src.rows, dims[lo][0], mean=True))
    if st.get("pool"):
        pv, pb, pr = _pool(val, bnd, src.rows)
        lp = lvl(st["pool"])
        out.append(_check(f"{tag} {name}.pool", get(st["pool"]), pv, pb, pr, dims[lp][0]))
        if st["out"] in _written(st, engine, commute, dims):
            full = get(st["out"])
            mv, _mb, mr = _pool(full.data, full.data, full.rows)
            out.append(_check(f"{tag} {name}.pool_is_max_of_full", get(st["pool"]), mv, None, mr, dims[lp][0], exact=True))
    return out


def _run_all_steps(f, w, engine, commute, tag):
    """Every step k: forward_until(k), every live buffer tapped, the stage checked, writes held over the lifetime."""
    held = {}                                                          # (buf, c0, c1) -> bits at the writing step
    for st in R.CRAFT_STEPS:
        k = st["step"]
        f.run(k)
        taps = {name: f.tap(name) for name in _live(k)}
        _stage(f, w, st, taps, engine, commute, tag)
        for s in _written(st, engine, commute, f.dims):
            bits = taps[s[0]][..., s[1]:s[2]]
            fin = ~np.isnan(bits)
            assert not (bits[fin] == SENT16).any(), (tag, k, s, "sentinel left")
            held[s] = bits
        for s, bits in held.items():
            if s[0] in taps:
                assert np.array_equal(taps[s[0]][..., s[1]:s[2]], bits, equal_nan=True), (tag, k, s, "overwritten")
        fused = engine == _lib.CONV_AUTO
        assert f.scores_untouched() == (k < (29 if fused else 30)), (tag, k, "scores written at the wrong step")


_CTX = {}


def _context(config, wkey, weights):
    if (config, wkey) not in _CTX:
        engine, commute = CONFIGS[config]
        old = os.environ.pop("B2O_UPCONV_COMMUTE", None)
        if commute:
            os.environ["B2O_UPCONV_COMMUTE"] = "1"
        try:
            ctx = _lib.Context(0)
        finally:
            os.environ.pop("B2O_UPCONV_COMMUTE", None)
            if old is not None:
                os.environ["B2O_UPCONV_COMMUTE"] = old
        ctx.load_craft(weights[wkey])
        ctx.set_conv_engine(engine)
        _CTX[(config, wkey)] = ctx
    return _CTX[(config, wkey)]


@pytest.fixture(scope="module")
def weights():
    return {"seed3": W.synthetic_craft_weights(3), "textlike": W.synthetic_craft_weights(3, textlike=True)}


def _image(n, h, w, seed):
    rng = np.random.default_rng(seed)
    img = rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8)
    img[:, : h // 3, : w // 3] = 255                               # flat white and black corners: ReLU-dead regions
    img[:, -(h // 4):, -(w // 4):] = 0
    return img


@pytest.mark.parametrize("config", list(CONFIGS))
@pytest.mark.parametrize("size", SIZES, ids=lambda s: "x".join(map(str, s)))
def test_craft_stages(cuda_device, weights, config, size):
    wkey = "textlike" if size == (2, 144, 200) else "seed3"
    engine, commute = CONFIGS[config]
    ctx = _context(config, wkey, weights)
    f = Forward(ctx, _image(*size, seed=sum(size)))
    _run_all_steps(f, weights[wkey], engine, commute, f"{config} {size}")


def test_craft_stages_bench_shape(cuda_device, weights):
    """32 x 1536 x 1536 (the bench step's detector batch, element offsets into a / b past 2^32): images 0 and 31, the
    first and last BAND rows of every level."""
    ctx = _context("auto", "seed3", weights)
    f = Forward(ctx, _image(32, 1536, 1536, seed=7), banded=True)
    _run_all_steps(f, weights["seed3"], _lib.CONV_AUTO, False, "auto (32, 1536, 1536)")


@pytest.mark.parametrize("config", list(CONFIGS))
def test_forward_until_last_is_forward_and_taps_are_refused_outside_lifetimes(cuda_device, weights, config):
    ctx = _context(config, "seed3", weights)
    f = Forward(ctx, _image(2, 33, 47, seed=3))
    f.run(LAST)
    until = f.scores.clone()
    f.scores.view(torch.int32).fill_(SENT32)
    f.ws.view(torch.int16).fill_(SENT16)
    ctx.craft_forward(f.img.data_ptr(), f.n, f.h, f.w, f.scores[SGUARD:].data_ptr(), f.ws.data_ptr(), f.nbytes, _stream())
    torch.cuda.synchronize()
    assert torch.equal(until.view(torch.int32), f.scores.view(torch.int32))
    assert bool((f.ws[f.nbytes:].view(torch.int16) == SENT16).all())
    ptr, cap = f.scratch.data_ptr(), f.scratch.numel()
    for k, dead, alive in [(5, "a", "cat4"), (5, "e", "p2"), (12, "d", "cat1"), (LAST, "h2", "h3")]:
        f.run(k)
        f.ctx.craft_tap(alive, f.ws.data_ptr(), f.n, f.h, f.w, ptr, cap, _stream())
        with pytest.raises(_lib.B2OError, match=r"\(-5\)"):
            f.ctx.craft_tap(dead, f.ws.data_ptr(), f.n, f.h, f.w, ptr, cap, _stream())
    for ws, n, h, w in [(f.ws.data_ptr() + 256, f.n, f.h, f.w), (f.ws.data_ptr(), f.n + 1, f.h, f.w),
                        (f.ws.data_ptr(), f.n, f.h + 1, f.w), (f.ws.data_ptr(), f.n, f.h, 64)]:
        with pytest.raises(_lib.B2OError, match=r"\(-5\)"):          # not the last forward's workspace or shape
            f.ctx.craft_tap("h3", ws, n, h, w, ptr, cap, _stream())
    with pytest.raises(_lib.B2OError, match=r"\(-2\)"):
        f.ctx.craft_tap("nope", f.ws.data_ptr(), f.n, f.h, f.w, ptr, cap, _stream())
    with pytest.raises(_lib.B2OError, match=r"\(-2\)"):
        f.ctx.craft_tap("h3", f.ws.data_ptr(), f.n, f.h, f.w, ptr, 16, _stream())
    with pytest.raises(_lib.B2OError, match=r"\(-2\)"):
        f.ctx.craft_forward_until(f.img.data_ptr(), f.n, f.h, f.w, f.scores[SGUARD:].data_ptr(), f.ws.data_ptr(),
                                  f.nbytes, LAST + 1, _stream())


# ------------------------------------------------------------------------------------------ CRNN conv backbone
CRNN_ENGINES = {"auto": _lib.CONV_AUTO, "tc_generic": _lib.CONV_TC_GENERIC, "simt": _lib.CONV_SIMT}
CRNN_SHAPES = {"in": (200, 31), "x1": (200, 31, 64), "x2": (200, 31, 128), "x3": (200, 31, 256), "p3": (100, 15, 256),
               "x4": (100, 15, 256), "x5": (100, 15, 512), "p5": (50, 7, 512), "x6": (50, 7, 512),
               "features": (50, 7, 512)}


@pytest.mark.parametrize("color", [False, True], ids=["gray", "color"])
@pytest.mark.parametrize("engine", list(CRNN_ENGINES))
@pytest.mark.parametrize("b", [1, 9, 257])
def test_crnn_backbone_stages(cuda_device, b, engine, color):
    """conv_1 (stem_crnn_kernel, gray and color) .. conv_7 and both fused pools, each from the device's own input (crops
    0, b // 2 and b - 1 of the batch), BN (Keras eps 1e-3, after the ReLU) folded here from the raw weights."""
    from keras_ocr_b200.recognition import Recognizer
    w = W.synthetic_crnn_weights(seed=2, color=color)
    rec = Recognizer(weights=w, build_params={"color": color})
    rec.ctx.set_conv_engine(CRNN_ENGINES[engine])
    rec.keep_workspace = True
    rng = np.random.default_rng(b)
    ch = 3 if color else 1
    crops = rng.integers(0, 256, (b, 31, 200) + ((3,) if color else ()), dtype=np.uint8)
    crops[:, :, 150:] = 0
    x = torch.empty((b, 200, 31) + ((3,) if color else ()), dtype=torch.float16, device="cuda")
    rec.ctx.crops_to_input(torch.from_numpy(crops).cuda().data_ptr(), b, x.data_ptr(), _stream(), color=color)
    rec.predict_device(x)
    sel = sorted({0, b // 2, b - 1})
    taps = {"in": x.double().cpu().numpy().reshape(b, 200, 31, ch)[sel]}
    for name, shape in CRNN_SHAPES.items():
        if name != "in" and not (name in ("x3", "x5") and engine == "auto"):
            taps[name] = rec.tap(name, (b,) + shape, torch.float16).double().cpu().numpy()[sel]
    for layer, src, dst, pool in R.CRNN_STEPS:
        val, bnd = R.crnn_layer_ref(w, layer, taps[src])
        tag = f"crnn b={b} {engine} {'color' if color else 'gray'} {layer}"
        rows = np.arange(val.shape[1])
        if dst in taps:
            _check(tag, Band(taps[dst], rows), val, bnd, rows, val.shape[1], mean=True)
        if pool:
            pv, pb, pr = _pool(val, bnd, rows)
            _check(tag + ".pool", Band(taps[pool], pr), pv, pb, pr, pv.shape[1])
            if dst in taps:
                mv, _mb, mr = _pool(taps[dst], taps[dst], rows)
                _check(tag + ".pool_is_max_of_full", Band(taps[pool], mr), mv, None, mr, mv.shape[1], exact=True)


def test_print_worst_ratios():
    """Runs last: the worst error / bound ratio of every stage over all the cases above."""
    for key in sorted(WORST):
        print(f"worst {key}: {WORST[key]:.3g}")
