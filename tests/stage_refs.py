"""fp64 CPU references of single CUDA stages, with per-element error bounds derived from the kernels' arithmetic.

Used by tests/test_gpu_conv_epilogues.py and tests/test_gpu_crnn_stages.py; checked on their own (no GPU) by
tests/test_stage_refs.py.  Every reference takes the values the kernel really sees (fp16-rounded activations and
weights) and returns ``(value, bound)``: the device result must satisfy ``|dev - value| <= bound`` element by element.

Bound of one convolution output (fp32 accumulation of K = taps * cin exact fp16 x fp16 products):
    e_acc = GAMMA(K) * sum|x * w|                          (GAMMA(K) = (K + 32) * 2^-23, see ``gamma``)
    e1    = e_acc * |s1| + 2^-24 * (|acc * s1| + |t1|)        (one fmaf)
    e2    = e1 * |s2| + 2^-24 * (|y1 * s2| + |t2|)            (second affine, CRNN convs; ReLU is 1-Lipschitz)
    fp16  : e = e2 * (1 + 2^-10) + 2^-11 * |y| + 2^-25      (round to nearest, subnormal floor)
A 2x2 max-pool output takes the largest of its four window bounds (|max a' - max a| <= max |a' - a|).
"""
import numpy as np
import torch
import torch.nn.functional as F

from keras_ocr_b200.weights import CRAFT_CONVS, CRNN_CONVS

U32 = 2.0 ** -24          # unit roundoff of fp32
U16 = 2.0 ** -11          # unit roundoff of fp16
SUB16 = 2.0 ** -25        # half the spacing of fp16 subnormals


def gamma(k):
    """Error factor of an fp32 sum of k exact products: 2^-23 per addition covers round-to-nearest adders and the
    tensor cores' aligned, truncating adds; the 32 extra terms cover one k16 block's internal alignment twice over."""
    return (k + 32) * 2.0 ** -23


def f16(a):
    """Round to fp16 and return float64 (numpy or torch)."""
    if isinstance(a, torch.Tensor):
        return a.to(torch.float16).to(torch.float64)
    return np.asarray(a, np.float64).astype(np.float16).astype(np.float64)


def _nchw(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float64)).permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous().numpy()


def _col(v):
    return torch.from_numpy(np.asarray(v, np.float64))[None, :, None, None]


def upsample_like(u_nchw, h, w):
    """UpsampleLike (oracle/craft.py::_upsample_like): bilinear, half-pixel centres."""
    return F.interpolate(u_nchw, size=(h, w), mode="bilinear", align_corners=False)


def conv_ref(x, wgt, k, dil, s1, t1, relu, s2=None, t2=None, up=None, out_f32=False, x_err=None, aff_err=None,
             round_w=True):
    """One convolution layer of the engine in fp64.  x (n,h,w,cin) and up (n,h/2,w/2,cout) hold fp16 values;
    wgt (cout,k,k,cin) is rounded to fp16 here (as build_layer does; round_w=False keeps the fp32 weights of the
    CUDA-core stems).  x_err: optional per-element bound on the input (propagated through |w|).  aff_err: optional
    per-channel bounds (s1, t1, s2, t2) on the device's own fp32 folding of s1 / t1 / s2 / t2 (``fold_err``).
    Returns NHWC float64 (value, bound)."""
    n, h, w, cin = x.shape
    xt = _nchw(x)
    wt = torch.from_numpy(np.ascontiguousarray(wgt, np.float32)).permute(0, 3, 1, 2).double()
    wt = f16(wt) if round_w else wt
    pad = dil * (k // 2)
    z = F.conv2d(xt, wt, padding=pad, dilation=dil)
    mag = F.conv2d(xt.abs(), wt.abs(), padding=pad, dilation=dil)
    terms = k * k * cin
    if up is not None:
        ut = _nchw(up)
        z = z + upsample_like(ut, h, w)
        mag = mag + upsample_like(ut.abs(), h, w)
        terms += 8                                          # the fp32 blend and its addition to the accumulator
    e = gamma(terms) * mag
    if x_err is not None:
        e = e + F.conv2d(_nchw(x_err), wt.abs(), padding=pad, dilation=dil)
    y = z * _col(s1) + _col(t1)
    e = e * _col(np.abs(s1)) + U32 * ((z * _col(s1)).abs() + _col(np.abs(t1)))
    if aff_err is not None:
        e = e + z.abs() * _col(aff_err[0]) + _col(aff_err[1])
    if relu:
        y = y.clamp_min(0.0)
    if s2 is not None:
        e = e * _col(np.abs(s2)) + U32 * ((y * _col(s2)).abs() + _col(np.abs(t2)))
        if aff_err is not None:
            e = e + y.abs() * _col(aff_err[2]) + _col(aff_err[3])
        y = y * _col(s2) + _col(t2)
    if not out_f32:
        e = e * (1 + 2 * U16) + U16 * y.abs() + SUB16
    return _nhwc(y), _nhwc(e)


def pool_ref(y, e):
    """2x2 / stride-2 max pool (floor for odd sizes) of a value and its bound."""
    return _nhwc(F.max_pool2d(_nchw(y), 2, 2)), _nhwc(F.max_pool2d(_nchw(e), 2, 2))


def maxpool2_exact(a):
    """2x2 / stride-2 max pool of an fp16 array (n,h,w,c), floor for odd sizes: exact."""
    n, h, w, c = a.shape
    a = a[:, : h // 2 * 2, : w // 2 * 2]
    return a.reshape(n, h // 2, 2, w // 2, 2, c).max(axis=(2, 4))


def tail_ref(x, w6, b6, w8, b8, x_err=None, round_w=True):
    """CRAFT head tail conv_cls.6 (1x1 16->16, ReLU) + conv_cls.8 (1x1 16->2) on a 16-channel map x (n,h,w,16).
    w6 (16 in, 16 out) and w8 (16 in, 2 out) are rounded to fp16 here; b6 / b8 stay fp32.  Both layers are serial
    fmaf chains of 16 terms in fp32; x_err (the bound on x) is propagated through |w6| and |w8|.  Returns (scores, bound)."""
    x = np.asarray(x, np.float64)
    w6, w8 = (f16(w6), f16(w8)) if round_w else (np.asarray(w6, np.float64), np.asarray(w8, np.float64))
    b6, b8 = np.asarray(b6, np.float64), np.asarray(b8, np.float64)
    ex = np.zeros_like(x) if x_err is None else np.asarray(x_err, np.float64)
    pre = x @ w6 + b6
    ea = ex @ np.abs(w6) + gamma(17) * ((np.abs(x) + ex) @ np.abs(w6) + np.abs(b6))
    a = np.maximum(pre, 0.0)
    o = a @ w8 + b8
    eo = ea @ np.abs(w8) + gamma(17) * ((a + ea) @ np.abs(w8) + np.abs(b8))
    return o, eo


# ------------------------------------------------------------------------------------------------ CRNN tail
def linspace_f32(n):
    """torch.linspace(-1, 1, n) as stn_sample_kernel evaluates it: step = fl(2 / (n - 1)), then ONE fused multiply-add
    from the nearer end (-1 + i * step for i < n / 2, 1 - (n - 1 - i) * step otherwise)."""
    step = np.float64(np.float32(2.0) / np.float32(n - 1))
    i = np.arange(n, dtype=np.float64)
    return np.where(i < n // 2, (-1.0 + i * step), (1.0 - (n - 1 - i) * step)).astype(np.float32)


def stn_coords_f32(theta, hh, ww):
    """Sample coordinates of stn_sample_kernel in float32, operation for operation (separately rounded products and
    sums, then 0.5 * (v + 1) * W).  theta (B,6) float32 -> x, y of shape (B, hh*ww), pixel order (row, col)."""
    th = np.asarray(theta, np.float32)
    gx, gy = linspace_f32(ww), linspace_f32(hh)
    gyy, gxx = np.meshgrid(gy, gx, indexing="ij")
    gxx, gyy = gxx.reshape(-1)[None], gyy.reshape(-1)[None]
    t = [th[:, i:i + 1] for i in range(6)]
    xs = (t[0] * gxx + t[1] * gyy) + t[2]                    # float32 numpy: every op rounded on its own
    ys = (t[3] * gxx + t[4] * gyy) + t[5]
    x = (np.float32(0.5) * (xs + np.float32(1.0))) * np.float32(ww)
    y = (np.float32(0.5) * (ys + np.float32(1.0))) * np.float32(hh)
    return x.astype(np.float32), y.astype(np.float32)


def stn_sample_ref(feat, theta):
    """stn_sample_kernel: coordinates in float32 as the kernel forms them, floor / clamp, the reference's clipped-corner
    weights (oracle.crnn.stn_sample) and the blend in fp64.  feat (B,Hh,Ww,C) fp16 values -> (value, weight magnitude
    sum |w_i * v_i|, which bounds the fp32 blend's error at 4 * 2^-24 times it)."""
    feat = np.asarray(feat, np.float64)
    b, hh, ww, c = feat.shape
    x, y = stn_coords_f32(theta, hh, ww)
    x0 = np.floor(np.clip(x, -1e6, 1e6)).astype(np.int64)
    y0 = np.floor(np.clip(y, -1e6, 1e6)).astype(np.int64)
    x1, y1 = np.clip(x0 + 1, 0, ww - 1), np.clip(y0 + 1, 0, hh - 1)
    x0, y0 = np.clip(x0, 0, ww - 1), np.clip(y0, 0, hh - 1)
    xf, yf = x.astype(np.float32), y.astype(np.float32)
    f32 = np.float32
    wa = (x1.astype(f32) - xf) * (y1.astype(f32) - yf)          # float32, as the kernel's __fmul_rn of two differences
    wb = (x1.astype(f32) - xf) * (yf - y0.astype(f32))
    wc = (xf - x0.astype(f32)) * (y1.astype(f32) - yf)
    wd = (xf - x0.astype(f32)) * (yf - y0.astype(f32))
    flat = feat.reshape(b, hh * ww, c)
    g = lambda yy, xx: np.take_along_axis(flat, (yy * ww + xx)[..., None], 1)   # noqa: E731
    terms = [wa[..., None].astype(np.float64) * g(y0, x0), wb[..., None].astype(np.float64) * g(y1, x0),
             wc[..., None].astype(np.float64) * g(y0, x1), wd[..., None].astype(np.float64) * g(y1, x1)]
    val = sum(terms).reshape(b, hh, ww, c)
    mag = sum(np.abs(t) for t in terms).reshape(b, hh, ww, c)
    return val, mag


def ulp16(a):
    """Spacing of fp16 numbers at |a| (2^-24 below the normal range)."""
    a = np.abs(np.asarray(a, np.float64))
    e = np.floor(np.log2(np.maximum(a, 2.0 ** -14)))
    return 2.0 ** (e - 10)


def lstm_emulated(xw, u, go_backwards=False, round_u=True, round_h=True):
    """keras LSTM (gates i, f, c, o; sigmoid / tanh) in fp64 with lstm_kernel's documented choices: U rounded to fp16,
    h rounded to fp16 between steps (and on output), go_backwards outputs kept in processing order.
    xw (B,T,512) = x @ W + b (the kernel reads it from the fp32 GEMM); u (128,512).  Returns (B,T,128)."""
    xw = torch.as_tensor(np.asarray(xw), dtype=torch.float64)
    u = torch.as_tensor(np.asarray(u), dtype=torch.float64)
    if round_u:
        u = f16(u)
    if go_backwards:
        xw = torch.flip(xw, [1])
    b, t, _ = xw.shape
    units = u.shape[0]
    h = torch.zeros(b, units, dtype=torch.float64)
    c = torch.zeros(b, units, dtype=torch.float64)
    outs = []
    for s in range(t):
        z = xw[:, s] + h @ u
        zi, zf, zc, zo = torch.split(z, units, dim=1)
        c = torch.sigmoid(zf) * c + torch.sigmoid(zi) * torch.tanh(zc)
        h = torch.sigmoid(zo) * torch.tanh(c)
        if round_h:
            h = f16(h)
        outs.append(h)
    return torch.stack(outs, 1).numpy()


def dense_ref(x, wgt, bias, relu=False, x_err=None, out_f32=False):
    """Dense layer x (rows, K) @ wgt (K, N) + bias as the conv engine runs it (1x1 over rows, fp16 weights)."""
    x = np.asarray(x, np.float64)
    rows, kk = x.shape
    w = np.asarray(wgt, np.float32).T.reshape(-1, 1, 1, kk)            # (cout, 1, 1, cin)
    n = w.shape[0]
    return [a.reshape(rows, n) for a in conv_ref(x.reshape(1, 1, rows, kk), w, 1, 1, np.ones(n), np.asarray(bias, np.float32),
                                                   relu, out_f32=out_f32,
                                                   x_err=None if x_err is None else np.asarray(x_err).reshape(1, 1, rows, kk))]


# ------------------------------------------------------------------------------------------------ CRAFT forward, stage by stage
CRAFT_MEAN = np.array([0.485, 0.456, 0.406]) * 255          # compute_input (detection.py:34-42)
CRAFT_STD = np.array([0.229, 0.224, 0.225]) * 255


def compute_input_f32(img):
    """compute_input with numpy semantics: a float32 array, in-place ops against float64 constants."""
    x = np.float32(img)
    x -= CRAFT_MEAN
    x /= CRAFT_STD
    return x


def craft_affine(w, name, bn):
    """(s1, t1, aff_err) of a CRAFT layer folded in fp64 from the raw .pth-named weights (BN eps 1e-5 before the ReLU),
    with bounds on the device's fp32 folding sc = g / sqrtf(var + 1e-5f), t1 = (b - mu) * sc + beta."""
    b = np.asarray(w[name + ".bias"], np.float64)
    if bn is None:
        z = np.zeros_like(b)
        return np.ones_like(b), b, (z, z, z, z)
    g, be = np.asarray(w[bn + ".weight"], np.float64), np.asarray(w[bn + ".bias"], np.float64)
    mu, var = np.asarray(w[bn + ".running_mean"], np.float64), np.asarray(w[bn + ".running_var"], np.float64)
    s = g / np.sqrt(var + 1e-5)
    t = (b - mu) * s + be
    s_err = 5 * U32 * np.abs(s)
    t_err = np.abs(b - mu) * s_err + 3 * U32 * np.abs((b - mu) * s) + 2 * U32 * np.abs(t)
    z = np.zeros_like(b)
    return s, t, (s_err, t_err, z, z)


def crnn_affine(w, name, bn):
    """(s1, t1, s2, t2, aff_err) of a CRNN conv: bias + ReLU, then Keras BN (eps 1e-3) folded in fp64 from the raw
    weights, with bounds on the device's fp32 folding sc = gamma / sqrtf(var + 1e-3f), t2 = beta - mu * sc."""
    b = np.asarray(w[name + ".bias"], np.float64)
    z = np.zeros_like(b)
    if bn is None:
        return np.ones_like(b), b, None, None, (z, z, z, z)
    g, be = np.asarray(w[bn + ".gamma"], np.float64), np.asarray(w[bn + ".beta"], np.float64)
    mu, var = np.asarray(w[bn + ".moving_mean"], np.float64), np.asarray(w[bn + ".moving_variance"], np.float64)
    s = g / np.sqrt(var + 1e-3)
    t = be - mu * s
    s_err = 5 * U32 * np.abs(s)
    return np.ones_like(b), b, s, t, (z, z, s_err, np.abs(mu) * s_err + 2 * U32 * (np.abs(mu * s) + np.abs(t)))


def maxpool3s1_exact(a):
    """3x3 / stride 1 'same' max pool (padding never wins) of an (n,h,w,c) array; NaN propagates."""
    return _nhwc(F.max_pool2d(_nchw(a), 3, 1, 1))


def upsample_coords_f32(n_out, n_in):
    """Source index pairs and float32 weights of upsample_kernel / upsample2x_kernel along one axis, as the kernel forms
    them: scale = fl(n_in / n_out), f = max(fma(o + 0.5f, scale, -0.5f), 0) (nvcc contracts the product and the
    subtraction into one FFMA; the fp64 product of two floats is exact, so one rounding of the fp64 result is that
    FFMA), i0 = trunc(f), i1 = min(i0 + 1, n_in - 1), l = f - i0, h = 1 - l (float32).  Returns (i0, i1, l, h)."""
    f32 = np.float32
    scale = f32(f32(n_in) / f32(n_out))
    o = np.arange(n_out).astype(f32) + f32(0.5)
    f = np.maximum((o.astype(np.float64) * np.float64(scale) - 0.5).astype(f32), f32(0))
    i0 = f.astype(np.int64)
    i1 = np.minimum(i0 + 1, n_in - 1)
    lam = (f - i0.astype(f32)).astype(f32)
    return i0, i1, lam, (f32(1) - lam).astype(f32)


def upsample_ref(x, rows_in, ih, rows_out, oh, ow):
    """UpsampleLike as the kernels compute it: float32 coordinates and weights (``upsample_coords_f32``), the blend
    hy * (hx * a + lx * b) + ly * (hx * c + lx * d) in fp64.  x (n, R, iw, c) holds source rows ``rows_in`` (real row
    index, -1 for a gap) of an ih-row map; returns the rows ``rows_out`` of the oh x ow result as (value, bound), NaN
    where a source row is not in x.  The bound is 4 * 2^-24 * sum|w * v| for the fp32 blend (contracted into FMAs or
    not) plus half an fp16 ulp for the output rounding."""
    x = np.asarray(x, np.float64)
    iw = x.shape[2]
    y0, y1, ly, hy = (v[rows_out] for v in upsample_coords_f32(oh, ih))
    x0, x1, lx, hx = upsample_coords_f32(ow, iw)
    pos = np.full(ih, -1)
    ok = np.asarray(rows_in) >= 0
    pos[np.asarray(rows_in)[ok]] = np.nonzero(ok)[0]
    p0, p1 = pos[y0], pos[y1]
    miss = (p0 < 0) | (p1 < 0)
    r0, r1 = x[:, np.maximum(p0, 0)], x[:, np.maximum(p1, 0)]
    ly, hy = ly.astype(np.float64)[None, :, None, None], hy.astype(np.float64)[None, :, None, None]
    lx, hx = lx.astype(np.float64)[None, None, :, None], hx.astype(np.float64)[None, None, :, None]
    val = hy * (hx * r0[:, :, x0] + lx * r0[:, :, x1]) + ly * (hx * r1[:, :, x0] + lx * r1[:, :, x1])
    mag = hy * (hx * np.abs(r0[:, :, x0]) + lx * np.abs(r0[:, :, x1])) + ly * (hx * np.abs(r1[:, :, x0]) + lx * np.abs(r1[:, :, x1]))
    e32 = 4 * U32 * mag
    bound = e32 + 0.5 * ulp16(np.abs(val) + e32)
    val[:, miss] = np.nan
    return val, bound


# The CRAFT workspace's buffers (kCraftBufs in keras-ocr_b200/csrc/api.cu, with the lifetimes plan_craft derives from
# kCraftSteps): name -> (level = resolution divisor, channels, first step, last step)
CRAFT_BUFS = {
    "x16": (1, 16, 0, 1), "a": (1, 64, 1, 2), "b": (1, 64, 2, 2), "p1": (2, 64, 2, 3), "c": (2, 128, 3, 4),
    "cat4": (2, 192, 4, 25), "p2": (4, 128, 4, 5), "d": (4, 256, 5, 6), "cat3": (4, 384, 6, 22), "e": (4, 256, 7, 7),
    "p3": (8, 256, 7, 8), "f": (8, 512, 8, 9), "cat2": (8, 768, 9, 19), "g": (8, 512, 10, 10), "p4": (16, 512, 10, 11),
    "hh": (16, 512, 11, 12), "cat1": (16, 1536, 12, 16), "mp": (16, 512, 13, 14), "s5a": (16, 1024, 14, 15),
    "u1a": (16, 512, 16, 17), "u1b": (16, 256, 17, 18), "u2a": (8, 256, 19, 20), "u2b": (8, 128, 20, 21),
    "u3a": (4, 128, 22, 23), "u3b": (4, 64, 23, 24), "u4a": (2, 64, 25, 26), "u4b": (2, 32, 26, 27), "h1": (2, 32, 27, 28),
    "h2": (2, 32, 28, 29), "h3": (2, 16, 29, 30), "z2": (16, 256, 18, 19), "z3": (8, 128, 21, 22), "z4": (4, 64, 24, 25),
}


def craft_dims(h, w):
    """Rows and columns of every level (floor-halved), keyed by the level's divisor."""
    dims, hh, ww = {}, h, w
    for lv in (1, 2, 4, 8, 16):
        dims[lv] = (hh, ww)
        hh, ww = hh // 2, ww // 2
    return dims


def _s(buf, c0=None, c1=None):
    return (buf, 0 if c0 is None else c0, CRAFT_BUFS[buf][1] if c1 is None else c1)


# The forward's steps (b2o_craft_forward_until numbering): kind, layer, input slice, output slice, pooled output; the
# decoder levels name the low-resolution half z of a commuted upconvN.conv.0, its skip slice and (upconv) the decoder
# tensor y whose upsampling the level takes.
# A "pool" step writes its full-resolution output only where the engine does not fuse the pool (``full`` False).
CRAFT_STEPS = [
    dict(step=0, kind="normalize", out=_s("x16")),
    dict(step=1, kind="stem", layer="basenet.slice1.0", src=_s("x16"), out=_s("a")),
    dict(step=2, kind="conv", layer="basenet.slice1.3", src=_s("a"), out=_s("b"), pool=_s("p1"), full=False),
    dict(step=3, kind="conv", layer="basenet.slice1.7", src=_s("p1"), out=_s("c")),
    dict(step=4, kind="conv", layer="basenet.slice1.10", src=_s("c"), out=_s("cat4", 64, 192), pool=_s("p2"), full=True),
    dict(step=5, kind="conv", layer="basenet.slice2.14", src=_s("p2"), out=_s("d")),
    dict(step=6, kind="conv", layer="basenet.slice2.17", src=_s("d"), out=_s("cat3", 128, 384)),
    dict(step=7, kind="conv", layer="basenet.slice3.20", src=_s("cat3", 128, 384), out=_s("e"), pool=_s("p3"), full=False),
    dict(step=8, kind="conv", layer="basenet.slice3.24", src=_s("p3"), out=_s("f")),
    dict(step=9, kind="conv", layer="basenet.slice3.27", src=_s("f"), out=_s("cat2", 256, 768)),
    dict(step=10, kind="conv", layer="basenet.slice4.30", src=_s("cat2", 256, 768), out=_s("g"), pool=_s("p4"), full=False),
    dict(step=11, kind="conv", layer="basenet.slice4.34", src=_s("p4"), out=_s("hh")),
    dict(step=12, kind="conv", layer="basenet.slice4.37", src=_s("hh"), out=_s("cat1", 1024, 1536)),
    dict(step=13, kind="maxpool3", src=_s("cat1", 1024, 1536), out=_s("mp")),
    dict(step=14, kind="conv", layer="basenet.slice5.1", src=_s("mp"), out=_s("s5a")),
    dict(step=15, kind="conv", layer="basenet.slice5.2", src=_s("s5a"), out=_s("cat1", 0, 1024)),
    dict(step=16, kind="conv", layer="upconv1.conv.0", src=_s("cat1"), out=_s("u1a")),
    dict(step=17, kind="conv", layer="upconv1.conv.3", src=_s("u1a"), out=_s("u1b")),
    dict(step=18, kind="up", layer="upconv2.conv.0", src=_s("u1b"), out=_s("cat2", 0, 256), z=_s("z2"), skip=_s("cat2", 256, 768)),
    dict(step=19, kind="upconv", layer="upconv2.conv.0", src=_s("cat2"), y=_s("u1b"), out=_s("u2a"), z=_s("z2"), skip=_s("cat2", 256, 768)),
    dict(step=20, kind="conv", layer="upconv2.conv.3", src=_s("u2a"), out=_s("u2b")),
    dict(step=21, kind="up", layer="upconv3.conv.0", src=_s("u2b"), out=_s("cat3", 0, 128), z=_s("z3"), skip=_s("cat3", 128, 384)),
    dict(step=22, kind="upconv", layer="upconv3.conv.0", src=_s("cat3"), y=_s("u2b"), out=_s("u3a"), z=_s("z3"), skip=_s("cat3", 128, 384)),
    dict(step=23, kind="conv", layer="upconv3.conv.3", src=_s("u3a"), out=_s("u3b")),
    dict(step=24, kind="up", layer="upconv4.conv.0", src=_s("u3b"), out=_s("cat4", 0, 64), z=_s("z4"), skip=_s("cat4", 64, 192)),
    dict(step=25, kind="upconv", layer="upconv4.conv.0", src=_s("cat4"), y=_s("u3b"), out=_s("u4a"), z=_s("z4"), skip=_s("cat4", 64, 192)),
    dict(step=26, kind="conv", layer="upconv4.conv.3", src=_s("u4a"), out=_s("u4b")),
    dict(step=27, kind="conv", layer="conv_cls.0", src=_s("u4b"), out=_s("h1")),
    dict(step=28, kind="conv", layer="conv_cls.2", src=_s("h1"), out=_s("h2")),
    dict(step=29, kind="conv", layer="conv_cls.4", src=_s("h2"), out=_s("h3")),
    dict(step=30, kind="tail", src=_s("h3")),
]
CRAFT_LAYERS = {name: (cin, cout, k, dil, bn, relu) for name, cin, cout, k, dil, bn, relu in CRAFT_CONVS}


def craft_layer_ref(w, layer, x, round_w=True, x_err=None, cols=None, up=None, stem16=False):
    """One CRAFT conv layer from the raw weights: conv_ref with the BN folded here in fp64 (``craft_affine``).
    cols = (c0, c1): only those input columns of the weight (the halves of a commuted upconvN.conv.0; the decoder half
    has no bias, BN or ReLU).  stem16: slice1.0 over the 16-channel input whose padding channels are weighted 0."""
    cin, cout, k, dil, bn, relu = CRAFT_LAYERS[layer]
    wt = np.transpose(np.asarray(w[layer + ".weight"], np.float32), (0, 2, 3, 1))       # OIHW -> (cout, k, k, cin)
    s1, t1, aff = craft_affine(w, layer, bn)
    if cols is not None:
        wt = wt[..., cols[0]:cols[1]]
        if cols[0] == 0:
            z = np.zeros(cout)
            s1, t1, relu, aff = np.ones(cout), z, 0, None
    if stem16:
        wt = np.concatenate([wt, np.zeros(wt.shape[:3] + (13,), np.float32)], -1)
    return conv_ref(x, wt, k, dil, s1, t1, relu, up=up, x_err=x_err, aff_err=aff, round_w=round_w)


def craft_tail_ref(w, x, x_err=None, round_w=True):
    """conv_cls.6 + conv_cls.8 (``tail_ref``) from the raw weights."""
    w6 = np.asarray(w["conv_cls.6.weight"], np.float64)[:, :, 0, 0].T
    w8 = np.asarray(w["conv_cls.8.weight"], np.float64)[:, :, 0, 0].T
    return tail_ref(x, w6, w["conv_cls.6.bias"], w8, w["conv_cls.8.bias"], x_err=x_err, round_w=round_w)


def craft_chain(w, img):
    """The whole forward by chaining CRAFT_STEPS in fp64 (no fp16 rounding anywhere, unrounded weights): the graph the
    stage checks restate, to be compared with oracle.craft.craft_forward.  img (n,h,w,3) uint8 -> scores (n,h/2,w/2,2)."""
    n, h, wd, _ = img.shape
    dims = craft_dims(h, wd)
    bufs = {name: np.zeros((n,) + dims[lv] + (c,)) for name, (lv, c, _f, _l) in CRAFT_BUFS.items()}
    get = lambda s: bufs[s[0]][..., s[1]:s[2]]                              # noqa: E731
    x64 = (np.asarray(img, np.float64) - CRAFT_MEAN) / CRAFT_STD
    scores = None
    for st in CRAFT_STEPS:
        kind = st["kind"]
        if kind == "normalize":
            bufs["x16"][..., :3] = x64
            continue
        if kind == "tail":
            scores = craft_tail_ref(w, get(st["src"]), round_w=False)[0]
            continue
        src = get(st["src"])
        if kind == "maxpool3":
            val = maxpool3s1_exact(src)
        elif kind == "up":
            lv = CRAFT_BUFS[st["out"][0]][0]
            oh, ow = dims[lv]
            val = upsample_ref(src, np.arange(src.shape[1]), src.shape[1], np.arange(oh), oh, ow)[0]
        else:
            val = craft_layer_ref(w, "basenet.slice1.0" if kind == "stem" else st["layer"], src, round_w=False,
                                  stem16=kind == "stem")[0]
        o = st["out"]
        bufs[o[0]][..., o[1]:o[2]] = val
        if st.get("pool"):
            p = st["pool"]
            bufs[p[0]][..., p[1]:p[2]] = pool_ref(val, val)[0]
    return scores


# ------------------------------------------------------------------------------------------------ CRNN conv backbone
# (layer, input tap, output tap, pooled tap): conv_1 .. conv_7 of b2o_crnn_forward; "in" is the crnn_in tensor
CRNN_STEPS = [("conv_1", "in", "x1", None), ("conv_2", "x1", "x2", None), ("conv_3", "x2", "x3", "p3"),
              ("conv_4", "p3", "x4", None), ("conv_5", "x4", "x5", "p5"), ("conv_6", "p5", "x6", None),
              ("conv_7", "x6", "features", None)]


def crnn_layer_ref(w, layer, x, round_w=None):
    """One CRNN conv (bias + ReLU, then the folded Keras BN where the layer has one) from the raw HWIO weights.
    conv_1 runs on the CUDA cores with fp32 weights and the bias as the accumulator's first term (round_w defaults to
    False for it, and its bound takes GAMMA(K) * |bias| for that)."""
    bn = {n: b for n, _ci, _co, _k, b in CRNN_CONVS}[layer]
    wt = np.transpose(np.asarray(w[layer + ".kernel"], np.float32), (3, 0, 1, 2))         # HWIO -> (cout, k, k, cin)
    s1, t1, s2, t2, aff = crnn_affine(w, layer, bn)
    if layer == "conv_1":
        aff = (aff[0], gamma(wt[0].size) * np.abs(t1), aff[2], aff[3])
    if round_w is None:
        round_w = layer != "conv_1"
    return conv_ref(x, wt, 3, 1, s1, t1, 1, s2, t2, aff_err=aff, round_w=round_w)
