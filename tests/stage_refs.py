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


def conv_ref(x, wgt, k, dil, s1, t1, relu, s2=None, t2=None, up=None, out_f32=False, x_err=None):
    """One convolution layer of the engine in fp64.  x (n,h,w,cin) and up (n,h/2,w/2,cout) hold fp16 values;
    wgt (cout,k,k,cin) is rounded to fp16 here (as build_layer does).  x_err: optional per-element bound on the input
    (propagated through |w|).  Returns NHWC float64 (value, bound)."""
    n, h, w, cin = x.shape
    xt = _nchw(x)
    wt = f16(torch.from_numpy(np.ascontiguousarray(wgt, np.float32)).permute(0, 3, 1, 2).double())
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
    if relu:
        y = y.clamp_min(0.0)
    if s2 is not None:
        e = e * _col(np.abs(s2)) + U32 * ((y * _col(s2)).abs() + _col(np.abs(t2)))
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


def tail_ref(x, w6, b6, w8, b8, x_err=None):
    """CRAFT head tail conv_cls.6 (1x1 16->16, ReLU) + conv_cls.8 (1x1 16->2) on a 16-channel map x (n,h,w,16).
    w6 (16 in, 16 out) and w8 (16 in, 2 out) are rounded to fp16 here; b6 / b8 stay fp32.  Both layers are serial
    fmaf chains of 16 terms in fp32; x_err (the bound on x) is propagated through |w6| and |w8|.  Returns (scores, bound)."""
    x = np.asarray(x, np.float64)
    w6, w8 = f16(w6), f16(w8)
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
