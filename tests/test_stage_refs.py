"""CPU: the stage references of tests/stage_refs.py against the oracle and against themselves (no GPU needed)."""
import numpy as np
import torch
import torch.nn.functional as F

from tests import stage_refs as R


def test_lstm_emulation_without_rounding_is_the_oracle_lstm():
    from oracle import crnn
    rng = np.random.default_rng(0)
    w = {"l.kernel": rng.standard_normal((128, 512)).astype(np.float32) * 0.09,
         "l.recurrent_kernel": rng.standard_normal((128, 512)).astype(np.float32) * 0.09,
         "l.bias": rng.standard_normal(512).astype(np.float32) * 0.05}
    x = rng.standard_normal((3, 50, 128)).astype(np.float32)
    wt = {k: torch.from_numpy(v) for k, v in w.items()}
    for back in (False, True):
        want = crnn.lstm(wt, torch.from_numpy(x), "l", go_backwards=back).numpy()
        xw = x.astype(np.float64) @ w["l.kernel"] + w["l.bias"]
        got = R.lstm_emulated(xw, w["l.recurrent_kernel"], go_backwards=back, round_u=False, round_h=False)
        assert np.abs(got - want).max() <= 2e-6
        rounded = R.lstm_emulated(xw, w["l.recurrent_kernel"], go_backwards=back)
        assert np.array_equal(rounded, R.f16(rounded))                   # h really is fp16 between steps
        assert 1e-5 < np.abs(rounded - want).max() < 2e-2


def test_stn_sample_restatement_is_the_oracle_sampler():
    from oracle import crnn
    rng = np.random.default_rng(1)
    feat = rng.standard_normal((8, 50, 7, 16)).astype(np.float16).astype(np.float32)
    thetas = [[1, 0, 0, 0, 1, 0], [1.1, 0.05, 0.45, -0.03, 1.05, 0.3], [0.9, 0.02, -0.6, 0.04, 1.1, -0.5],
              [0, 0, -1 / 7, 0, 0, -0.2], [-1, 0, 0, 0, -1, 0]]
    thetas += list(np.array([1, 0, 0, 0, 1, 0]) + rng.standard_normal((3, 6)) * 0.2)
    theta = np.asarray(thetas, np.float32)
    want = crnn.stn_sample(torch.from_numpy(feat), torch.from_numpy(theta)).numpy()
    got, mag = R.stn_sample_ref(feat, theta)
    assert np.abs(got - want).max() <= 1e-5 * np.abs(feat).max()
    assert (mag >= np.abs(got) - 1e-12).all()
    x, y = R.stn_coords_f32(theta, 50, 7)
    assert x[0, 0] == 0.0 and x[0, 6] == 7.0 and y[0, 0] == 0.0 and y[0, -1] == 50.0   # identity: first / last column, row
    for n in (7, 50):
        assert np.abs(R.linspace_f32(n) - torch.linspace(-1, 1, n).numpy()).max() <= 2.0 ** -23
        lo = R.linspace_f32(n)[: n // 2]
        assert np.array_equal(lo, -R.linspace_f32(n)[::-1][: n // 2])                    # symmetric ends


def test_upsample_add_reference_is_upsample_then_concat_conv():
    """The commuted form the kernel computes (1x1 conv of the skip + upsampled low-resolution conv of the decoder
    tensor) equals the reference's UpsampleLike + Concatenate + 1x1 conv (oracle/craft.py::_upsample_like)."""
    from oracle import craft
    rng = np.random.default_rng(2)
    n, h, w, cy, cs, co = 2, 8, 10, 24, 16, 32
    y = rng.standard_normal((n, h // 2, w // 2, cy))
    skip = rng.standard_normal((n, h, w, cs)).astype(np.float16).astype(np.float64)
    wt = R.f16(rng.standard_normal((co, cy + cs)) * 0.2)
    s1, t1 = rng.uniform(0.5, 1.5, co), rng.standard_normal(co) * 0.1
    yt = torch.from_numpy(y).permute(0, 3, 1, 2)
    cat = torch.cat([craft._upsample_like(yt, torch.zeros(n, 1, h, w)), torch.from_numpy(skip).permute(0, 3, 1, 2)], 1)
    want = F.relu(F.conv2d(cat, torch.from_numpy(wt)[:, :, None, None]) * torch.from_numpy(s1)[None, :, None, None]
                  + torch.from_numpy(t1)[None, :, None, None]).permute(0, 2, 3, 1).numpy()
    low = y @ wt[:, :cy].T                                           # the decoder half at low resolution
    got, bound = R.conv_ref(skip, wt[:, cy:].reshape(co, 1, 1, cs), 1, 1, s1, t1, 1, up=low, out_f32=True)
    assert np.abs(got - want).max() <= 1e-12
    assert (bound > 0).all()


def _fp32_layer(x, wgt, k, dil, s1, t1, relu, s2=None, t2=None, up=None):
    """The same layer evaluated in fp32 (im2col + one fp32 GEMM, fmaf-like epilogue, fp16 output)."""
    xt = torch.from_numpy(np.asarray(x, np.float32)).permute(0, 3, 1, 2)
    n, _, h, w = xt.shape
    wt = torch.from_numpy(wgt).half().float().permute(0, 3, 1, 2)
    cols = F.unfold(xt, k, dilation=dil, padding=dil * (k // 2))          # (n, cin*k*k, h*w)
    acc = (wt.reshape(wt.shape[0], -1) @ cols).reshape(n, -1, h, w)
    if up is not None:
        acc = acc + R.upsample_like(torch.from_numpy(np.asarray(up, np.float32)).permute(0, 3, 1, 2), h, w)
    col = lambda v: torch.from_numpy(np.asarray(v, np.float32))[None, :, None, None]   # noqa: E731
    y = acc * col(s1) + col(t1)
    if relu:
        y = y.clamp_min(0)
    if s2 is not None:
        y = y * col(s2) + col(t2)
    return y.half().double().permute(0, 2, 3, 1).numpy()


def test_bound_holds_for_the_reference_evaluated_in_fp32():
    rng = np.random.default_rng(3)
    for n, h, w, cin, cout, k, dil, aff, upc in [(2, 9, 11, 64, 32, 3, 1, True, False), (1, 7, 6, 512, 16, 3, 2, False, False),
                                                 (1, 1, 40, 3584, 16, 1, 1, False, False), (2, 6, 8, 64, 32, 1, 1, False, True)]:
        x = rng.standard_normal((n, h, w, cin)).astype(np.float16)
        wgt = (rng.standard_normal((cout, k, k, cin)) * np.sqrt(2.0 / (cin * k * k))).astype(np.float32)
        s1, t1 = rng.uniform(-1.5, 1.5, cout).astype(np.float32), (rng.standard_normal(cout) * 0.2).astype(np.float32)
        s2 = rng.uniform(0.5, 1.5, cout).astype(np.float32) if aff else None
        t2 = (rng.standard_normal(cout) * 0.2).astype(np.float32) if aff else None
        up = rng.standard_normal((n, h // 2, w // 2, cout)).astype(np.float16) if upc else None
        val, bound = R.conv_ref(x, wgt, k, dil, s1, t1, 1, s2, t2, up=up)
        got = _fp32_layer(x, wgt, k, dil, s1, t1, 1, s2, t2, up=up)
        assert (np.abs(got - val) <= bound).all()
        if h >= 2:
            pv, pb = R.pool_ref(val, bound)
            assert (np.abs(R.maxpool2_exact(got) - pv) <= pb).all()
            assert np.array_equal(R.maxpool2_exact(got), _nchw_pool(got))
    # the tail: fp32 evaluation of the fp16 map against the fp64 tail of the unrounded map
    x = rng.standard_normal((2, 5, 7, 16))
    ex = R.U16 * np.abs(x) + R.SUB16
    w6, b6 = rng.standard_normal((16, 16)) * 0.35, rng.standard_normal(16) * 0.1
    w8, b8 = rng.standard_normal((16, 2)) * 0.3, np.array([0.5, -0.5])
    val, bound = R.tail_ref(x, w6, b6, w8, b8, x_err=ex)
    x32 = torch.from_numpy(R.f16(x)).float()
    a = torch.relu(x32 @ torch.from_numpy(R.f16(w6)).float() + torch.from_numpy(b6).float())
    o = (a @ torch.from_numpy(R.f16(w8)).float() + torch.from_numpy(b8).float()).double().numpy()
    assert (np.abs(o - val) <= bound).all()


def _nchw_pool(a):
    return F.max_pool2d(torch.from_numpy(a).permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1).numpy()


def test_ulp16():
    assert R.ulp16(1.0) == 2.0 ** -10 and R.ulp16(0.75) == 2.0 ** -11 and R.ulp16(0.0) == 2.0 ** -24
    assert R.ulp16(65504.0) == 32.0
