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


# ------------------------------------------------------------------------------------------------ CRAFT / CRNN stage tables
def test_craft_stage_chain_is_the_oracle_forward():
    """Chaining CRAFT_STEPS in fp64 (the graph tests/test_gpu_craft_stages.py checks stage by stage, BN folded from the
    raw weights) reproduces oracle.craft.craft_forward, at a size where every decoder level takes the general
    upsampling (33 x 47) and at a multiple of 32."""
    from keras_ocr_b200 import weights as W
    from oracle import craft
    w = W.synthetic_craft_weights(3)
    rng = np.random.default_rng(4)
    for n, h, wd in [(2, 33, 47), (1, 32, 64)]:
        img = rng.integers(0, 256, (n, h, wd, 3), dtype=np.uint8)
        got = R.craft_chain(w, img)
        x = torch.from_numpy(R.compute_input_f32(img)).permute(0, 3, 1, 2)
        want = craft.craft_forward(w, x).numpy()
        assert got.shape == want.shape == (n, h // 2, wd // 2, 2)
        assert np.abs(got - want).max() <= 1e-4 * np.abs(want).max(), np.abs(got - want).max()


def test_crnn_backbone_chain_is_the_oracle_features():
    from keras_ocr_b200 import weights as W
    from oracle import crnn
    rng = np.random.default_rng(5)
    for color in (False, True):
        w = W.synthetic_crnn_weights(seed=2, color=color)
        crops = rng.integers(0, 256, (2, 31, 200) + ((3,) if color else ()), dtype=np.uint8)
        c = crops.astype(np.float64)[..., None] if not color else crops.astype(np.float64)
        x = np.flip(np.transpose(c, (0, 2, 1, 3)), 2) / 255.0                     # crnn_in: (b, 200, 31, ch)
        taps = {"in": x}
        for layer, src, dst, pool in R.CRNN_STEPS:
            taps[dst] = R.crnn_layer_ref(w, layer, taps[src], round_w=False)[0]
            if pool:
                taps[pool] = R.pool_ref(taps[dst], taps[dst])[0]
        want = crnn.crnn_features(w, crops.astype(np.float32) / 255.0).permute(0, 2, 3, 1).numpy()
        assert np.abs(taps["features"] - want).max() <= 1e-4 * np.abs(want).max()


# decoder size pairs (n_out <- n_in) of the CRAFT sizes tests/test_gpu_craft_stages.py runs that are not exactly 2x, i.e.
# the ones upsample_kernel (not upsample2x_kernel) computes, plus exact 2x pairs
UPSAMPLE_PAIRS = [(25, 12), (23, 11), (11, 5), (5, 2), (9, 4), (18, 9), (16, 8), (36, 18), (1024, 512), (2, 1), (3, 1)]


def _torch_weights(n_out, n_in):
    """torch's float32 bilinear weights along one axis, read off F.interpolate of one-hot rows: [source, output]."""
    eye = torch.eye(n_in, dtype=torch.float32).reshape(n_in, 1, n_in, 1)
    return F.interpolate(eye, size=(n_out, 1), mode="bilinear", align_corners=False)[:, 0, :, 0].numpy()


def test_upsample_coordinates_are_torch_float_coordinates():
    for n_out, n_in in UPSAMPLE_PAIRS:
        i0, i1, lam, hi = R.upsample_coords_f32(n_out, n_in)
        mine = np.zeros((n_in, n_out), np.float32)
        o = np.arange(n_out)
        np.add.at(mine, (i0, o), hi)
        np.add.at(mine, (i1, o), lam)
        assert np.array_equal(mine, _torch_weights(n_out, n_in)), (n_out, n_in)
        assert (i0 <= i1).all() and (i1 < n_in).all() and ((lam >= 0) & (lam < 1)).all()


def test_upsample_reference_is_interpolate():
    """upsample_ref with float32 coordinates is F.interpolate (fp64 coordinates) up to the coordinates' float32
    rounding, and its bound covers the same blend done in float32 and rounded to fp16."""
    rng = np.random.default_rng(6)
    for n_out, n_in in [(25, 12), (11, 5), (16, 8)]:
        x = R.f16(rng.standard_normal((2, n_in, n_in + 3, 8)))
        val, bound = R.upsample_ref(x, np.arange(n_in), n_in, np.arange(n_out), n_out, 2 * n_in + 1)
        want = R._nhwc(R.upsample_like(R._nchw(x), n_out, 2 * n_in + 1))
        assert np.abs(val - want).max() <= 1e-5 * np.abs(x).max()
        y32 = torch.from_numpy(x).float().permute(0, 3, 1, 2)
        got = F.interpolate(y32, size=(n_out, 2 * n_in + 1), mode="bilinear", align_corners=False)
        got = R.f16(got.permute(0, 2, 3, 1).double()).numpy()
        assert (np.abs(got - val) <= bound).all()
        part = R.upsample_ref(x[:, :3], np.array([0, 1, 2]), n_in, np.arange(n_out), n_out, 2 * n_in + 1)[0]
        assert np.isnan(part[:, -1]).all() and np.array_equal(part[:, 0], val[:, 0])    # rows past the band: NaN
