"""Each stage of the CRNN tail measured on its own: every stage is fed the device's OWN input, read from the tap of the
previous stage (``Recognizer.tap``), and compared with an fp64 reference of that stage alone, so an error of one
kernel is not hidden under the differences the earlier layers accumulate.

Bounds (tests/stage_refs.py for the conv arithmetic):

* features -> theta (stn.conv_a as a 1x1 GEMM + stn_col2im, stn.conv_b, stn.dense_a, stn_theta): two fp64 chains from
  the device's features -- one with the device's fp16 rounding points emulated (the per-tap GEMM columns, sa, sb, d1),
  one plain (``oracle.crnn.stn_theta`` on the fp16 weights the kernels hold).  Both are compared relative to the
  magnitude of the last layer, M = |d1| @ |W| + |b|: at most 2^-10 * M against the emulation (one fp16 ulp of d1 through
  stn.dense_b) and 2^-8 * M against the plain chain (the roundings of the GEMM columns, sa, sb and d1).
* features + device theta -> warped: the sample coordinates are restated in float32 operation for operation (the kernel's
  fused linspace, separate products and sums, floor, clamp) and the blend done in fp64; at most one fp16 ulp plus
  4 * 2^-24 * sum|w_i * v_i| for the fp32 blend.  Known thetas (identity, past the last row and column, exact integer
  coordinates, negative coordinates) drive the sampler to its edges through a zero ``stn.dense_b.kernel``.
* warped -> fc_9: the conv bound of tests/stage_refs.py (1x1 over B * 50 rows, K = 3584).
* fc_9 -> l1 and l1 -> l2: a Keras LSTM in fp64 with the kernel's documented choices (U rounded to fp16, h rounded to fp16
  between steps, go_backwards outputs in processing order, l1 = fp16(hf + hb)) from x @ W + b of the device's own input:
  at most 2^-9 absolute (two fp16 ulps of l1 in [1, 2)); against the unrounded ``oracle.crnn.lstm`` (fp32 weights, no
  fp16 h) at most 2^-7 absolute.
* l2 -> logits: fp32 on both sides, ``GAMMA(257) * (|l2| @ |w| + |b|)`` per element, K = 3, 37, 301 and 1024; the labels
  are exactly the greedy collapse of the device's own logits.
Measured on an H100 80GB HBM3 (700 W): theta 0.17 of the tight and 0.074 of the loose bound, warped 0.5 of its bound (the device rounds the fp64 blend to nearest), fc_9 0.83
(mostly the half-ulp output rounding), l1 / l2 within 9.8e-4 / 4.9e-4 of the emulation and 1.4e-3 of the oracle LSTM,
logits 0.009 of their bound.
Batches 1, 7, 8, 9 and 17 cover partial 8-crop LSTM CTAs; stages 3 to 5 also run on a recognizer without the spatial
transformer, where fc_9 reads the features directly.
"""
import numpy as np
import pytest
import torch

from keras_ocr_b200 import weights as W
from tests import stage_refs as R

pytestmark = pytest.mark.gpu

THETA_TIGHT = 2.0 ** -10          # x (|d1| @ |w| + |b|) of stn.dense_b: device vs the fp16-emulating chain
THETA_LOOSE = 2.0 ** -8           # the same against the plain fp64 chain
LSTM_TIGHT = 2.0 ** -9            # device LSTM vs the fp16-emulating fp64 LSTM (absolute, outputs in [-2, 2])
LSTM_LOOSE = 2.0 ** -7            # device LSTM vs the unrounded oracle.crnn.lstm (absolute)


def _recognizer(w, **kw):
    from keras_ocr_b200.recognition import Recognizer
    rec = Recognizer(weights=w, **kw)
    rec.keep_workspace = True
    return rec


def _run(rec, b, seed):
    rng = np.random.default_rng(seed)
    crops = rng.integers(0, 256, (b, 31, 200), dtype=np.uint8)
    crops[:, :, 120 + 7 * (seed % 5):] = 0                      # a zero tail, as a warpBox crop has
    t = torch.from_numpy(crops).to(rec.device)
    x = torch.empty((b, 200, 31), dtype=torch.float16, device=rec.device)
    rec.ctx.crops_to_input(t.data_ptr(), b, x.data_ptr(), torch.cuda.current_stream().cuda_stream)
    labels = rec.predict_device(x).cpu().numpy()
    taps = {"labels": labels}
    shapes = {"features": ((b, 50, 7, 512), torch.float16), "fc_9": ((b, 50, 128), torch.float16),
              "l1": ((b, 50, 128), torch.float16), "l2": ((b, 50, 256), torch.float16),
              "logits": ((b, 48, len(rec.alphabet) + 1), torch.float32)}
    if rec.stn:
        shapes.update(theta=((b, 6), torch.float32), warped=((b, 50, 7, 512), torch.float16))
    for name, (shape, dt) in shapes.items():
        taps[name] = rec.tap(name, shape, dt).double().cpu().numpy()
    return taps


def _ratio(tag, dev, val, bound):
    r = float((np.abs(dev - val) / bound).max())
    print(f"{tag}: worst error / bound = {r:.3g}")
    assert r <= 1.0, (tag, r)


# ------------------------------------------------------------------------------------------ 1. localisation net
def _loc_net(w, feat, emulate):
    """stn.conv_a (1x1 GEMM over 25 taps x 16 channels + stn_col2im), stn.conv_b, stn.dense_a, stn_theta in fp64 from
    the device's features, with (emulate) or without the device's fp16 rounding points; returns (theta, d1)."""
    rnd = R.f16 if emulate else (lambda v: v)
    b = feat.shape[0]
    wa = R.f16(w["stn.conv_a.kernel"])                                      # (5,5,512,16)
    wg = wa.transpose(2, 0, 1, 3).reshape(512, 400)                         # stn.conv_a_gemm: column tap * 16 + c
    cols = rnd((feat.reshape(-1, 512) @ wg).reshape(b, 50, 7, 5, 5, 16))
    pre = np.broadcast_to(np.asarray(w["stn.conv_a.bias"], np.float64), (b, 50, 7, 16)).copy()
    for ky in range(5):                                                     # out[h][w] += cols[h + ky - 2][w + kx - 2][ky][kx]
        for kx in range(5):
            hs, ws = slice(max(0, 2 - ky), min(50, 52 - ky)), slice(max(0, 2 - kx), min(7, 9 - kx))
            hi, wi = slice(hs.start + ky - 2, hs.stop + ky - 2), slice(ws.start + kx - 2, ws.stop + kx - 2)
            pre[:, hs, ws] += cols[:, hi, wi, ky, kx]
    sa = rnd(np.maximum(pre, 0.0))
    wb = np.transpose(w["stn.conv_b.kernel"], (3, 0, 1, 2))                 # HWIO -> (cout, k, k, cin)
    sb = rnd(R.conv_ref(sa, wb, 5, 1, np.ones(32), w["stn.conv_b.bias"], 1, out_f32=True)[0])
    d1 = rnd(R.dense_ref(sb.reshape(b, 11200), w["stn.dense_a.kernel"], w["stn.dense_a.bias"], relu=True, out_f32=True)[0])
    return d1 @ np.asarray(w["stn.dense_b.kernel"], np.float64) + np.asarray(w["stn.dense_b.bias"], np.float64), d1


def _check_theta(w, taps):
    from oracle import crnn
    feat = taps["features"]
    emul, d1 = _loc_net(w, feat, emulate=True)
    plain, _ = _loc_net(w, feat, emulate=False)
    w16 = {k: torch.from_numpy(np.asarray(v, np.float64)) for k, v in w.items() if k.startswith("stn.")}
    for k in ("stn.conv_a.kernel", "stn.conv_b.kernel", "stn.dense_a.kernel"):
        w16[k] = R.f16(w16[k])
    oracle = crnn.stn_theta(w16, torch.from_numpy(feat).permute(0, 3, 1, 2)).numpy()
    assert np.allclose(plain, oracle, rtol=1e-9, atol=1e-12)                 # the plain chain IS the oracle's net
    mag = np.abs(d1) @ np.abs(np.asarray(w["stn.dense_b.kernel"], np.float64)) + np.abs(w["stn.dense_b.bias"])
    _ratio("theta vs fp16-emulating chain", taps["theta"], emul, THETA_TIGHT * mag)
    _ratio("theta vs plain fp64", taps["theta"], plain, THETA_LOOSE * mag)


# ------------------------------------------------------------------------------------------ 2. sampler
def _check_warped(taps, feat_key="features"):
    val, mag = R.stn_sample_ref(taps[feat_key], taps["theta"].astype(np.float32))
    bound = R.ulp16(val) + 4 * R.U32 * mag
    _ratio("warped", taps["warped"], val, bound)


# ------------------------------------------------------------------------------------------ 3.-5. fc_9, BiLSTM, fc_12
def _check_tail(w, taps, stn=True):
    from oracle import crnn
    b = taps["fc_9"].shape[0]
    src = taps["warped"] if stn else taps["features"]
    val, bound = R.dense_ref(src.reshape(b * 50, 3584), w["fc_9.kernel"], w["fc_9.bias"], relu=True)
    _ratio("fc_9", taps["fc_9"].reshape(b * 50, 128), val, bound)

    def bilstm_in(x, layer):
        names = ("lstm_10", "lstm_10_back") if layer == 1 else ("lstm_11", "lstm_11_back")
        wk = R.f16(np.concatenate([w[n + ".kernel"] for n in names], 1))
        bias = np.concatenate([w[n + ".bias"] for n in names]).astype(np.float64)
        return x @ wk + bias, names

    xw, (nf, nb) = bilstm_in(taps["fc_9"], 1)
    hf = R.lstm_emulated(xw[..., :512], w[nf + ".recurrent_kernel"])
    hb = R.lstm_emulated(xw[..., 512:], w[nb + ".recurrent_kernel"], go_backwards=True)
    l1 = R.f16(hf + hb)
    err = float(np.abs(taps["l1"] - l1).max())
    print(f"l1 vs emulation: {err:.3g}")
    assert err <= LSTM_TIGHT, err
    wt = {k: torch.from_numpy(np.asarray(v)) for k, v in w.items()}
    x = torch.from_numpy(taps["fc_9"]).float()
    loose = (crnn.lstm(wt, x, nf) + crnn.lstm(wt, x, nb, go_backwards=True)).numpy()
    err = float(np.abs(taps["l1"] - loose).max())
    print(f"l1 vs oracle.crnn.lstm: {err:.3g}")
    assert err <= LSTM_LOOSE, err

    xw, (nf, nb) = bilstm_in(taps["l1"], 2)
    l2 = np.concatenate([R.lstm_emulated(xw[..., :512], w[nf + ".recurrent_kernel"]),
                         R.lstm_emulated(xw[..., 512:], w[nb + ".recurrent_kernel"], go_backwards=True)], -1)
    err = float(np.abs(taps["l2"] - l2).max())
    print(f"l2 vs emulation: {err:.3g}")
    assert err <= LSTM_TIGHT, err
    x = torch.from_numpy(taps["l1"]).float()
    loose = torch.cat([crnn.lstm(wt, x, nf), crnn.lstm(wt, x, nb, go_backwards=True)], -1).numpy()
    err = float(np.abs(taps["l2"] - loose).max())
    print(f"l2 vs oracle.crnn.lstm: {err:.3g}")
    assert err <= LSTM_LOOSE, err
    _check_logits(w, taps)


def _greedy(logits):
    """Greedy CTC on logits: first maximum, blank = K - 1, repeats merged, -1 padding."""
    b, t, k = logits.shape
    best = logits.argmax(-1)
    out = np.full((b, t), -1, np.int64)
    for i in range(b):
        n, prev = 0, -1
        for c in best[i]:
            if c != k - 1 and c != prev:
                out[i, n] = c
                n += 1
            prev = c
    return out


def _check_logits(w, taps):
    l2 = taps["l2"][:, 2:]
    wk, bk = np.asarray(w["fc_12.kernel"], np.float64), np.asarray(w["fc_12.bias"], np.float64)
    val = l2 @ wk + bk
    bound = R.gamma(257) * (np.abs(l2) @ np.abs(wk) + np.abs(bk))
    _ratio("logits", taps["logits"], val, bound)
    assert np.array_equal(taps["labels"], _greedy(taps["logits"]))


# ------------------------------------------------------------------------------------------ tests
@pytest.fixture(scope="module")
def weights():
    return W.synthetic_crnn_weights(seed=2)


@pytest.fixture(scope="module")
def rec(cuda_device, weights):
    return _recognizer(weights)


@pytest.mark.parametrize("b", [1, 7, 8, 9, 17])
def test_crnn_stages_one_at_a_time(rec, weights, b):
    taps = _run(rec, b, seed=100 + b)
    _check_theta(weights, taps)
    _check_warped(taps)
    _check_tail(weights, taps)


def test_crnn_stages_without_spatial_transformer(cuda_device):
    w = W.synthetic_crnn_weights(seed=5, stn=False)
    taps = _run(_recognizer(w, build_params={"stn": False}), 9, seed=7)
    _check_tail(w, taps, stn=False)


def _integer_theta(xt, yt):
    """theta = [0, 0, c, 0, 0, d] whose float32 coordinates are exactly (xt, yt) for every output pixel."""
    def find(target, axis):
        c0 = np.float32(2.0 * target / (7, 50)[axis] - 1.0)
        for step in range(-64, 65):
            c = np.float32(c0 + np.float32(step) * np.spacing(c0))
            if np.all(R.stn_coords_f32(np.array([[0, 0, c, 0, 0, c]], np.float32), 50, 7)[axis] == target):
                return c
        raise AssertionError("no float32 theta lands exactly on the integer")
    return np.array([0, 0, find(xt, 0), 0, 0, find(yt, 1)], np.float32)


@pytest.mark.parametrize("theta", ["identity", "past_last_row_and_column", "integer_coordinates", "negative_coordinates"])
def test_stn_sample_edges_with_known_theta(cuda_device, theta):
    """stn_sample_kernel at its edges: stn.dense_b.kernel = 0 and its bias = the affine transform, so the device theta is
    exactly that transform; the warped tap is checked against the float32-coordinate restatement."""
    known = {"identity": [1, 0, 0, 0, 1, 0],
             "past_last_row_and_column": [1.1, 0.05, 0.45, -0.03, 1.05, 0.3],          # samples past row 49 / column 6
             "integer_coordinates": _integer_theta(3, 20),
             "negative_coordinates": [0.9, 0.02, -0.6, 0.04, 1.1, -0.5]}[theta]
    w = dict(W.synthetic_crnn_weights(seed=2))
    w["stn.dense_b.kernel"] = np.zeros((64, 6), np.float32)
    w["stn.dense_b.bias"] = np.asarray(known, np.float32)
    taps = _run(_recognizer(w), 3, seed=11)
    assert np.array_equal(taps["theta"], np.tile(np.asarray(known, np.float32), (3, 1)).astype(np.float64))
    x, y = R.stn_coords_f32(taps["theta"].astype(np.float32), 50, 7)
    if theta == "past_last_row_and_column":
        assert (x > 7).any() and (y > 50).any()
    if theta == "negative_coordinates":
        assert (x < 0).any() and (y < 0).any()
    if theta == "integer_coordinates":
        assert (x == 3).all() and (y == 20).all()
    _check_warped(taps)


@pytest.mark.parametrize("k", [3, 37, 301, 1024])
def test_fc_ctc_logits_and_labels(cuda_device, k):
    alphabet = "0123456789abcdefghijklmnopqrstuvwxyz" if k == 37 else (
        "ab" if k == 3 else "".join(chr(0x4E00 + i) for i in range(k - 1)))
    w = W.synthetic_crnn_weights(seed=5, alphabet=alphabet)
    rec = _recognizer(w, alphabet=alphabet)
    taps = _run(rec, 9, seed=k)
    _check_logits(w, taps)
