"""Training the recognizer's output layer on the GPU (``b2o_crnn_features``, ``b2o_ctc_loss_grad``, ``b2o_rmsprop_step``,
``b2o_crnn_set_top``, ``Recognizer.fit_top``) against the fp64 references of tests/ctc_train_refs.py.

Bounds.  u = 2^-24, gamma(n) = n u / (1 - n u).
* Logits: the serial fmaf chain from the bias over 256 products is within gamma(257) (sum_c |x'_c w_ck| + |bias_k|) of
  the fp64 product of the same fp32 inputs (x' = the dropped-out features, rebuilt exactly by the reference).
* Loss: the reference runs on the kernel's own fp32 logits, so only the CTC arithmetic is judged.  The kernel's alpha is
  the lexicon kernel's (tests/test_gpu_lexicon.py derives its bound): with delta_t = 10u + 2u R_t + gamma(K + 8) the error
  of q at step t (R_t = the step's logit range) and eps = sum_t (3u + delta_t), L_b is within
  tau_L = 1.01 (eps + u) + u |L_b| + 1e-12.
* g = dL/dlogits (the workspace's first b * 48 * K floats): p carries delta_t, q delta_t + u.  Every alpha and beta state
  is within eps relative of exact (each update is at most two additions and a multiplication of non-negative numbers
  times a q, the rescaling is exact), so each fp64 product alpha beta is within 2 eps, and gamma = (its class's sum) / Z_t
  within 4 eps + 2u (sums of positive terms in fp64 add < 1e-15).  r = gamma / q and each term gamma p / q of D then
  carry 4 eps + 3 delta_t + 6u, and D the same plus the fp32 rounding.  g = p (D - r) rounded twice:
  |dg| <= |dp| |D - r| + p (|dD| + |dr|) + 2u |g| <= (4 eps + 4 delta_t + 10u) p (D + r).  The test uses
  tau_g = 1.01 (4 eps + 4 delta_t + 10u) p (D + r) + 1e-30 with p, D, r from the reference (r = gamma / q); the absolute
  1e-30 covers states that fall 2^134 below the largest and lose their bits as subnormals (no input here comes near).
* grad_W = (1/B) sum x' g: the chunked fmaf chains over n = B * 48 rows and the ordered sum of the chunks are within
  gamma(n + 1) sum |x' g| of the exact sum of the kernel's g, the division by B adds u; with the g errors,
  tau_W = (1/B) (sum |x'| tau_g + gamma(n + 1) sum |x' g|) + u |grad_W|, and grad_bias alike with x' = 1.
* RMSprop: acc = rho acc + (1 - rho) g^2 is four roundings of non-negative terms (the fp32 1 - rho one more): within 5u
  acc; the step lr g / (sqrt(acc) + eps) then within 10u relative; param within that plus u |param|.
The worst ratio to each bound is printed.

The loss and gradient check runs at b = 13 and 16 (one chunk of the split-K sums), 17 (a one-crop second chunk), 64 and
256 (4 and 16 chunks: the batch sizes training runs at), each case asserting its chunk count as read off the workspace
size the library reports; the bounds above hold for any chunking.  A final kernel that added only some chunks, used the
wrong chunk stride or divided by the wrong B fails there (RMSprop, being scale-free, would still train).  Measured on an
H100 80GB HBM3 (700 W), worst over all 12 cases and both dropout rates: logits 0.033, L_b 0.066, g 0.0043, grad_W
0.00087, grad_bias 0.00073 of their bounds.  Dropout keys of rows past 174,762 (row * 12,288 >= 2^31) are checked on a
200,004-row cache: logits 0.015, grad_W 0.043 of their bounds.  ``fit_top`` is restated call by call through the C ABI
and must match it bit for bit.  These checks add about 9 s to the file's run time on that H100.
"""
import numpy as np
import pytest
import torch

from keras_ocr_b200 import _lib, weights as W
from keras_ocr_b200.recognition import DEFAULT_ALPHABET, Lexicon, Recognizer
from tests import ctc_train_refs as TR

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
T = 48


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _gamma(n):
    return n * U / (1 - n * U)


@pytest.fixture(scope="module")
def ctx(cuda_device):
    return _lib.Context(0)


def _targets(rng, k, b):
    """b label sequences over K-1 labels: lengths 1..48, some with doubled letters, the longest alignable ones."""
    out = []
    for i in range(b):
        kind = i % 5
        if kind == 0:
            n = int(rng.integers(1, 4))
            seq = [int(c) for c in rng.integers(0, k - 1, n)]
        elif kind == 1 and k > 2:                                  # 48 labels, no doubled letter: the diagonal path only
            seq = [int(j % (k - 1)) for j in range(48)] if k > 2 else [0]
        elif kind == 2:                                            # doubled letters
            n = int(rng.integers(2, 12))
            seq = [int(c) for c in rng.integers(0, k - 1, n)]
            for j in range(1, n, 3):
                seq[j] = seq[j - 1]
        elif kind == 3:                                            # one label repeated: 24 copies need 47 steps
            seq = [int(rng.integers(0, k - 1))] * int(rng.integers(1, 25))
        else:
            n = int(rng.integers(10, 40))
            seq = [int(c) for c in rng.integers(0, k - 1, n)]
            while len(seq) + sum(a == b for a, b in zip(seq, seq[1:])) > 48:
                seq.pop()
        out.append(seq)
    return out


def _csr(targets):
    off = np.zeros(len(targets) + 1, np.int32)
    off[1:] = np.cumsum([len(t) for t in targets])
    lab = np.array([c for t in targets for c in t], np.int16)
    return torch.from_numpy(off).cuda(), torch.from_numpy(lab).cuda()


def _problem(k, n_rows, seed):
    rng = np.random.default_rng(seed)
    feats = np.tanh(rng.normal(size=(n_rows, T, 256)) * 1.5).astype(np.float16)     # LSTM outputs lie in (-1, 1)
    w = (rng.normal(size=(256, k)) * rng.choice([0.05, 0.3])).astype(np.float32)
    bias = (rng.normal(size=k) * 0.5).astype(np.float32)
    if k > 2:
        bias[k - 1] += 2.0                                         # blank-heavy, as a trained model is
    return rng, feats, w, bias


def run_loss_grad(ctx, feats_t, n_rows, index, k, w_t, b_t, off, lab, dropout, seed, step, grads=True):
    """(loss, grad_w, grad_b, logits, g) as host arrays (grads False: the loss-only call, g etc. None)."""
    b = len(index)
    idx = torch.from_numpy(np.asarray(index, np.int32)).cuda()
    loss = torch.empty(b, dtype=torch.float32, device="cuda")
    logits = torch.empty((b, T, k), dtype=torch.float32, device="cuda")
    gw = torch.empty((256, k), dtype=torch.float32, device="cuda") if grads else None
    gb = torch.empty(k, dtype=torch.float32, device="cuda") if grads else None
    nbytes = ctx.ctc_train_workspace_bytes(b, k)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    ptr = lambda t: t.data_ptr() if t is not None else None         # noqa: E731
    ctx.ctc_loss_grad(feats_t.data_ptr(), n_rows, idx.data_ptr(), b, k, w_t.data_ptr(), b_t.data_ptr(), off.data_ptr(),
                      lab.data_ptr(), dropout, seed, step, loss.data_ptr(), ptr(gw), ptr(gb), logits.data_ptr(),
                      ws.data_ptr() if grads else None, nbytes if grads else 0, _stream())
    g = ws[:b * T * k * 4].view(torch.float32).view(b, T, k).cpu().numpy() if grads else None
    host = lambda t: t.cpu().numpy() if t is not None else None     # noqa: E731
    return loss.cpu().numpy(), host(gw), host(gb), logits.cpu().numpy(), g


def _a256(x):
    return (x + 255) // 256 * 256


def device_chunks(ctx, b, k):
    """The number of split-K chunks the kernels sum grad_W over at batch b, read off the workspace size the library
    reports (g, then per chunk 256 x K and K partial sums, each slot 256-byte aligned)."""
    nbytes = ctx.ctc_train_workspace_bytes(b, k)
    found = [n for n in range(1, b + 1) if _a256(b * T * k * 4) + _a256(n * 256 * k * 4) + _a256(n * k * 4) == nbytes]
    assert len(found) == 1, (b, k, nbytes)
    return found[0]


# (b, K, chunks): batches of one chunk of 16 crops, of one crop more (a one-crop tail), and the batch sizes training runs
# at (64 by default, 256 in scripts/bench_fit_top.py); K = 37 is not a multiple of the 64-class tiles, 1024 the widest grid.
LOSS_GRAD_CASES = [(13, 2, 1), (13, 37, 1), (13, 38, 1), (13, 1024, 1), (16, 37, 1), (16, 1024, 1), (17, 37, 2),
                   (17, 1024, 2), (64, 37, 4), (64, 1024, 4), (256, 37, 16), (256, 1024, 16)]


# ------------------------------------------------------------------------------------------ 1. loss and gradient
@pytest.mark.parametrize("b,k,chunks", LOSS_GRAD_CASES,
                         ids=[str(k) if b == 13 else f"{k}-b{b}" for b, k, _ in LOSS_GRAD_CASES])
def test_loss_grad_vs_fp64(ctx, b, k, chunks):
    n_rows = b + 16
    assert device_chunks(ctx, b, k) == chunks
    rng, feats, w, bias = _problem(k, n_rows, seed=k if b == 13 else 1000 * b + k)
    targets = _targets(rng, k, b)
    off, lab = _csr(targets)
    index = rng.permutation(n_rows)[:b]
    ft, wt, bt = torch.from_numpy(feats).cuda(), torch.from_numpy(w).cuda(), torch.from_numpy(bias).cuda()
    report = []
    for dropout, seed, step in ((0.0, 0, 0), (0.25, 7, 3)):
        loss, gw, gb, logits, g = run_loss_grad(ctx, ft, n_rows, index, k, wt, bt, off, lab, dropout, seed, step)
        x = TR.dropped(feats, index, dropout, seed, step)
        ref_lg = TR.logits(x, w, bias)
        tau_lg = _gamma(257) * (np.abs(x).astype(np.float64) @ np.abs(w).astype(np.float64) + np.abs(bias))
        r_lg = np.abs(logits - ref_lg) / tau_lg
        assert r_lg.max() <= 1.0, (k, dropout, float(r_lg.max()))
        lgd = logits.astype(np.float64)
        delta = 10 * U + 2 * U * (lgd.max(-1) - lgd.min(-1)) + _gamma(k + 8)           # (b, 48)
        eps = (3 * U + delta).sum(-1)                                                  # (b,)
        ref_g, tau_g, r_l = np.zeros_like(lgd), np.zeros_like(lgd), 0.0
        for i in range(b):
            L, gi, info = TR.loss_grad(lgd[i], targets[i])
            tau_l = 1.01 * (eps[i] + U) + U * abs(L) + 1e-12
            r_l = max(r_l, abs(float(loss[i]) - L) / tau_l)
            assert abs(float(loss[i]) - L) <= tau_l, (k, dropout, i, float(loss[i]), L)
            p, q, gam, D = info["p"], info["q"], info["gamma"], info["D"]
            ref_g[i] = gi
            tau_g[i] = 1.01 * (4 * eps[i] + 4 * delta[i][:, None] + 10 * U) * p * (D[:, None] + gam / q) + 1e-30
        r_g = np.abs(g - ref_g) / tau_g
        assert r_g.max() <= 1.0, (k, dropout, float(r_g.max()))
        n = b * T
        xd = x.astype(np.float64)
        ref_w = np.einsum("btc,btk->ck", xd, g.astype(np.float64), optimize=True) / b
        tau_w = (np.einsum("btc,btk->ck", np.abs(xd), tau_g, optimize=True) + _gamma(n + 1) *
                 np.einsum("btc,btk->ck", np.abs(xd), np.abs(g.astype(np.float64)), optimize=True)) / b + \
            U * np.abs(ref_w) + 1e-30
        ref_gw, ref_gb = TR.batch_grads(x, ref_g)
        r_w = np.abs(gw - ref_gw) / tau_w
        tau_b = (tau_g.sum((0, 1)) + _gamma(n + 1) * np.abs(g).sum((0, 1))) / b + U * np.abs(ref_gb) + 1e-30
        r_b = np.abs(gb - ref_gb) / tau_b
        assert r_w.max() <= 1.0 and r_b.max() <= 1.0, (k, dropout, float(r_w.max()), float(r_b.max()))
        loss_only = run_loss_grad(ctx, ft, n_rows, index, k, wt, bt, off, lab, dropout, seed, step, grads=False)[0]
        assert np.array_equal(loss_only.view(np.int32), loss.view(np.int32))
        report.append(f"dropout {dropout}: worst logits {r_lg.max():.3g}, L_b {r_l:.3g}, g {r_g.max():.3g}, "
                      f"grad_W {r_w.max():.3g}, grad_bias {r_b.max():.3g} of their bounds")
    print(f"ctc_loss_grad b={b} ({chunks} chunks) K={k}: " + "; ".join(report))


def test_invalid_targets_and_rows(ctx):
    k, n_rows = 37, 6
    rng, feats, w, bias = _problem(k, n_rows, seed=1)
    targets = [[1, 2], [], [k - 1], [3] * 25, [4, 5], [6]]
    off, lab = _csr(targets)
    ft, wt, bt = torch.from_numpy(feats).cuda(), torch.from_numpy(w).cuda(), torch.from_numpy(bias).cuda()
    loss, gw, gb, _, g = run_loss_grad(ctx, ft, n_rows, [0, 1, 2, 3, 4, 99], k, wt, bt, off, lab, 0.0, 0, 0)
    assert np.isfinite(loss[[0, 4]]).all() and np.all(loss[1:4] == np.inf) and np.isnan(loss[5])
    assert not g[1:4].any() and not g[5].any()
    ok, gw2, gb2, _, _ = run_loss_grad(ctx, ft, n_rows, [0, 4], k, wt, bt, *_csr([[1, 2], [4, 5]]), 0.0, 0, 0)
    assert np.array_equal(ok.view(np.int32), loss[[0, 4]].view(np.int32))
    # the invalid crops add nothing: the sums are those of the two valid crops, divided by 6 instead of 2
    assert np.allclose(gw * 6, gw2 * 2, rtol=1e-5, atol=1e-7) and np.allclose(gb * 6, gb2 * 2, rtol=1e-5, atol=1e-7)


# dataset rows whose dropout key row * 48 * 256 passes 2^31 (174,763 * 12,288 > 2^31): the key must be formed in 64 bits
BIG_ROWS = np.array([0, 174_763, 200_003])
BIG_N_ROWS = 200_004


def test_dropout_keys_past_2_31(ctx):
    """The logits of crops at rows 174,763 and 200,003 of a 200,004-row cache (4.9 GB of features, only the used rows
    written) against fp64 on the mask rebuilt from 64-bit keys, within the gamma(257) bound of section 1."""
    assert int(BIG_ROWS[1]) * T * 256 >= 2 ** 31 > (int(BIG_ROWS[1]) - 1) * T * 256
    k, dropout, seed, step = 38, 0.25, 7, 3
    rng, small, w, bias = _problem(k, len(BIG_ROWS), seed=31)
    feats = torch.empty((BIG_N_ROWS, T, 256), dtype=torch.float16, device="cuda")
    try:
        feats[torch.from_numpy(BIG_ROWS).cuda()] = torch.from_numpy(small).cuda()
        targets = _targets(rng, k, len(BIG_ROWS))
        off, lab = _csr(targets)
        wt, bt = torch.from_numpy(w).cuda(), torch.from_numpy(bias).cuda()
        loss, gw, gb, logits, g = run_loss_grad(ctx, feats, BIG_N_ROWS, BIG_ROWS, k, wt, bt, off, lab, dropout, seed,
                                                step)
    finally:
        del feats
        torch.cuda.empty_cache()
    x = TR.drop(small, BIG_ROWS, dropout, seed, step)
    tau = _gamma(257) * (np.abs(x).astype(np.float64) @ np.abs(w).astype(np.float64) + np.abs(bias))
    r = np.abs(logits - TR.logits(x, w, bias)) / tau
    # grad_partial_kernel forms the mask again: grad_W on the device's own g, within section 1's chain bound
    xd, gd = x.astype(np.float64), g.astype(np.float64)
    ref_w = np.einsum("btc,btk->ck", xd, gd) / len(BIG_ROWS)
    tau_w = _gamma(len(BIG_ROWS) * T + 1) * np.einsum("btc,btk->ck", np.abs(xd), np.abs(gd)) / len(BIG_ROWS) + \
        U * np.abs(ref_w) + 1e-30
    r_w = np.abs(gw - ref_w) / tau_w
    print(f"dropout keys past 2^31: worst logits {r.max():.3g}, grad_W {r_w.max():.3g} of their bounds")
    assert np.isfinite(loss).all() and r.max() <= 1.0 and r_w.max() <= 1.0


# ------------------------------------------------------------------------------------------ 2.-3. through the CRNN
def _synth(seeds):
    from oracle.train_crnn_full import synth_crop
    made = [synth_crop(s) for s in seeds]
    return np.stack([m[0] for m in made]), [m[1] for m in made]


def _input(rec, crops):
    t = torch.from_numpy(np.ascontiguousarray(crops)).cuda()
    x = torch.empty((len(crops), 200, 31), dtype=torch.float16, device="cuda")
    rec.ctx.crops_to_input(t.data_ptr(), len(crops), x.data_ptr(), _stream())
    return x


def test_features_logits_and_lexicon_agree(ctx):
    hw = W.synthetic_crnn_weights(decisive=True)
    rec = Recognizer(weights=hw)
    rec.keep_workspace = True
    crops, words = _synth(range(70_000_000, 70_000_045))
    b = len(crops)
    x = _input(rec, crops)
    rec.predict_device(x)
    logits_inf = rec.tap("logits", (b, T, 37), torch.float32).cpu().numpy()
    l2 = rec.tap("l2", (b, 50, 256), torch.float16).cpu().numpy()
    feats = torch.empty((b, T, 256), dtype=torch.float16, device="cuda")
    nbytes = rec.ctx.crnn_workspace_bytes(b)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    n0 = rec.ctx.launch_count()
    rec.ctx.crnn_features(x.data_ptr(), b, feats.data_ptr(), ws.data_ptr(), nbytes, _stream())
    assert np.array_equal(feats.cpu().numpy().view(np.int16), l2[:, 2:].view(np.int16))
    n_feat_launches = rec.ctx.launch_count() - n0
    targets = [[rec.alphabet.index(c) for c in wd] for wd in words]
    off, lab = _csr(targets)
    wt = torch.from_numpy(hw["fc_12.kernel"]).cuda()
    bt = torch.from_numpy(hw["fc_12.bias"]).cuda()
    loss, *_, logits, _ = run_loss_grad(ctx, feats, b, np.arange(b), 37, wt, bt, off, lab, 0.0, 0, 0)
    assert np.array_equal(logits.view(np.int32), logits_inf.view(np.int32))     # the logits inference decodes
    # L_b = -(lexicon score of the crop's own text), within both kernels' bounds (equal by construction)
    lgd = logits.astype(np.float64)
    delta = 10 * U + 2 * U * (lgd.max(-1) - lgd.min(-1)) + _gamma(37 + 8)
    same = 0
    for i in range(b):
        lex = Lexicon([words[i]], rec.alphabet)
        o, lb = lex.device_arrays("cuda")
        out = torch.empty((1, 1, T), dtype=torch.int32, device="cuda")
        lp = torch.empty((1, 1), dtype=torch.float32, device="cuda")
        lws = torch.empty(ctx.lexicon_workspace_bytes(1, 1, 1), dtype=torch.uint8, device="cuda")
        ctx.ctc_lexicon_decode(torch.from_numpy(logits[i:i + 1]).cuda().data_ptr(), 1, 37, o.data_ptr(), lb.data_ptr(),
                               1, 1, out.data_ptr(), lp.data_ptr(), lws.data_ptr(), lws.numel(), _stream())
        score = float(lp.cpu().numpy()[0, 0])
        tau = 1.01 * ((3 * U + delta[i]).sum() + U) + U * abs(score) + 1e-12
        assert abs(float(loss[i]) + score) <= 2 * tau, (i, float(loss[i]), score)
        same += float(loss[i]) == -score
    print(f"features: {n_feat_launches} launches, bit-identical to the l2 tap; logits bit-identical to inference; "
          f"L_b = -lexicon score bit for bit on {same}/{b} crops")


# ------------------------------------------------------------------------------------------ 4. determinism
def test_determinism_and_batch_independence(ctx):
    k, n_rows, b = 38, 40, 37
    rng, feats, w, bias = _problem(k, n_rows, seed=9)
    targets = _targets(rng, k, b)
    index = rng.permutation(n_rows)[:b]
    ft, wt, bt = torch.from_numpy(feats).cuda(), torch.from_numpy(w).cuda(), torch.from_numpy(bias).cuda()
    off, lab = _csr(targets)
    a = run_loss_grad(ctx, ft, n_rows, index, k, wt, bt, off, lab, 0.25, 5, 11)
    c = run_loss_grad(ctx, ft, n_rows, index, k, wt, bt, off, lab, 0.25, 5, 11)
    for x, y in zip(a, c):
        assert np.array_equal(x.view(np.int32), y.view(np.int32))
    perm = rng.permutation(b)
    p = run_loss_grad(ctx, ft, n_rows, index[perm], k, wt, bt, *_csr([targets[i] for i in perm]), 0.25, 5, 11)
    assert np.array_equal(p[0].view(np.int32), a[0][perm].view(np.int32))
    one = run_loss_grad(ctx, ft, n_rows, index[3:4], k, wt, bt, *_csr(targets[3:4]), 0.25, 5, 11)
    assert one[0].view(np.int32)[0] == a[0].view(np.int32)[3]


# ------------------------------------------------------------------------------------------ 5. RMSprop and set_top
def test_rmsprop_vs_fp64(ctx):
    rng = np.random.default_rng(2)
    n = 5000
    param = rng.normal(size=n).astype(np.float32)
    acc = np.abs(rng.normal(size=n) * 1e-3).astype(np.float32)
    acc[:100] = 0
    grad = (rng.normal(size=n) * 10.0 ** rng.uniform(-6, 0, n)).astype(np.float32)
    pt, gt, at = (torch.from_numpy(a.copy()).cuda() for a in (param, grad, acc))
    ctx.rmsprop_step(pt.data_ptr(), gt.data_ptr(), at.data_ptr(), n, 1e-3, 0.9, 1e-7, _stream())
    ref_p, ref_a = TR.rmsprop(param, grad, acc.astype(np.float64), 1e-3, np.float64(np.float32(0.9)), 1e-7)
    step = ref_p - param.astype(np.float64)
    r_a = np.abs(at.cpu().numpy() - ref_a) / (5 * U * ref_a + 1e-45)
    r_p = np.abs(pt.cpu().numpy() - ref_p) / (10 * U * np.abs(step) + U * np.abs(ref_p) + 1e-45)
    assert r_a.max() <= 1.0 and r_p.max() <= 1.0, (float(r_a.max()), float(r_p.max()))
    print(f"rmsprop: worst acc {r_a.max():.3g}, param {r_p.max():.3g} of their bounds")


def test_set_top(ctx):
    hw = W.synthetic_crnn_weights(decisive=True)
    rng = np.random.default_rng(4)
    top_w = (hw["fc_12.kernel"] + rng.normal(size=(256, 37)).astype(np.float32) * 0.3).astype(np.float32)
    top_b = (hw["fc_12.bias"] + rng.normal(size=37).astype(np.float32)).astype(np.float32)
    crops, _ = _synth(range(71_000_000, 71_000_064))
    rec = Recognizer(weights=hw)
    wt, bt = torch.from_numpy(top_w).cuda(), torch.from_numpy(top_b).cuda()
    rec.ctx.crnn_set_top(wt.data_ptr(), bt.data_ptr(), 37, _stream())
    other = Recognizer(weights=dict(hw, **{"fc_12.kernel": top_w, "fc_12.bias": top_b}))
    x = _input(rec, crops)
    assert np.array_equal(rec.predict_device(x).cpu().numpy(), other.predict_device(x).cpu().numpy())
    assert rec.ctx.lib.b2o_crnn_set_top(rec.ctx.handle, wt.data_ptr(), bt.data_ptr(), 38, None) == -2
    assert rec.ctx.lib.b2o_crnn_set_top(rec.ctx.handle, None, bt.data_ptr(), 37, None) == -2


# ------------------------------------------------------------------------------------------ 6.-7. end to end
N_TRAIN, N_HELD = 4096, 1024
EPOCHS, LR = 16, 3e-3
TRAIN_SEEDS = range(80_000_000, 80_000_000 + N_TRAIN)           # disjoint from each other and from the fixture's
HELD_SEEDS = range(90_000_000, 90_000_000 + N_HELD)              # training seeds (10_000_000 + i)
MARGIN = 0.01


@pytest.fixture(scope="module")
def word_crops():
    return _synth(TRAIN_SEEDS), _synth(HELD_SEEDS)


def _rate(rec, crops, words):
    got = rec.recognize_crops(crops)
    return float(np.mean([a == b for a, b in zip(got, words)])), got


def test_fit_top_new_alphabet(ctx, word_crops, tmp_path):
    import time
    (tc, tw), (hc, hwords) = word_crops
    hw = W.synthetic_crnn_weights(decisive=True)
    base, _ = _rate(Recognizer(weights=hw), hc, hwords)
    alphabet = DEFAULT_ALPHABET[::-1] + "-"                       # 38 classes, every label re-indexed
    rec = Recognizer(alphabet=alphabet, weights=hw)
    before, _ = _rate(rec, hc, hwords)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    hist = rec.fit_top(tc, tw, epochs=EPOCHS, batch_size=64, learning_rate=LR, seed=3, validation=(hc[:512], hwords[:512]))
    torch.cuda.synchronize()
    secs = time.perf_counter() - t0
    rate, got = _rate(rec, hc, hwords)
    print(f"fit_top, new alphabet: held-out exact reads {before:.4f} before, {rate:.4f} after ({EPOCHS} epochs of "
          f"{N_TRAIN} crops, {secs:.2f} s); the trained model reads {base:.4f}; loss {hist['loss']}; "
          f"val_loss {hist['val_loss']}")
    assert len(hist["loss"]) == len(hist["val_loss"]) == EPOCHS
    assert hist["val_loss"][-1] < hist["val_loss"][0]
    assert rate >= base - MARGIN
    path = str(tmp_path / "fitted.npz")
    rec.save_weights(path)
    loaded = Recognizer(alphabet=alphabet, weights=path)
    assert loaded.recognize_crops(hc) == got
    rec2 = Recognizer(alphabet=alphabet, weights=hw)             # the same run again: bit-identical weights
    rec2.fit_top(tc[:2048], tw[:2048], epochs=2, batch_size=64, learning_rate=LR, seed=3)
    rec3 = Recognizer(alphabet=alphabet, weights=hw)
    rec3.fit_top(tc[:2048], tw[:2048], epochs=2, batch_size=64, learning_rate=LR, seed=3)
    for name in ("fc_12.kernel", "fc_12.bias"):
        assert np.array_equal(rec2._tensors[name].view(np.int32), rec3._tensors[name].view(np.int32))


def test_fine_tuning_does_no_harm(ctx, word_crops):
    (tc, tw), (hc, hwords) = word_crops
    hw = W.synthetic_crnn_weights(decisive=True)
    rec = Recognizer(weights=hw)
    before, _ = _rate(rec, hc, hwords)
    rec.fit_top(tc[:2048], tw[:2048], epochs=1, batch_size=64, seed=1)
    after, _ = _rate(rec, hc, hwords)
    print(f"fine-tuning the trained top: held-out exact reads {before:.4f} -> {after:.4f}")
    assert after >= before


def _logits(rec, crops):
    rec.keep_workspace = True
    rec.predict_device(_input(rec, crops))
    return rec.tap("logits", (len(crops), T, len(rec.alphabet) + 1), torch.float32).cpu().numpy()


def test_fit_top_is_its_abi_calls(ctx, tmp_path):
    """fit_top, restated as the calls its docstring describes: per epoch a default_rng(seed) permutation, batches of
    batch_size in its order with a short last one (70 = 32 + 32 + 6), dropout keyed on a step counter that runs on
    across epochs, two RMSprop accumulators carried over, the history as the means of the fp32 losses, the validation
    loss without dropout after each epoch.  Tensors and history bit for bit; the installed top reads like a recognizer
    loaded from save_weights."""
    n, bs, epochs, lr, dropout, seed = 70, 32, 2, 3e-3, 0.25, 5
    hw = W.synthetic_crnn_weights(decisive=True)
    crops, words = _synth(range(75_000_000, 75_000_000 + n))
    v_crops, v_words = _synth(range(75_100_000, 75_100_019))
    rec = Recognizer(weights=hw)
    hist = rec.fit_top(crops, words, epochs=epochs, batch_size=bs, learning_rate=lr, dropout=dropout, seed=seed,
                       validation=(v_crops, v_words))
    k = len(rec.alphabet) + 1
    ref = Recognizer(weights=hw)

    def features(c):
        x = _input(ref, c)
        out = torch.empty((len(c), T, 256), dtype=torch.float16, device="cuda")
        ws = torch.empty(ref.ctx.crnn_workspace_bytes(len(c)), dtype=torch.uint8, device="cuda")
        ref.ctx.crnn_features(x.data_ptr(), len(c), out.data_ptr(), ws.data_ptr(), ws.numel(), _stream())
        return out
    feats, v_feats = features(crops), features(v_crops)
    labels = [[rec.alphabet.index(c) for c in wd] for wd in words]
    v_labels = [[rec.alphabet.index(c) for c in wd] for wd in v_words]
    w = torch.from_numpy(hw["fc_12.kernel"].copy()).cuda()
    bias = torch.from_numpy(hw["fc_12.bias"].copy()).cuda()
    acc_w, acc_b = torch.zeros_like(w), torch.zeros_like(bias)
    rng = np.random.default_rng(seed)
    want = {"loss": [], "val_loss": []}
    step = 0
    for _ in range(epochs):
        perm = rng.permutation(n)
        seen = np.empty(n, np.float32)
        for i in range(0, n, bs):
            idx = perm[i:i + bs]
            loss, gw, gb, _, _ = run_loss_grad(ctx, feats, n, idx, k, w, bias, *_csr([labels[j] for j in idx]),
                                               dropout, seed, step)
            seen[i:i + len(idx)] = loss
            for p, g, a in ((w, gw, acc_w), (bias, gb, acc_b)):
                gt = torch.from_numpy(g).cuda()
                ctx.rmsprop_step(p.data_ptr(), gt.data_ptr(), a.data_ptr(), p.numel(), lr, 0.9, 1e-7, _stream())
            step += 1
        want["loss"].append(float(seen.astype(np.float64).mean()))
        v_loss = run_loss_grad(ctx, v_feats, len(v_crops), np.arange(len(v_crops)), k, w, bias, *_csr(v_labels), 0.0,
                               0, 0, grads=False)[0]
        want["val_loss"].append(float(v_loss.astype(np.float64).mean()))
    assert step == 6 and hist == want, (hist, want)
    for name, t in (("fc_12.kernel", w), ("fc_12.bias", bias)):
        assert np.array_equal(rec._tensors[name].view(np.int32), t.cpu().numpy().view(np.int32)), name
    path = str(tmp_path / "top.npz")
    rec.save_weights(path)
    assert np.array_equal(_logits(rec, v_crops).view(np.int32), _logits(Recognizer(weights=path), v_crops).view(np.int32))
    print(f"fit_top as its ABI calls: history {hist}")


# ------------------------------------------------------------------------------------------ 8. argument checks
def test_abi_rejects_bad_arguments(ctx):
    lib, h = ctx.lib, ctx.handle
    k, b = 37, 2
    feats = torch.zeros((4, T, 256), dtype=torch.float16, device="cuda")
    w = torch.zeros((256, 1025), dtype=torch.float32, device="cuda")
    bias = torch.zeros(1025, dtype=torch.float32, device="cuda")
    off, lab = _csr([[1], [2]])
    loss = torch.empty(b, dtype=torch.float32, device="cuda")
    gw, gb = torch.empty_like(w), torch.empty_like(bias)
    nbytes = ctx.ctc_train_workspace_bytes(b, k)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    P = lambda t: t.data_ptr()                                    # noqa: E731

    def call(kk=k, bb=b, dropout=0.0, n_rows=4, f=P(feats), g_w=P(gw), g_b=P(gb), size=nbytes, wsp=P(ws)):
        return lib.b2o_ctc_loss_grad(h, f, n_rows, None, bb, kk, P(w), P(bias), P(off), P(lab), dropout, 0, 0, P(loss),
                                     g_w, g_b, None, wsp, size, None)
    assert call() == 0
    for kwargs in ({"kk": 1}, {"kk": 1025}, {"dropout": 1.0}, {"dropout": -0.1}, {"dropout": float("nan")},
                   {"bb": -1}, {"n_rows": 0}, {"f": None}, {"f": P(feats) + 2}, {"g_b": None}):
        assert call(**kwargs) == -2, kwargs
        assert lib.b2o_last_error(h)
    assert call(size=nbytes - 1) == -4 and call(wsp=None) == -4
    assert call(g_w=None, g_b=None, wsp=None, size=0) == 0          # the loss alone needs no workspace
    assert lib.b2o_ctc_train_workspace_bytes(2, 1) == 0 and lib.b2o_ctc_train_workspace_bytes(0, 37) == 0
    assert lib.b2o_rmsprop_step(h, P(gw), P(gw), P(gw), -1, 1e-3, 0.9, 1e-7, None) == -2
    assert lib.b2o_rmsprop_step(h, None, P(gw), P(gw), 10, 1e-3, 0.9, 1e-7, None) == -2
    assert lib.b2o_rmsprop_step(h, P(gw), P(gw), P(gw), 10, 1e-3, 1.5, 1e-7, None) == -2
    rec = Recognizer(weights=W.synthetic_crnn_weights(decisive=True))
    assert rec.ctx.lib.b2o_crnn_features(rec.ctx.handle, P(feats), 2, None, P(ws), nbytes, None) == -2
    small = rec.ctx.crnn_workspace_bytes(2) - 1
    big = torch.empty(small + 1, dtype=torch.uint8, device="cuda")
    xin = torch.zeros((2, 200, 31), dtype=torch.float16, device="cuda")
    assert rec.ctx.lib.b2o_crnn_features(rec.ctx.handle, P(xin), 2, P(feats), P(big), small, None) == -4
    torch.cuda.synchronize()


def test_fit_top_rejects_before_launching(ctx):
    rec = Recognizer(weights=W.synthetic_crnn_weights(decisive=True))
    crops = np.full((3, 31, 200), 255, np.uint8)
    n0 = rec.ctx.launch_count()
    for texts in (["ab", "", "c"], ["ab", "A", "c"], ["ab", "x" * 49, "c"], ["ab", "oo" * 13, "c"], ["a", "b"]):
        with pytest.raises(ValueError):
            rec.fit_top(crops, texts)
    with pytest.raises(ValueError, match="text 1"):
        rec.fit_top(crops, ["ab", "AB", "c"])
    for kwargs in ({"epochs": 0}, {"batch_size": 0}, {"learning_rate": -1.0}, {"dropout": 1.0}, {"seed": -1},
                   {"validation": (crops, ["a", "b", ""])}, {"validation": (crops[:2], ["a", "b", "c"])}):
        with pytest.raises(ValueError):
            rec.fit_top(crops, ["a", "b", "c"], **kwargs)
    with pytest.raises(ValueError):
        rec.fit_top(crops[:, :30], ["a", "b", "c"])
    assert rec.ctx.launch_count() == n0
