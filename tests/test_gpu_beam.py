"""CTC beam-search decoding on the GPU (``b2o_ctc_beam_decode``, ``b2o_crnn_forward_beam``) against tests/beam_refs.py.

Bound.  The fp64 reference runs on the same fp32 logits.  Let u = 2^-24, R_t = max_c l - min_c l of step t.  The kernel's
lp[t,c] = logf(expf(l_c - m) / s + 1e-7): the subtraction costs u |l_c - m| <= u R_t relative after the exponential,
expf 2 ulp (4u), the fixed-order sum s of K positive terms gamma(K + 8) relative with its own terms' errors, the division
and the + 1e-7 one rounding each, so p_c + 1e-7 is within (10u + 2u R_t + gamma(K + 8)) relative; logf turns that into
an absolute error (x 1.01) plus one ulp of the result, 2u |lp|.  That is d_t, the per-step bound on |lp_fp32 - lp|.
A beam's p_b and p_nb are sums of lp along its history, merged by logaddexp; logaddexp is 1-Lipschitz in the max-norm of
its arguments, so input errors carry over unchanged and each step adds d_t and its own rounding: one fp32 addition
(u |v|), at most three logaddexp (each u |v| for the final addition and about 6u for expf / log1pf of a value <= 1).
|v| <= V = sum_t max_c |lp[t,c]| + 1 bounds every score (a path's terms are lp values; the merged mass is at most
(1 + K 1e-7)^48).  Hence every fp32 score is within  tau = sum_t d_t + 48 (4u V + 24u)  of the exact score of the same
beam.  When the reference's smallest selection gap (``prune_margin``) and the gap between consecutive returned paths
(``rank_margin``) both exceed 2 tau, the kernel keeps and orders exactly the same beams: labels identical and
|logp - ref| <= tau.  Otherwise (a near-tie) each returned path still satisfies logp <= its exact forward
log-probability + tau, since a beam score sums a subset of the path's alignments.  The worst ratio to tau is printed;
DESIGN.md section 2 records it.
"""
import os

import numpy as np
import pytest
import torch

from keras_ocr_b200 import _lib, weights as W
from tests import beam_refs as BR

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
T = 48


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _gamma(n):
    return n * U / (1 - n * U)


def tau(logits):
    """(B,) bound of the module docstring for (B,48,K) fp32 logits."""
    lg = np.asarray(logits, np.float64)
    lp = BR.log_probs(lg)
    k = lg.shape[-1]
    d = 1.01 * (10 * U + 2 * U * (lg.max(-1) - lg.min(-1)) + _gamma(k + 8)) + 2 * U * np.abs(lp).max(-1)
    v = np.abs(lp).max(-1).sum(-1) + 1.0
    return d.sum(-1) + T * (4 * U * v + 24 * U)


@pytest.fixture(scope="module")
def ctx(cuda_device):
    return _lib.Context(0)


def decode(ctx, logits, w, p):
    x = torch.from_numpy(np.ascontiguousarray(logits, np.float32)).cuda()
    b, _, k = x.shape
    labels = torch.empty((b, p, T), dtype=torch.int32, device="cuda")
    logp = torch.empty((b, p), dtype=torch.float32, device="cuda")
    ctx.ctc_beam_decode(x.data_ptr(), b, k, w, p, labels.data_ptr(), logp.data_ptr(), _stream())
    return labels.cpu().numpy(), logp.cpu().numpy()


def _rows(paths, p):
    out = np.full((p, T), -1, np.int32)
    for i, s in enumerate(paths):
        out[i, :len(s)] = s
    return out


def check_against_ref(logits, labels, logp, w, what):
    """Per crop: identical beams where the reference's margins exceed 2 tau, the forward bound elsewhere.  Returns
    (worst |logp - ref| / tau over crops with identical labels, number of near-tie crops)."""
    taus = tau(logits)
    lps = BR.log_probs(logits)
    worst, near = 0.0, 0
    for i in range(len(logits)):
        p = labels.shape[1]
        paths, ref, info = BR.beam_search(lps[i], w, top_paths=p)
        got = [tuple(int(c) for c in row if c >= 0) for row in labels[i, :len(paths)]]
        assert np.all(np.diff(logp[i, :len(paths)]) <= 0), (what, i)
        assert len(set(got)) == len(got), (what, i)
        same = got == paths
        if min(info["prune_margin"], info["rank_margin"]) > 2 * taus[i]:
            assert same, (what, i, info, taus[i])
        if same:
            r = float(np.abs(logp[i, :len(paths)] - ref).max() / taus[i])
            assert r <= 1.0, (what, i, r)
            worst = max(worst, r)
        else:
            near += 1
            for s, v in zip(got, logp[i]):
                assert v <= BR.forward_logprob(lps[i], s) + taus[i], (what, i, s)
    return worst, near


def crafted(k, b, seed):
    """Random logits at several temperatures, peaked ones, and deliberate near-ties (two labels, or a label and blank,
    a few fp32 ulps apart)."""
    rng = np.random.default_rng(seed)
    out = np.empty((b, T, k), np.float32)
    for i in range(b):
        kind = i % 6
        x = rng.normal(size=(T, k))
        if kind == 0:
            x /= 0.3
        elif kind == 2:
            x *= 3.0
        elif kind == 3:                                           # peaked: the greedy path dominates
            x[np.arange(T), rng.integers(0, k, T)] += 30.0
        elif kind == 4:                                           # near-ties between the two best labels of a step
            top = rng.integers(0, k, (T, 2))
            x[np.arange(T), top[:, 0]] = 4.0
            x[np.arange(T), top[:, 1]] = np.nextafter(np.float32(4.0), np.float32(5.0))
        elif kind == 5:                                           # realistic: blank mostly, a label now and then
            x[:, k - 1] += 6.0
            x[::5, rng.integers(0, k - 1)] += 8.0
        out[i] = x
    return out


# ------------------------------------------------------------------------------------------ 1. the decoder alone
@pytest.mark.parametrize("k", [3, 37, 301, 1024])
def test_decoder_vs_fp64(ctx, k):
    report = []
    for w in (1, 2, 5, 100, 128):
        logits = crafted(k, 17, seed=k * 1000 + w)
        labels, logp = decode(ctx, logits, w, w)
        worst, near = check_against_ref(logits, labels, logp, w, (k, w))
        report.append(f"W={w}: worst {worst:.3g} of tau, near-tie crops {near}/17")
        for p in sorted({1, 3} & set(range(1, w + 1))):          # fewer paths: the first rows of the same search
            lab_p, lp_p = decode(ctx, logits, w, p)
            assert np.array_equal(lab_p, labels[:, :p]) and np.array_equal(lp_p.view(np.int32), logp[:, :p].view(np.int32))
        for b in (1, 7):                                          # a crop decodes alike in any batch
            lab_b, lp_b = decode(ctx, logits[:b], w, w)
            assert np.array_equal(lab_b, labels[:b]) and np.array_equal(lp_b.view(np.int32), logp[:b].view(np.int32))
        lab2, lp2 = decode(ctx, logits, w, w)                     # and on every run
        assert np.array_equal(lab2, labels) and np.array_equal(lp2.view(np.int32), logp.view(np.int32))
    print(f"beam K={k}: " + "; ".join(report))


@pytest.mark.parametrize("k", [3, 37, 1024])
def test_decoder_uniform_tie_rule(ctx, k):
    """Uniform logits: every step ties exactly.  The kernel orders equal fp32 scores by label sequence, and decodes as
    the reference does except where two differently shaped prefixes have equal exact scores (their computed scores
    then differ in the last bits, a near-tie of the margin rule)."""
    logits = np.zeros((2, T, k), np.float32)
    for w in (5, 128):
        labels, logp = decode(ctx, logits, w, w)
        assert np.array_equal(labels[0], labels[1])
        for i in range(w - 1):
            if logp[0, i] == logp[0, i + 1] and labels[0, i + 1, 0] >= 0:
                a = tuple(int(c) for c in labels[0, i] if c >= 0)
                b = tuple(int(c) for c in labels[0, i + 1] if c >= 0)
                assert a < b, (k, w, i)
        worst, near = check_against_ref(logits[:1], labels[:1], logp[:1], w, ("uniform", k, w))
        paths, _, _ = BR.beam_search(BR.log_probs(logits[0]), w, top_paths=w)
        same = sum(tuple(int(c) for c in row if c >= 0) == s for row, s in zip(labels[0], paths))
        print(f"uniform K={k} W={w}: {same}/{len(paths)} paths identical to the reference, near-tie crops {near}")


def test_decoder_c3_logits(cuda_device, ctx, golden_dir):
    from keras_ocr_b200.recognition import Recognizer
    g = np.load(os.path.join(golden_dir, "c3_crops.npz"))
    rec = Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True))
    rec.keep_workspace = True
    x = _input(rec, g["crops"])
    greedy = rec.predict_device(x).cpu().numpy()
    logits = rec.tap("logits", (256, T, 37), torch.float32).cpu().numpy()
    for w in (1, 10, 100):
        labels, logp = decode(ctx, logits, w, min(w, 3))
        worst, near = check_against_ref(logits, labels, logp, w, ("c3", w))
        differ = int((labels[:, 0] != greedy).any(-1).sum())
        print(f"C3 W={w}: worst {worst:.3g} of tau, near-tie crops {near}/256, top-1 differs from greedy on {differ}")


# ------------------------------------------------------------------------------------------ 2. through the CRNN
def _input(rec, crops):
    t = torch.from_numpy(np.ascontiguousarray(crops)).to(rec.device)
    x = torch.empty((len(crops), 200, 31), dtype=torch.float16, device=rec.device)
    rec.ctx.crops_to_input(t.data_ptr(), len(crops), x.data_ptr(), _stream())
    return x


def test_crnn_forward_beam(cuda_device, ctx, golden_dir):
    from keras_ocr_b200.recognition import Recognizer
    crops = np.load(os.path.join(golden_dir, "c3_crops.npz"))["crops"][:17]
    rec = Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True))
    rec.keep_workspace = True
    x = _input(rec, crops)
    labels, logp = rec.predict_device(x, with_scores=True, beam_width=10, top_paths=3)
    assert labels.shape == (17, 3, T) and logp.shape == (17, 3)
    labels, logp = labels.cpu().numpy(), logp.cpu().numpy()
    logits = rec.tap("logits", (17, T, 37), torch.float32).cpu().numpy()
    lab_d, lp_d = decode(ctx, logits, 10, 3)                      # the decoder alone on the device's own logits
    assert np.array_equal(lab_d, labels) and np.array_equal(lp_d.view(np.int32), logp.view(np.int32))
    again = rec.predict_device(x, with_scores=True, beam_width=10, top_paths=3)
    assert np.array_equal(again[0].cpu().numpy(), labels) and np.array_equal(again[1].cpu().numpy(), logp)
    for i in (0, 8, 16):
        la, lpa = rec.predict_device(x[i:i + 1], with_scores=True, beam_width=10, top_paths=3)
        assert np.array_equal(la.cpu().numpy()[0], labels[i]) and np.array_equal(lpa.cpu().numpy()[0], logp[i])
    one = rec.predict_device(x, beam_width=10)                    # top_paths = 1: the greedy call's shapes
    assert one.shape == (17, T) and np.array_equal(one.cpu().numpy(), labels[:, 0])
    lab1, lp1 = rec.predict_device(x, with_scores=True, beam_width=10)
    assert lp1.shape == (17,) and np.array_equal(lp1.cpu().numpy(), logp[:, 0])
    texts = rec.recognize_crops(crops, return_scores=True, beam_width=10, top_paths=3)
    assert len(texts) == 17 and all(len(t) == 3 and len(c) == 3 for t, c in texts)
    assert all(c[0] >= c[1] >= c[2] for _, c in texts)


# ------------------------------------------------------------------------------------------ 3. the chained pages
def test_chained_pages_beam(cuda_device):
    from keras_ocr_b200 import distributed as D
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    from keras_ocr_b200.recognition import Recognizer, labels_to_text
    from oracle import synth

    cw, rw = W.synthetic_craft_weights(3, textlike=True), W.synthetic_crnn_weights(2, decisive=True)
    rng = np.random.default_rng(1000)
    pages = np.stack([synth.text_image(rng, 768, 768, 32, return_layout=True)[0] for _ in range(2)])
    det, rec = Detector(weights=cw), Recognizer(weights=rw)
    pipe = Pipeline(detector=det, recognizer=rec, scale=2)
    greedy = pipe.recognize(pages)
    rec.keep_workspace = True
    beam = pipe.recognize(pages, recognition_kwargs={"beam_width": 10})
    n = sum(len(g) for g in beam)
    logits = rec.tap("logits", (n, T, 37), torch.float32).cpu().numpy()
    rec.keep_workspace = False
    assert [[b.view(np.int32).tolist() for _, b in g] for g in beam] == \
        [[b.view(np.int32).tolist() for _, b in g] for g in greedy]
    words = [t for g in beam for t, _ in g]
    taus, lps = tau(logits), BR.log_probs(logits)
    near = 0
    for i, word in enumerate(words):
        paths, _, info = BR.beam_search(lps[i], 10, top_paths=1)
        if min(info["prune_margin"], info["rank_margin"]) > 2 * taus[i]:
            assert word == labels_to_text(_rows(paths, 1), rec.alphabet)[0], i
        else:
            near += 1
    differ = sum(a != b for a, b in zip(words, [t for g in greedy for t, _ in g]))
    print(f"C4 beam W=10: {n} words, {differ} differ from greedy, {near} near-tie words")

    scored = pipe.recognize(pages, recognition_kwargs={"beam_width": 10, "top_paths": 3}, return_scores=True)
    assert [len(g) for g in scored] == [len(g) for g in beam]
    for g, gb in zip(scored, beam):
        for (texts, box, det_score, conf), (text, _) in zip(g, gb):
            assert isinstance(texts, list) and len(texts) == 3 and texts[0] == text
            assert isinstance(conf, list) and len(conf) == 3 and conf[0] >= conf[1] >= conf[2] and 0 <= conf[2]
            assert conf[0] <= 1 and np.float32(det_score) >= np.float32(0.7)

    records = pipe.recognize_records(pages, beam_width=10)
    decoded = D._decode_blocks([records.cpu()], 128, rec.alphabet)
    assert [[t for t, _ in g] for g in decoded] == [[t for t, _ in g] for g in beam]


# ------------------------------------------------------------------------------------------ 4. the C-ABI refuses
def test_abi_rejects_out_of_range(cuda_device, ctx):
    from keras_ocr_b200.recognition import Recognizer
    x = torch.zeros((2, T, 37), dtype=torch.float32, device="cuda")
    labels = torch.empty((2, 128, T), dtype=torch.int32, device="cuda")
    logp = torch.empty((2, 128), dtype=torch.float32, device="cuda")
    lib, h = ctx.lib, ctx.handle
    for b, k, w, p in [(2, 37, 0, 1), (2, 37, 129, 1), (2, 37, 5, 0), (2, 37, 5, 6), (2, 1, 5, 1), (2, 1025, 5, 1),
                       (-1, 37, 5, 1)]:
        assert lib.b2o_ctc_beam_decode(h, x.data_ptr(), b, k, w, p, labels.data_ptr(), logp.data_ptr(), None) == -2
        assert lib.b2o_last_error(h)
    assert lib.b2o_ctc_beam_decode(h, None, 2, 37, 5, 1, labels.data_ptr(), None, None) == -2
    rec = Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True))
    nbytes = rec.ctx.crnn_workspace_bytes(2)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    xin = torch.zeros((2, 200, 31), dtype=torch.float16, device="cuda")
    for w, p in [(0, 1), (129, 1), (5, 6), (5, 0)]:
        assert rec.ctx.lib.b2o_crnn_forward_beam(rec.ctx.handle, xin.data_ptr(), 2, w, p, labels.data_ptr(), None,
                                                 ws.data_ptr(), nbytes, None) == -2
    torch.cuda.synchronize()
