"""GPU: character scores -- ``b2o_ctc_char_scores`` alone against tests/char_score_refs.py, its memory contract and
rejections, the product path through the CRNN workspace, the recognizer and pipeline flags, and what the scores say
about misread characters on degraded pages.

Bound.  As in tests/test_gpu_char_boxes.py, the kernel's lp[t,c] is within d_t of the exact value (u = 2^-24, R_t the
step's logit range): d_t = 1.01 (10u + 2u R_t + gamma(K + 8)) + 2u max_c |lp[t,c]|.  Every value the kernel forms --
alpha, beta, the gamma sweep and its running sum -- is a log-sum over partial alignments, and logsumexp passes input
errors on as their weighted mean (weights: the terms' shares of the sum; to first order in u).  So an F's error is a
weighted mean over the alignments pi of the edited reading, weight w_pi = exp(sigma_pi - F), of the errors made along
pi's route.  Along a route every step lies in exactly one of alpha, the gamma sweep or beta, and the lp errors add up
to at most sum_t d_t.  Each step costs at most two fp32 additions of log values plus one logsumexp (exp, a sum of <= 3
terms, log of a value in [1, 3]: at most 6u); the running sum over t adds 48 logsumexps, the A and B terms 4 more --
fewer than 200 roundings in all.  An addition rounds by u |result|, and every value on pi's route is a log-sum of
partial alignments that includes pi's own prefix (or suffix), so |result| <= |sigma_pi| (lp <= 1e-7, negligible).
The weighted mean of |sigma_pi| is |F| + H(w) <= |F| + 48 log 3 < |F| + 53 (Gibbs: at most 3 moves per step).  So
    dF = sum_t d_t + 200 u (|F| + 59)
bounds the error of every F, and of logp = F(y).  A posterior pi_e = exp(F_e - L) then moves by a factor within
exp(+-(dF_e + dL)), dL = sum_e' pi_e' dF_e' (L's error, the weighted mean again), and its fp32 evaluation (exp of
F_e - m, a K-term sum, a division) adds a relative gamma(K + 9), and at most 2^-120 absolutely where exp underflows:
    tau_e = pi_e (expm1(dF_e + dL) + gamma(K + 9)) + 2^-120.
The confidence is within tau of the reference's; the posteriors listed at a position sum to at most 1 + sum_e tau_e,
and to 1 within it when every edit is listed.  Where each consecutive gap of the reference's ranking down to place
A+1 exceeds twice the larger tau of its pair (or both values are impossible edits, F = -inf in any precision), the
kernel's alternative labels are the reference's.
"""
import os

import numpy as np
import pytest
import torch

import bench
from keras_ocr_b200 import _lib, weights as W
from keras_ocr_b200.detection import Detector
from keras_ocr_b200.pipeline import Pipeline
from keras_ocr_b200.recognition import CharLM, Lexicon, Recognizer, char_scores_host
from tests import beam_refs as BR
from tests import char_score_refs as CR
from tests.test_gpu_beam import crafted
from tests.test_gpu_char_boxes import readings

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
T = 48
A_MAX = _lib.MAX_CHAR_ALTERNATIVES
ERR_ARG, ERR_STATE = -2, -5


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def gamma(n):
    return n * U / (1 - n * U)


def lp_error(logits):
    """sum_t d_t per crop, as the module docstring gives it."""
    lg = np.asarray(logits, np.float64)
    lp = BR.log_probs(lg)
    k = lg.shape[-1]
    d = 1.01 * (10 * U + 2 * U * (lg.max(-1) - lg.min(-1)) + gamma(k + 8)) + 2 * U * np.abs(lp).max(-1)
    return d.sum(-1)


def bounds(f, sum_d):
    """(dF (n, K), pi (n, K), tau (n, K)) of one reading's fp64 edit scores F, as the module docstring derives them."""
    k = f.shape[1]
    df = sum_d + 200 * U * (np.where(np.isfinite(f), np.abs(f), 0.0) + 59)
    with np.errstate(invalid="ignore"):
        m = f.max(1, keepdims=True)
        pi = np.where(np.isfinite(m), np.exp(f - m), 0.0)
    pi = pi / np.maximum(pi.sum(1, keepdims=True), 1e-300)
    dl = (pi * df).sum(1, keepdims=True)
    return df, pi, pi * (np.expm1(df + dl) + gamma(k + 9)) + 2.0 ** -120


@pytest.fixture(scope="module")
def ctx(cuda_device):
    c = _lib.Context(0)
    yield c
    c.close()


def char_scores(ctx, logits, labels, a, guard=0):
    """The kernel on host arrays; every output pre-filled with garbage, ``guard`` extra elements after each."""
    b, p = labels.shape[:2]
    conf = torch.full((b * p * T + guard,), 7.5, dtype=torch.float32, device="cuda")
    al = torch.full((b * p * T * a + guard,), 77, dtype=torch.int32, device="cuda")
    ap = torch.full((b * p * T * a + guard,), 7.5, dtype=torch.float32, device="cuda")
    logp = torch.full((b * p + guard,), 7.5, dtype=torch.float32, device="cuda")
    x, lab = _dev(logits.astype(np.float32)), _dev(labels)
    ctx.ctc_char_scores(x.data_ptr(), b, logits.shape[2], lab.data_ptr(), p, a, conf.data_ptr(),
                        al.data_ptr() if a else None, ap.data_ptr() if a else None, logp.data_ptr(), _stream())
    out = [t.cpu().numpy() for t in (conf, al, ap, logp)]
    if guard:
        assert (out[0][-guard:] == 7.5).all() and (out[1][-guard:] == 77).all() and (out[2][-guard:] == 7.5).all()
        assert (out[3][-guard:] == 7.5).all()
        out = [o[:-guard] for o in out]
    return (out[0].reshape(b, p, T), out[1].reshape(b, p, T, a), out[2].reshape(b, p, T, a), out[3].reshape(b, p))


def check_scores(logits, labels, conf, al, ap, logp):
    """Against the fp64 recipe (tests/test_char_score_refs.py checks it against the definition).  Returns (worst error
    in units of tau, positions whose labels were compared, positions within a near-tie)."""
    sum_d = lp_error(logits)
    lps = BR.log_probs(logits)
    k, a = logits.shape[2], al.shape[-1]
    worst, same, near = 0.0, 0, 0
    for i in range(len(logits)):
        for j in range(labels.shape[1]):
            row = labels[i, j]
            n = int(np.argmax(row < 0)) if (row < 0).any() else T
            y = [int(c) for c in row[:n]]
            assert np.isnan(conf[i, j, n:]).all() and (al[i, j, n:] == -1).all() and np.isnan(ap[i, j, n:]).all()
            if any(c > k - 2 for c in y):                         # a label outside [0, K-2]: the L = -inf rule
                assert logp[i, j] == -np.inf and (conf[i, j, :n] == 0).all()
                assert (al[i, j, :n] == -1).all() and (ap[i, j, :n] == 0).all()
                continue
            f, ref_logp = CR.recipe(lps[i], y)
            if np.isfinite(ref_logp):
                tol = sum_d[i] + 200 * U * (abs(ref_logp) + 59)
                assert abs(float(logp[i, j]) - ref_logp) <= tol, (i, j, logp[i, j], ref_logp)
            else:
                assert logp[i, j] == -np.inf
            if not n:
                continue
            rc, rl, rp, _ = CR.scores(f, y, a)
            _, pi, tau = bounds(f, sum_d[i])
            for q in range(n):
                if not np.isfinite(f[q]).any():
                    assert conf[i, j, q] == 0 and (al[i, j, q] == -1).all() and (ap[i, j, q] == 0).all()
                    continue
                err = abs(float(conf[i, j, q]) - rc[q])
                assert err <= tau[q, y[q]], (i, j, q, err, tau[q, y[q]])
                worst = max(worst, err / tau[q, y[q]])
                if a >= k:                                        # every edit is listed: the posteriors sum to 1
                    assert abs(float(ap[i, j, q, :k].astype(np.float64).sum()) - 1.0) <= tau[q].sum(), (i, j, q)
                    assert (al[i, j, q, k:] == -1).all() and (ap[i, j, q, k:] == 0).all()
                elif a:
                    assert float(ap[i, j, q].astype(np.float64).sum()) <= 1.0 + tau[q].sum()
                if not a:
                    continue
                order = np.lexsort((np.arange(k), -pi[q]))[:min(a + 1, k)]
                gaps = pi[q, order[:-1]] - pi[q, order[1:]]
                need = 2 * np.maximum(tau[q, order[:-1]], tau[q, order[1:]])
                impossible = np.isneginf(f[q, order[:-1]]) & np.isneginf(f[q, order[1:]])
                if ((gaps > need) | impossible).all():
                    assert np.array_equal(al[i, j, q], rl[q]), (i, j, q, al[i, j, q], rl[q])
                    ok = rl[q] >= 0
                    assert (np.abs(ap[i, j, q][ok] - rp[q][ok]) <= tau[q, rl[q][ok]]).all(), (i, j, q)
                    same += 1
                else:
                    near += 1
    return worst, same, near


# ------------------------------------------------------------------------------------------ 1. the kernel alone
@pytest.mark.parametrize("k", [3, 37, 127, 1024])
def test_kernel_vs_fp64(ctx, k):
    rng = np.random.default_rng(k)
    report = []
    for p in (1, 8):
        logits = crafted(k, 12 if k < 1024 else 6, seed=k + p)
        labels = readings(logits, p, rng)
        full = char_scores(ctx, logits, labels, A_MAX)
        worst, same, near = check_scores(logits, labels, *full)
        report.append(f"P={p}: worst {worst:.3g} of tau, {same} rankings identical, {near} near-tie positions")
        for a in (0, 1):                                          # fewer alternatives: the same scores, a prefix
            conf, al, ap, logp = char_scores(ctx, logits, labels, a)
            assert np.array_equal(conf.view(np.int32), full[0].view(np.int32))
            assert np.array_equal(logp.view(np.int32), full[3].view(np.int32))
            assert np.array_equal(al, full[1][..., :a]) and np.array_equal(ap.view(np.int32), full[2][..., :a].view(np.int32))
        for b in (1, 5):                                          # a crop scores alike alone and in any batch
            part = char_scores(ctx, logits[:b], labels[:b], A_MAX)
            for x, y in zip(part, full):
                assert np.array_equal(x.view(np.int32), y[:b].view(np.int32))
    print(f"K={k}: " + "; ".join(report))


def test_memory_contract(ctx):
    """Guard elements after every output stay untouched; every slot, padded ones included, is written over garbage;
    a second run gives the same bits."""
    rng = np.random.default_rng(5)
    logits = crafted(37, 7, seed=5)
    labels = readings(logits, 3, rng)
    a = char_scores(ctx, logits, labels, 4, guard=64)
    b = char_scores(ctx, logits, labels, 4, guard=64)
    for x, y in zip(a, b):
        assert np.array_equal(x.view(np.int32), y.view(np.int32))
    conf, al, ap, logp = a
    assert not (conf == 7.5).any() and not (al == 77).any() and not (ap == 7.5).any() and not (logp == 7.5).any()


def test_abi_rejects_out_of_range(ctx):
    L, s = ctx.lib, _stream()
    x = torch.zeros((2, T, 1024), dtype=torch.float32, device="cuda")
    lab = torch.full((2, 129, T), -1, dtype=torch.int32, device="cuda")
    out = torch.full((2 * 129 * T * 9,), 7.5, dtype=torch.float32, device="cuda")
    outl = torch.full((2 * 129 * T * 9,), 77, dtype=torch.int32, device="cuda")
    n0 = ctx.launch_count()

    def call(k=37, p=1, a=0, conf=True, alt=True, b=2):
        return L.b2o_ctc_char_scores(ctx.handle, x.data_ptr(), b, k, lab.data_ptr(), p, a,
                                     out.data_ptr() if conf else None, outl.data_ptr() if alt else None,
                                     out.data_ptr() if alt else None, None, s)
    for kw in ({"k": 1}, {"k": 1025}, {"p": 0}, {"p": 129}, {"a": -1}, {"a": 9}, {"conf": False},
               {"a": 2, "alt": False}, {"b": -1}):
        assert call(**kw) == ERR_ARG, kw
    assert ctx.launch_count() == n0 and (out == 7.5).all() and (outl == 77).all()
    assert call(k=2, p=128, a=8) == 0 and call(k=1024, a=0, alt=False) == 0 and call(b=0) == 0
    torch.cuda.synchronize()


def test_state_rule(cuda_device, golden_dir):
    """b2o_crnn_char_scores needs the logits of the context's last forward: after b2o_crnn_features it refuses."""
    rec = Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True))
    g = np.load(os.path.join(golden_dir, "c3_crops.npz"))
    x = _input(rec, g["crops"][:8])
    b = len(x)
    nbytes = rec.ctx.crnn_workspace_bytes(b)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    labels = torch.empty((b, T), dtype=torch.int32, device="cuda")
    conf = torch.full((b, T), 7.5, dtype=torch.float32, device="cuda")
    L, s = rec.ctx.lib, _stream()
    rec.ctx.crnn_forward_logits(x.data_ptr(), b, labels.data_ptr(), None, ws.data_ptr(), nbytes, s)
    assert L.b2o_crnn_char_scores(rec.ctx.handle, b, labels.data_ptr(), 1, 0, conf.data_ptr(), None, None, None,
                                  ws.data_ptr(), nbytes, s) == 0
    first = conf.clone()
    feats = torch.empty((b, T, 256), dtype=torch.float16, device="cuda")
    rec.ctx.crnn_features(x.data_ptr(), b, feats.data_ptr(), ws.data_ptr(), nbytes, s)
    conf.fill_(7.5)
    assert L.b2o_crnn_char_scores(rec.ctx.handle, b, labels.data_ptr(), 1, 0, conf.data_ptr(), None, None, None,
                                  ws.data_ptr(), nbytes, s) == ERR_STATE
    assert L.b2o_crnn_char_scores(rec.ctx.handle, b, labels.data_ptr(), 1, 9, conf.data_ptr(), None, None, None,
                                  ws.data_ptr(), nbytes, s) == ERR_ARG
    assert (conf == 7.5).all() and not torch.equal(first, conf)


# ------------------------------------------------------------------------------------------ 2. the product path
def _input(rec, crops):
    t = torch.from_numpy(np.ascontiguousarray(crops)).to(rec.device)
    x = torch.empty((len(crops), 200, 31), dtype=torch.float16, device=rec.device)
    rec.ctx.crops_to_input(t.data_ptr(), len(crops), x.data_ptr(), _stream())
    return x


def _decoders(alphabet):
    lm = CharLM.fit(["hello", "world", "text", "abc"] * 50 + [f"w{i}" for i in range(50)], alphabet, order=4)
    return {"greedy": {}, "beam": {"beam_width": 10}, "top_paths": {"beam_width": 10, "top_paths": 3},
            "lexicon": {"lexicon": Lexicon(["hello", "world", "text", "abc", "zz"] + [f"w{i}" for i in range(50)])},
            "lm": {"beam_width": 8, "language_model": lm}, "pattern": {"beam_width": 8, "pattern": "[a-z]+[0-9]*"}}


def _bits(x):
    """A word element as comparable bits: strings as they are, float32 arrays and floats by their bits."""
    if isinstance(x, (list, tuple)):
        return [_bits(v) for v in x]
    if isinstance(x, np.ndarray):
        return (x.dtype.str, x.shape, np.ascontiguousarray(x).view(np.uint8).tobytes())
    if isinstance(x, (float, np.floating)):
        return np.float32(x).view(np.int32).item()
    return x


@pytest.mark.parametrize("decoder", ["greedy", "beam", "top_paths", "lexicon", "lm", "pattern"])
def test_product_path(cuda_device, golden_dir, decoder):
    g = np.load(os.path.join(golden_dir, "c3_crops.npz"))
    crops = g["crops"][:48]
    rec = Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True))
    rec.keep_workspace = True
    kw = _decoders(rec.alphabet)[decoder]
    p = kw.get("top_paths", 1)
    x = _input(rec, crops)
    labels, logp, conf, al, ap = rec.predict_device(x, with_scores=True, char_scores=A_MAX, **kw)
    logits = rec.tap("logits", (len(x), T, 37), torch.float32)
    plain = rec.predict_device(x, with_scores=True, **kw)      # the decoder's outputs do not change
    assert torch.equal(plain[0], labels) and torch.equal(plain[1].view(torch.int32), logp.view(torch.int32))
    ref = char_scores(rec.ctx, logits.cpu().numpy(), labels.cpu().numpy().reshape(len(x), p, T), A_MAX)
    for got, want in zip((conf, al, ap), ref[:3]):
        assert np.array_equal(got.cpu().numpy().reshape(want.shape).view(np.int32), want.view(np.int32))
    for a in (0, 3):
        words = rec.recognize_crops(crops, return_scores=True, return_char_boxes=True, return_char_scores=True,
                                    char_alternatives=a, **kw)
        without = rec.recognize_crops(crops, return_scores=True, return_char_boxes=True, **kw)
        assert [_bits(w[:-1]) for w in words] == [_bits(w) for w in without]
        texts = [w[0] for w in words]
        want = char_scores_host(conf.cpu().numpy(), texts, rec.alphabet,
                                *((al[..., :a].cpu().numpy(), ap[..., :a].cpu().numpy()) if a else ()))
        assert [_bits(w[-1]) for w in words] == [_bits(q) for q in want]
    # recognize_from_boxes: the crops of a page, read from their boxes
    page = np.full((31 * 8, 200 * 6, 3), 255, np.uint8)
    boxes = []
    for i in range(48):
        r, c = divmod(i, 6)
        page[31 * r:31 * r + 31, 200 * c:200 * c + 200] = crops[i][..., None]
        boxes.append(np.array([[200 * c, 31 * r], [200 * c + 200, 31 * r], [200 * c + 200, 31 * r + 31],
                               [200 * c, 31 * r + 31]], np.float32))
    got = rec.recognize_from_boxes([page], [boxes], return_scores=True, return_char_scores=True, char_alternatives=2,
                                   **kw)[0]
    without = rec.recognize_from_boxes([page], [boxes], return_scores=True, **kw)[0]
    assert [_bits(w[:-1]) for w in got] == [_bits(w) for w in without]
    assert all(len(q[0] if p == 1 else q[0][0]) == len(w[0] if p == 1 else w[0][0]) for w in got for q in [w[-1]])


@pytest.fixture(scope="module")
def pipe(cuda_device):
    det = Detector(weights=W.synthetic_craft_weights(3, textlike=True), device=0)
    rec = Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True), device=0)
    return Pipeline(detector=det, recognizer=rec, scale=bench.SCALE, max_size=2048)


@pytest.fixture(scope="module")
def pages():
    return bench.make_pages(0)[:8]                          # two sub-batches of min_chunk pages under inflight=2


CALLS = {
    "plain": ({}, {}),
    "scores_cells": ({"return_scores": True, "return_char_boxes": True}, {}),
    "rotations": ({"return_scores": True}, {"rotations": (0, 2), "beam_width": 4}),
    "page_vote_top_paths": ({}, {"rotations": (0, 2), "rotation_vote": "page", "beam_width": 6, "top_paths": 2}),
    "polygons": ({"return_polygons": True, "return_scores": True}, {}),
    "lines": ({"return_lines": True}, {}),
    "blocks": ({"return_blocks": True, "return_char_boxes": True}, {}),
}


@pytest.mark.parametrize("name", sorted(CALLS))
def test_pipeline_flag_changes_nothing_else(pipe, pages, name):
    kwargs, rkw = CALLS[name]
    pipe.inflight = 2
    try:
        base = pipe.recognize(pages, recognition_kwargs=dict(rkw), **kwargs)
        got = pipe.recognize(pages, recognition_kwargs=dict(rkw), return_char_scores=True, char_alternatives=3,
                             **kwargs)
    finally:
        pipe.inflight = 1

    def words(res):
        if kwargs.get("return_blocks"):
            return [w for g in res for blk in g for ln in blk[2] for w in ln[2]]
        if kwargs.get("return_lines"):
            return [w for g in res for ln in g for w in ln[2]]
        return [w for g in res for w in g]
    if kwargs.get("return_lines") or kwargs.get("return_blocks"):
        strip = lambda r: [[(t, _bits(b)) for t, b, *_ in g] for g in r]     # noqa: E731
        assert strip(base) == strip(got)
    wb, wg = words(base), words(got)
    assert len(wb) == len(wg) > 0
    assert [_bits(w) for w in wb] == [_bits(w[:-1]) for w in wg]
    p = rkw.get("top_paths", 1)
    for w in wg:
        texts = [w[0]] if p == 1 else w[0]
        sc = [w[-1]] if p == 1 else w[-1]
        for t, (c, alts) in zip(texts, sc):
            assert c.shape == (len(t),) and c.dtype == np.float32 and len(alts) == len(t)
            assert all(len(a) == 3 for a in alts)


def test_refused_combinations_raise_before_any_launch(pipe, pages):
    rec = pipe.recognizer
    n0 = pipe.detector.ctx.launch_count() + rec.ctx.launch_count()
    box = [[np.array([[0, 0], [50, 0], [50, 20], [0, 20]], np.float32)]]
    for kw in ({"return_char_scores": True, "char_alternatives": 9}, {"char_alternatives": 2},
               {"return_char_scores": True, "max_windows": 2}):
        rkw = {k: v for k, v in kw.items() if k == "max_windows"}
        flags = {k: v for k, v in kw.items() if k != "max_windows"}
        with pytest.raises(ValueError):
            pipe.recognize(pages[:1], recognition_kwargs=rkw, **flags)
        with pytest.raises(ValueError):
            rec.recognize_from_boxes(list(pages[:1]), box, **kw)
        if not rkw:
            with pytest.raises(ValueError):
                rec.recognize_crops(np.zeros((1, 31, 200), np.uint8), **kw)

    class Other:
        def detect(self, images, **kwargs):
            return [[] for _ in images]

    with pytest.raises(NotImplementedError):
        Pipeline(detector=Other(), recognizer=rec).recognize(pages[:1], return_char_scores=True)
    assert pipe.detector.ctx.launch_count() + rec.ctx.launch_count() == n0


# ------------------------------------------------------------------------------------------ 3. what the scores say
def true_length_chars(result, items, a_index=-1):
    """Per character of every word read at its true length: (confidence, read == true, true label's rank among the
    alternatives or None).  A word matches the one item whose centre its box holds, as window_refs.exact_reads."""
    import cv2
    out = []
    for word in result:
        box = np.asarray(word[1], np.float32).reshape(-1, 1, 2)
        inside = [t for t, c in items if cv2.pointPolygonTest(box, (float(c[0]), float(c[1])), False) >= 0]
        if len(inside) != 1 or len(inside[0]) != len(word[0]):
            continue
        conf, alts = word[a_index]
        for j, (r, t) in enumerate(zip(word[0], inside[0])):
            chars = [ch for ch, _ in alts[j]]
            out.append((float(conf[j]), r == t, chars.index(t) if t in chars else None))
    return out


def test_scores_flag_misread_characters(pipe):
    """On the degraded pseudo-language pages of tests/test_gpu_lm.py misread characters have a lower mean confidence
    than correctly read ones, and the true character is among the top 4 alternatives of most misread characters."""
    from tests.test_gpu_lm import SEVERITY, TEST_SEEDS, pseudo_pages
    pages, items = pseudo_pages(TEST_SEEDS, SEVERITY)
    res = pipe.recognize(pages, return_char_scores=True, char_alternatives=4)
    chars = [c for g, it in zip(res, items) for c in true_length_chars(g, it)]
    right = [c for c, ok, _ in chars if ok]
    wrong = [(c, rank) for c, ok, rank in chars if not ok]
    top4 = sum(rank is not None for _, rank in wrong)
    print(f"degraded pages: {len(chars)} characters of true-length readings, {len(wrong)} misread; mean confidence "
          f"right {np.mean(right):.4f}, misread {np.mean([c for c, _ in wrong]):.4f}; true character in the top 4 of "
          f"{top4}/{len(wrong)} misread")
    assert len(wrong) >= 10 and len(right) >= 100
    assert np.mean([c for c, _ in wrong]) < np.mean(right)
    assert top4 > len(wrong) / 2
