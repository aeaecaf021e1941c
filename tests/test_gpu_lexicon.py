"""Lexicon-constrained decoding on the GPU (``b2o_ctc_lexicon_decode``, ``b2o_crnn_forward_lexicon``) against the fp64
references of tests/lexicon_refs.py.

Bound.  The fp64 reference runs on the same fp32 logits.  Let u = 2^-24, R_t = max_c l - min_c l of step t.  The kernel's
q[t,c] = expf(l_c - m) / s + 1e-7 is the value whose logf the beam decoder takes, so by the derivation of
tests/test_gpu_beam.py it is within delta_t = 10u + 2u R_t + gamma(K + 8) relative of the exact softmax + 1e-7.  Every
state update is (a + b [+ c]) * q: at most two additions and one multiplication of non-negative numbers, 3u relative,
plus q's own delta_t.  Every alignment's product therefore carries at most sum_t (3u + delta_t) relative error (first
order; x 1.01 covers the rest), and so does their sum, all terms being positive.  The power-of-two rescaling is exact,
the last addition costs u, log turns a relative error e into an absolute one of at most 1.01 e, the fp64 log and
E ln 2 add less than 1e-12, and the rounding to float32 half an ulp, at most u |score|.  Hence an entry's fp32 score is
within  tau_L = 1.01 (sum_t (3u + delta_t) + u) + u |score| + 1e-12  of its exact score.  (The subnormal range is
only reached by a state more than 2^134 below the largest.)  Where the reference's gaps between consecutive
scores of the returned entries and the first one left out all exceed 2 tau_L and are not exact ties, the kernel returns
exactly the reference's entries in its order.  Elsewhere (a near-tie) every returned score is still within tau_L of
that entry's exact score and no better entry than the P-th is missed by more than 2 tau_L.  The worst ratio to tau_L is
printed; DESIGN.md section 2 records it.
"""
import os

import numpy as np
import pytest
import torch

from keras_ocr_b200 import _lib, weights as W
from keras_ocr_b200.recognition import Lexicon
from tests import beam_refs as BR
from tests import lexicon_refs as LR
from tests.test_gpu_beam import crafted

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
T = 48


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _gamma(n):
    return n * U / (1 - n * U)


def tau_base(logits):
    """(B,) the entry-independent part of tau_L for (B,48,K) fp32 logits."""
    lg = np.asarray(logits, np.float64)
    k = lg.shape[-1]
    delta = 10 * U + 2 * U * (lg.max(-1) - lg.min(-1)) + _gamma(k + 8)
    return 1.01 * ((3 * U + delta).sum(-1) + U) + 1e-12


def alphabet_for(k):
    return "".join(chr(0x4E00 + i) for i in range(k - 1))


def make_lexicon(rng, k, n):
    """n distinct entries over K-1 labels: mostly short words, doubled letters, long entries (up to 48 labels, across
    the kernel's 8 / 16 / 48 label ranges) and entries that cannot be aligned in 48 steps."""
    hi = 12 if k > 3 else 20
    out, seen = [], set()
    while len(out) < n:
        r = rng.random()
        if r < 0.02:
            e = tuple(int(c) for c in rng.integers(0, k - 1, int(rng.integers(17, 49))))
        elif r < 0.03:
            c = int(rng.integers(0, k - 1))
            e = (c,) * int(rng.integers(24, 30))                  # 24 fits (47 steps); 25 and more cannot be aligned
        else:
            e = tuple(int(c) for c in rng.integers(0, k - 1, int(rng.integers(1, hi + 1))))
            if len(e) >= 2 and rng.random() < 0.3:
                e = e[:1] + e[:1] + e[2:]
        if e not in seen:
            seen.add(e)
            out.append(e)
    return out


def to_lexicon(entries, k):
    a = alphabet_for(k)
    return Lexicon(["".join(a[c] for c in e) for e in entries], alphabet=a)


@pytest.fixture(scope="module")
def ctx(cuda_device):
    return _lib.Context(0)


def decode(ctx, logits, lex, p):
    x = torch.from_numpy(np.ascontiguousarray(logits, np.float32)).cuda()
    b, _, k = x.shape
    off, lab = lex.device_arrays("cuda")
    labels = torch.empty((b, p, T), dtype=torch.int32, device="cuda")
    logp = torch.empty((b, p), dtype=torch.float32, device="cuda")
    nbytes = ctx.lexicon_workspace_bytes(b, len(lex), p)
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device="cuda")
    ctx.ctc_lexicon_decode(x.data_ptr(), b, k, off.data_ptr(), lab.data_ptr(), len(lex), p, labels.data_ptr(),
                           logp.data_ptr(), ws.data_ptr(), nbytes, _stream())
    return labels.cpu().numpy(), logp.cpu().numpy()


def row_entries(labels):
    return [tuple(int(c) for c in row if c >= 0) for row in labels]


def check_against_ref(logits, labels, logp, entries, ref, what):
    """Per crop: the reference's entries in its order where its margins exceed 2 tau_L, the score bound everywhere.
    Returns (worst |logp - ref| / tau_L, number of near-tie crops)."""
    base = tau_base(logits)
    where = {e: i for i, e in enumerate(entries)}
    worst, near = 0.0, 0
    p = labels.shape[1]
    for i in range(len(logits)):
        idx, top, info = LR.top_entries(ref[i], p)
        n = len(idx)
        got = row_entries(labels[i, :n])
        assert np.all(labels[i, n:] == -1) and np.all(logp[i, n:] == -np.inf), (what, i)
        assert np.all(np.diff(logp[i, :n]) <= 0), (what, i)
        j = [where[e] for e in got]                               # KeyError: a returned row is not an entry
        assert len(set(j)) == n, (what, i)
        tau = base[i] + U * np.abs(ref[i, j])
        r = np.abs(logp[i, :n] - ref[i, j]) / tau
        assert np.all(r <= 1.0), (what, i, float(r.max()))
        worst = max(worst, float(r.max()) if n else 0.0)
        tau_max = base[i] + U * (np.abs(top).max() if n else 0.0)
        if info["ties"] == 0 and info["margin"] > 2 * tau_max:
            assert j == list(idx), (what, i, info)
        else:
            near += 1
            if n:
                assert logp[i, n - 1] >= top[-1] - 2 * tau_max, (what, i)
    return worst, near


# ------------------------------------------------------------------------------------------ 1. the decoder alone
@pytest.mark.parametrize("k", [3, 37, 301, 1024])
def test_decoder_vs_fp64(ctx, k):
    rng = np.random.default_rng(k)
    report = []
    for n, crops in ((1, 17), (1000, 17), (1025, 17), (100_000, 6)):
        entries = make_lexicon(rng, k, n)
        lex = to_lexicon(entries, k)
        logits = crafted(k, crops, seed=k * 7 + n)
        ref = np.stack([LR.scores_many(lp, entries) for lp in BR.log_probs(logits)])
        labels, logp = decode(ctx, logits, lex, 128)
        worst, near = check_against_ref(logits, labels, logp, entries, ref, (k, n))
        for p in (1, 5):                                          # fewer paths: the first rows of the same result
            lab_p, lp_p = decode(ctx, logits, lex, p)
            assert np.array_equal(lab_p, labels[:, :p]) and np.array_equal(lp_p.view(np.int32), logp[:, :p].view(np.int32))
        report.append(f"n={n}: worst {worst:.3g} of tau_L, near-tie crops {near}/{crops}")
    print(f"lexicon K={k}: " + "; ".join(report))


def test_bad_labels_and_offsets_score_minus_inf(ctx):
    k = 37
    logits = crafted(k, 6, seed=5)
    offsets = torch.tensor([0, 2, 4, 6, 8, 8, 9], dtype=torch.int32, device="cuda")
    labels = torch.tensor([1, 2, 3, k - 1, 4, -1, 5, 30000, 6], dtype=torch.int16, device="cuda")
    x = torch.from_numpy(logits).cuda()
    out = torch.empty((6, 8, T), dtype=torch.int32, device="cuda")
    logp = torch.empty((6, 8), dtype=torch.float32, device="cuda")
    nbytes = ctx.lexicon_workspace_bytes(6, 6, 8)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    ctx.ctc_lexicon_decode(x.data_ptr(), 6, k, offsets.data_ptr(), labels.data_ptr(), 6, 8, out.data_ptr(),
                           logp.data_ptr(), ws.data_ptr(), nbytes, _stream())
    out, logp = out.cpu().numpy(), logp.cpu().numpy()
    for i in range(6):                                            # blank, -1, out of range and empty entries: -inf
        assert sorted(row_entries(out[i, :2])) == [(1, 2), (6,)]
        assert np.all(out[i, 2:] == -1) and np.all(logp[i, 2:] == -np.inf) and np.all(np.isfinite(logp[i, :2]))


def test_exhaustive_k3(ctx):
    """All label sequences of length 1..6 over K = 3: the top entry is the best of them by exact enumeration."""
    import itertools
    entries = [e for n in range(1, 7) for e in itertools.product(range(2), repeat=n)]
    lex = to_lexicon(entries, 3)
    logits = crafted(3, 24, seed=3)
    ref = np.stack([LR.scores(lp, entries) for lp in BR.log_probs(logits)])
    labels, logp = decode(ctx, logits, lex, 1)
    worst, near = check_against_ref(logits, labels, logp, entries, ref, "exhaustive")
    clear = 0
    for i in range(len(logits)):
        idx, _, info = LR.top_entries(ref[i], 1)
        if info["ties"] == 0 and info["margin"] > 2 * (tau_base(logits[i:i + 1])[0] + U * abs(ref[i, idx[0]])):
            assert row_entries(labels[i])[0] == entries[int(np.argmax(ref[i]))]
            clear += 1
    print(f"exhaustive K=3: {clear}/24 crops clear, worst {worst:.3g} of tau_L, near-tie crops {near}")


# ------------------------------------------------------------------------------------------ 2. invariance
def test_batch_run_and_order_invariance(ctx):
    k = 37
    rng = np.random.default_rng(11)
    entries = make_lexicon(rng, k, 3000)
    lex = to_lexicon(entries, k)
    logits = crafted(k, 17, seed=17)
    labels, logp = decode(ctx, logits, lex, 5)
    for b in (1, 7):
        lab_b, lp_b = decode(ctx, logits[:b], lex, 5)
        assert np.array_equal(lab_b, labels[:b]) and np.array_equal(lp_b.view(np.int32), logp[:b].view(np.int32))
    for i in (3, 16):
        lab_1, lp_1 = decode(ctx, logits[i:i + 1], lex, 5)
        assert np.array_equal(lab_1[0], labels[i]) and np.array_equal(lp_1[0].view(np.int32), logp[i].view(np.int32))
    lab2, lp2 = decode(ctx, logits, lex, 5)
    assert np.array_equal(lab2, labels) and np.array_equal(lp2.view(np.int32), logp.view(np.int32))
    perm = rng.permutation(len(entries))
    lab_s, lp_s = decode(ctx, logits, to_lexicon([entries[i] for i in perm], k), 5)
    assert np.array_equal(lp_s.view(np.int32), logp.view(np.int32))
    for i in range(17):                                           # the same entries, up to the order of exact ties
        a = dict(zip(row_entries(labels[i]), logp[i].view(np.int32)))
        b = dict(zip(row_entries(lab_s[i]), lp_s[i].view(np.int32)))
        last = logp[i, -1].view(np.int32)
        assert {e: v for e, v in a.items() if v != last} == {e: v for e, v in b.items() if v != last}
    extra = make_lexicon(np.random.default_rng(12), k, 20000)
    bigger = entries + [e for e in extra if e not in set(entries)]
    lab_x, lp_x = decode(ctx, logits, to_lexicon(bigger, k), 5)
    for i in range(17):                                           # an entry's score does not change in a larger lexicon
        got = dict(zip(row_entries(lab_x[i]), lp_x[i].view(np.int32)))
        for e, v in zip(row_entries(labels[i]), logp[i].view(np.int32)):
            if e in got:
                assert got[e] == v


# ------------------------------------------------------------------------------------------ 3. through the CRNN
def _input(rec, crops):
    t = torch.from_numpy(np.ascontiguousarray(crops)).to(rec.device)
    x = torch.empty((len(crops), 200, 31), dtype=torch.float16, device=rec.device)
    rec.ctx.crops_to_input(t.data_ptr(), len(crops), x.data_ptr(), _stream())
    return x


def _c3_lexicon(g, alphabet, n_distractors):
    from keras_ocr_b200.recognition import labels_to_text
    from oracle import synth
    words = [w for w in dict.fromkeys(labels_to_text(g["labels"].astype(np.int32), alphabet)) if w]
    rng = np.random.default_rng(2024)
    seen, target = set(words), len(words) + n_distractors
    while len(words) < target:
        w = synth.random_word(rng)
        if w not in seen:
            seen.add(w)
            words.append(w)
    return words


def test_crnn_forward_lexicon(cuda_device, ctx, golden_dir):
    from keras_ocr_b200.recognition import Recognizer, labels_to_text
    g = np.load(os.path.join(golden_dir, "c3_crops.npz"))
    rec = Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True))
    rec.keep_workspace = True
    words = _c3_lexicon(g, rec.alphabet, 10_000)
    lex = Lexicon(words, rec.alphabet)
    x = _input(rec, g["crops"])
    labels, logp = rec.predict_device(x, with_scores=True, lexicon=lex, top_paths=3)
    assert labels.shape == (256, 3, T) and logp.shape == (256, 3)
    labels, logp = labels.cpu().numpy(), logp.cpu().numpy()
    logits = rec.tap("logits", (256, T, 37), torch.float32).cpu().numpy()
    lab_d, lp_d = decode(ctx, logits, lex, 3)                     # the decoder alone on the CRNN's own logits
    assert np.array_equal(lab_d, labels) and np.array_equal(lp_d.view(np.int32), logp.view(np.int32))
    entries = [tuple(rec.alphabet.index(c) for c in w) for w in words]
    ref = np.stack([LR.scores_many(lp, entries) for lp in BR.log_probs(logits)])
    worst, near = check_against_ref(logits, labels, logp, entries, ref, "c3")
    listed = rec.predict_device(x, with_scores=True, lexicon=words, top_paths=3)   # a plain list decodes alike
    assert np.array_equal(listed[0].cpu().numpy(), labels) and np.array_equal(listed[1].cpu().numpy(), logp)
    one = rec.predict_device(x, lexicon=lex)                       # top_paths = 1: the greedy call's shapes
    assert one.shape == (256, T) and np.array_equal(one.cpu().numpy(), labels[:, 0])
    greedy = labels_to_text(rec.predict_device(x).cpu().numpy(), rec.alphabet)
    truth = labels_to_text(g["labels"].astype(np.int32), rec.alphabet)
    top = [t[0] for t in rec.recognize_crops(g["crops"], lexicon=lex, top_paths=3)]
    print(f"C3 lexicon ({len(words)} entries): worst {worst:.3g} of tau_L, near-tie crops {near}/256; "
          f"top entry = oracle reading on {sum(a == b for a, b in zip(top, truth))}/256, "
          f"greedy = oracle reading on {sum(a == b for a, b in zip(greedy, truth))}/256")


# ------------------------------------------------------------------------------------------ 4. the chained pages
def test_chained_pages_lexicon(cuda_device, ctx):
    from keras_ocr_b200 import distributed as D
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    from keras_ocr_b200.recognition import Recognizer, confidences
    from oracle import synth

    cw, rw = W.synthetic_craft_weights(3, textlike=True), W.synthetic_crnn_weights(2, decisive=True)
    rng = np.random.default_rng(1000)
    laid = [synth.text_image(rng, 768, 768, 32, return_layout=True) for _ in range(2)]
    pages = np.stack([p[0] for p in laid])
    words = list(dict.fromkeys(w for p in laid for w in p[1]))
    drng = np.random.default_rng(7)
    while len(words) < 1000:
        w = synth.random_word(drng)
        if w not in words:
            words.append(w)
    det, rec = Detector(weights=cw), Recognizer(weights=rw)
    lex = Lexicon(words, rec.alphabet)
    pipe = Pipeline(detector=det, recognizer=rec, scale=2)
    greedy = pipe.recognize(pages)
    rec.keep_workspace = True
    got = pipe.recognize(pages, recognition_kwargs={"lexicon": lex})
    n = sum(len(g) for g in got)
    logits = rec.tap("logits", (n, T, 37), torch.float32).cpu().numpy()
    rec.keep_workspace = False
    assert [[b.view(np.int32).tolist() for _, b in g] for g in got] == \
        [[b.view(np.int32).tolist() for _, b in g] for g in greedy]
    texts = [t for g in got for t, _ in g]
    assert all(t in set(words) for t in texts)
    _, lp_d = decode(ctx, logits, lex, 1)
    scored = pipe.recognize(pages, recognition_kwargs={"lexicon": lex}, return_scores=True)
    assert [t for g in scored for t, *_ in g] == texts
    conf = np.array([c for g in scored for *_, c in g], np.float32)
    assert np.array_equal(conf, confidences(lp_d[:, 0]))
    listed = pipe.recognize(pages, recognition_kwargs={"lexicon": words, "top_paths": 2}, return_scores=True)
    assert [ts[0] for g in listed for ts, *_ in g] == texts

    records = pipe.recognize_records(pages, lexicon=lex)
    decoded = D._decode_blocks([records.cpu()], 128, rec.alphabet)
    assert [[t for t, _ in g] for g in decoded] == [[t for t, _ in g] for g in got]
    records = pipe.recognize_records(pages, lexicon=lex, scores=True)
    decoded = D._decode_blocks([records.cpu()], 128, rec.alphabet, scores=True)
    assert [t for g in decoded for t, *_ in g] == texts
    assert np.array_equal(np.array([c for g in decoded for *_, c in g], np.float32), conf)
    differ = sum(a != b for a, b in zip(texts, [t for g in greedy for t, _ in g]))
    print(f"C4 lexicon ({len(words)} entries): {n} words, {differ} differ from greedy")


# ------------------------------------------------------------------------------------------ 5. the C-ABI refuses
def test_abi_rejects_out_of_range(cuda_device, ctx):
    from keras_ocr_b200.recognition import Recognizer
    x = torch.zeros((2, T, 37), dtype=torch.float32, device="cuda")
    off = torch.tensor([0, 1, 2], dtype=torch.int32, device="cuda")
    lab = torch.tensor([0, 1], dtype=torch.int16, device="cuda")
    out = torch.empty((2, 128, T), dtype=torch.int32, device="cuda")
    logp = torch.empty((2, 128), dtype=torch.float32, device="cuda")
    nbytes = ctx.lexicon_workspace_bytes(2, 2, 128)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    lib, h = ctx.lib, ctx.handle
    for b, k, n, p in [(2, 37, 0, 1), (2, 37, (1 << 20) + 1, 1), (2, 37, 2, 0), (2, 37, 2, 129), (2, 1, 2, 1),
                       (2, 1025, 2, 1), (-1, 37, 2, 1)]:
        assert lib.b2o_ctc_lexicon_decode(h, x.data_ptr(), b, k, off.data_ptr(), lab.data_ptr(), n, p, out.data_ptr(),
                                          logp.data_ptr(), ws.data_ptr(), nbytes, None) == -2
        assert lib.b2o_last_error(h)
    assert lib.b2o_ctc_lexicon_decode(h, x.data_ptr(), 2, 37, None, lab.data_ptr(), 2, 1, out.data_ptr(), None,
                                      ws.data_ptr(), nbytes, None) == -2
    assert lib.b2o_ctc_lexicon_decode(h, x.data_ptr(), 2, 37, off.data_ptr(), lab.data_ptr(), 2, 1, out.data_ptr(), None,
                                      ws.data_ptr(), nbytes - 1, None) == -4
    rec = Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True))
    cb = rec.ctx.crnn_workspace_bytes(2)
    ws2 = torch.empty(cb + 256 + nbytes, dtype=torch.uint8, device="cuda")
    xin = torch.zeros((2, 200, 31), dtype=torch.float16, device="cuda")
    for n, p, size, code in [(0, 1, ws2.numel(), -2), (2, 129, ws2.numel(), -2), (2, 1, cb, -4)]:
        assert rec.ctx.lib.b2o_crnn_forward_lexicon(rec.ctx.handle, xin.data_ptr(), 2, off.data_ptr(), lab.data_ptr(),
                                                    n, p, out.data_ptr(), None, ws2.data_ptr(), size, None) == code
    torch.cuda.synchronize()
