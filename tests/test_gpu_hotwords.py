"""CTC beam search with hotwords on the GPU (``b2o_ctc_beam_hotword_decode``, ``b2o_crnn_forward_beam_hotword``)
against tests/hotword_refs.py, and the ``hotwords=`` option on every read path.

Bound.  The reference ranks by F = A + G + H with A in fp64 and G, H, l(</s> | h) computed in float32 exactly as the
kernel computes them; the kernel's A is within tau (tests/test_gpu_beam.py) of the exact one and F, F_end add at most
two float32 roundings each, so every kernel F_end is within tau_F = tau + 4u (|F_end| + 1) of the reference's.  Where
the reference's margins exceed 2 tau_F the kernel returns the same readings, |A - ref| <= tau and |F_end - ref| <=
tau_F; elsewhere (a near-tie, counted and bounded) every returned reading's A is at most its exact forward
log-probability + tau.
"""
import os

import numpy as np
import pytest
import torch

from keras_ocr_b200 import _lib, weights as W
from keras_ocr_b200.recognition import CharLM, Hotwords, Recognizer
from tests import beam_refs as BR
from tests import hotword_refs as HR
from tests.test_gpu_beam import T, U, crafted, decode, tau
from tests.test_gpu_lm import (SEVERITY, TEST_SEEDS, _pages, chain_model, chain_words, lm_decode, pseudo_pages,
                               pseudo_words)

pytestmark = pytest.mark.gpu


def _stream():
    return torch.cuda.current_stream().cuda_stream


@pytest.fixture(scope="module")
def ctx(cuda_device):
    return _lib.Context(0)


def _alphabet(k):
    return "".join(chr(0x61 + i) if i < 26 else chr(0x100 + i) for i in range(k - 1))


def hot_decode(ctx, logits, hw, w, p, lm=None, fused=True):
    x = torch.from_numpy(np.ascontiguousarray(logits, np.float32)).cuda()
    b, _, k = x.shape
    labels = torch.empty((b, p, T), dtype=torch.int32, device="cuda")
    logp = torch.empty((b, p), dtype=torch.float32, device="cuda")
    fu = torch.empty((b, p), dtype=torch.float32, device="cuda") if fused else None
    ctx.ctc_beam_hotword_decode(x.data_ptr(), b, k, w, p, None if lm is None else lm.descriptor("cuda:0"),
                                hw.descriptor("cuda:0"), labels.data_ptr(), logp.data_ptr(),
                                fu.data_ptr() if fused else None, _stream())
    return labels.cpu().numpy(), logp.cpu().numpy(), (fu.cpu().numpy() if fused else None)


def _paths(labels):
    return [tuple(int(c) for c in row if c >= 0) for row in labels]


def word_list(logits, k, n, seed):
    """``n`` distinct words over the k-1 labels: the greedy readings of the crops, single-label edits of them (so the
    list competes with what the image says) and random words."""
    rng = np.random.default_rng(seed)
    al = _alphabet(k)
    near = []
    for x in logits:
        g = BR.collapse(np.argmax(x, -1), k - 1)[:12]
        if g:
            near.append(g)
            e = list(g)
            e[int(rng.integers(len(e)))] = int(rng.integers(k - 1))
            near.append(tuple(e))
    out, seen = [], set()
    for s in near + [tuple(rng.integers(0, k - 1, int(rng.integers(1, 13)))) for _ in range(4 * n)]:
        word = "".join(al[c] for c in s)
        if word and word not in seen:
            seen.add(word)
            out.append(word)
        if len(out) == n:
            break
    return Hotwords(out, weight=1.0, alphabet=al)


def check_hot(logits, labels, logp, fused, hw, w, what, lm=None):
    taus, lps = tau(logits), BR.log_probs(logits)
    seqs = HR.encode(hw.words, hw.alphabet)
    model = {} if lm is None else dict(zip(("keys", "rows"), lm.host_tables()), order=lm.order, alpha=lm.alpha,
                                      beta=lm.beta)
    worst, near = 0.0, 0
    for i in range(len(logits)):
        p = labels.shape[1]
        paths, a, fend, info = HR.beam_search_hot(lps[i], w, seqs, hw.weight, top_paths=p, **model)
        got = _paths(labels[i, :len(paths)])
        tf = taus[i] + 4 * U * (np.abs(fend).max() + 1)
        assert np.all(np.diff(fused[i, :len(paths)]) <= 0), (what, i)
        assert len(set(got)) == len(got), (what, i)
        same = got == paths
        if min(info["prune_margin"], info["rank_margin"]) > 2 * tf:
            assert same, (what, i, info, tf)
        if same:
            assert np.abs(logp[i, :len(paths)] - a).max() <= taus[i], (what, i)
            r = float(np.abs(fused[i, :len(paths)] - fend).max() / tf)
            assert r <= 1.0, (what, i, r)
            worst = max(worst, r)
        else:
            near += 1
            for s, v in zip(got, logp[i]):
                assert v <= BR.forward_logprob(lps[i], s) + taus[i], (what, i, s)
    return worst, near


# ------------------------------------------------------------------------------------------ 1. the decoder alone
@pytest.mark.parametrize("with_model", [False, True])
@pytest.mark.parametrize("k", [5, 37, 127])
def test_decoder_vs_reference(ctx, k, with_model):
    report = []
    big = None
    for w, n in ((1, 12), (4, 12), (16, 6), (128, 2)):
        lm = chain_model(k + w, k, order=3 + w % 3).weighted(0.8, 0.3) if with_model else None
        logits = crafted(k, n, seed=9000 + k * 10 + w)
        for size in (1, 100, 100000):
            if size == 100000 and w not in (4, 128):
                continue
            hw = word_list(logits, k, size, seed=size + w).weighted(0.5 + (w % 3))
            if size == 100000:
                big = hw
            labels, logp, fused = hot_decode(ctx, logits, hw, w, w, lm)
            worst, near = check_hot(logits, labels, logp, fused, hw, w, (k, w, size), lm)
            assert near <= max(1, n // 3), (k, w, size, near)
            report.append(f"W={w} n={len(hw)}: worst {worst:.3g} of tau_F, near-tie crops {near}/{n}")
        for p in sorted({1, 3} & set(range(1, w + 1))):             # top_paths prefixes
            lab_p, lp_p, fu_p = hot_decode(ctx, logits, hw, w, p, lm)
            assert np.array_equal(lab_p, labels[:, :p]) and np.array_equal(lp_p.view(np.int32), logp[:, :p].view(np.int32))
            assert np.array_equal(fu_p.view(np.int32), fused[:, :p].view(np.int32))
        lab_b, _, fu_b = hot_decode(ctx, logits[:1], hw, w, w, lm)  # alone, in any batch, on every run
        assert np.array_equal(lab_b, labels[:1]) and np.array_equal(fu_b.view(np.int32), fused[:1].view(np.int32))
        more = np.concatenate([logits[::-1], crafted(k, 5, seed=1)])
        lab_c, lp_c, _ = hot_decode(ctx, more, hw, w, w, lm)
        assert np.array_equal(lab_c[:n][::-1], labels) and np.array_equal(lp_c[:n][::-1].view(np.int32),
                                                                           logp.view(np.int32))
        again = hot_decode(ctx, logits, hw, w, w, lm)
        assert np.array_equal(again[0], labels) and np.array_equal(again[2].view(np.int32), fused.view(np.int32))
    assert big is not None and len(big) == 100000
    print(f"beam+hotwords K={k} model={with_model}: " + "; ".join(report))


@pytest.mark.parametrize("k", [5, 37, 127])
def test_zero_weight_and_empty_list_are_the_plain_and_lm_search_bit_for_bit(ctx, k):
    lm = chain_model(k, k, order=4)
    logits = crafted(k, 24, seed=k)
    al = _alphabet(k)
    lists = (word_list(logits, k, 100, seed=3).weighted(0.0), Hotwords([], weight=3.0, alphabet=al))
    for w in (1, 4, 16, 128):
        p = min(w, 3)
        ref_l, ref_p = decode(ctx, logits, w, p)
        lm_l, lm_p, lm_f = lm_decode(ctx, logits, lm, w, p)
        for hw in lists:
            labels, logp, fused = hot_decode(ctx, logits, hw, w, p)
            assert np.array_equal(labels, ref_l) and np.array_equal(logp.view(np.int32), ref_p.view(np.int32))
            labels, logp, fused = hot_decode(ctx, logits, hw, w, p, lm)
            assert np.array_equal(labels, lm_l) and np.array_equal(logp.view(np.int32), lm_p.view(np.int32))
            assert np.array_equal(fused.view(np.int32), lm_f.view(np.int32))


def _crnn_input(rec, n=None):
    crops = np.load(os.path.join(os.path.dirname(__file__), "golden", "c3_crops.npz"))["crops"]
    crops = crops if n is None else crops[:n]
    t = torch.from_numpy(np.ascontiguousarray(crops)).cuda()
    x = torch.empty((len(crops), 200, 31), dtype=torch.float16, device="cuda")
    rec.ctx.crops_to_input(t.data_ptr(), len(crops), x.data_ptr(), _stream())
    return crops, x


def test_zero_weight_through_the_crnn(cuda_device):
    rec = Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True))
    _, x = _crnn_input(rec)
    lm = CharLM.fit(chain_words(3, 2000, rec.alphabet), rec.alphabet, order=5)
    words = chain_words(4, 500, rec.alphabet)
    for hw in (Hotwords(sorted(set(words)), weight=0.0, alphabet=rec.alphabet), Hotwords([], alphabet=rec.alphabet)):
        for w in (1, 10, 100):
            p = min(w, 3)
            a = rec.predict_device(x, with_scores=True, beam_width=w, top_paths=p)
            b = rec.predict_device(x, with_scores=True, beam_width=w, top_paths=p, hotwords=hw)
            assert torch.equal(a[0], b[0]) and torch.equal(a[1].view(torch.int32), b[1].view(torch.int32))
            a = rec.predict_device(x, with_scores=True, beam_width=w, top_paths=p, language_model=lm)
            b = rec.predict_device(x, with_scores=True, beam_width=w, top_paths=p, language_model=lm, hotwords=hw)
            assert torch.equal(a[0], b[0]) and torch.equal(a[1].view(torch.int32), b[1].view(torch.int32))


def test_memory_contract(ctx):
    """Nothing is written outside labels[:, :P], logp[:, :P], fused[:, :P]; fused and logp may be NULL."""
    k, b, w, p = 37, 5, 16, 3
    logits = crafted(k, b, seed=3)
    hw = word_list(logits, k, 100, seed=5).weighted(2.0)
    for lm in (None, chain_model(11, k, order=5)):
        ref = hot_decode(ctx, logits, hw, w, p, lm)
        x = torch.from_numpy(logits).cuda()
        guard = 1024
        lab = torch.full((b * p * T + 2 * guard,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
        lp = torch.full((b * p + 2 * guard,), 1234.5, dtype=torch.float32, device="cuda")
        fu = torch.full((b * p + 2 * guard,), -777.25, dtype=torch.float32, device="cuda")
        for with_logp, with_fused in ((True, True), (True, False), (False, True), (False, False)):
            ctx.ctc_beam_hotword_decode(x.data_ptr(), b, k, w, p, None if lm is None else lm.descriptor("cuda:0"),
                                        hw.descriptor("cuda:0"), lab[guard:].data_ptr(),
                                        lp[guard:].data_ptr() if with_logp else None,
                                        fu[guard:].data_ptr() if with_fused else None, _stream())
            h_lab, h_lp, h_fu = lab.cpu().numpy(), lp.cpu().numpy(), fu.cpu().numpy()
            assert (h_lab[:guard] == 0x5A5A5A5A).all() and (h_lab[guard + b * p * T:] == 0x5A5A5A5A).all()
            assert np.array_equal(h_lab[guard:guard + b * p * T].reshape(b, p, T), ref[0])
            for arr, fill, on, want in ((h_lp, 1234.5, with_logp, ref[1]), (h_fu, -777.25, with_fused, ref[2])):
                assert (arr[:guard] == fill).all() and (arr[guard + b * p:] == fill).all()
                if on:
                    assert np.array_equal(arr[guard:guard + b * p].reshape(b, p).view(np.int32), want.view(np.int32))
                else:
                    assert (arr[guard:guard + b * p] == fill).all()
            lp.fill_(1234.5)
            fu.fill_(-777.25)


def test_abi_rejects_out_of_range(ctx):
    lm = chain_model(5, 37, order=3)
    hw = Hotwords(["ab", "abc", "b"], alphabet=_alphabet(37))
    x = torch.zeros((2, T, 37), dtype=torch.float32, device="cuda")
    labels = torch.empty((2, 128, T), dtype=torch.int32, device="cuda")
    lib, h = ctx.lib, ctx.handle
    good = hw.descriptor("cuda:0")
    n0 = ctx.launch_count()

    def call(b=2, k=37, w=5, p=1, desc=good, model=None, logits=x.data_ptr()):
        return lib.b2o_ctc_beam_hotword_decode(h, logits, b, k, w, p, model, desc, labels.data_ptr(), None, None,
                                               None)

    for kw in ({"w": 0}, {"w": 129}, {"p": 0}, {"p": 6}, {"k": 1}, {"k": 128}, {"b": -1}, {"logits": None},
               {"desc": None}):
        assert call(**kw) == -2 and lib.b2o_last_error(h)
    for field, value in (("n_nodes", 0), ("n_nodes", (1 << 24) + 2), ("n_edges", 2), ("keys_dev", None),
                         ("child_dev", None), ("final_dev", None), ("weight", -1.0), ("weight", float("nan")),
                         ("weight", float("inf"))):
        d = _lib.HotwordsDesc(good.n_nodes, good.n_edges, good.keys_dev, good.child_dev, good.final_dev, good.weight)
        setattr(d, field, value)
        assert call(desc=d) == -2 and lib.b2o_last_error(h)
    bad_lm = _lib.CharLMDesc(1, 1, None, None, 0.0, 0.0)
    assert call(model=bad_lm) == -2 and lib.b2o_last_error(h)
    assert call(model=lm.descriptor("cuda:0"), k=128) == -2
    rec = Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True))
    nbytes = rec.ctx.crnn_workspace_bytes(2)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    xin = torch.zeros((2, 200, 31), dtype=torch.float16, device="cuda")
    m0 = rec.ctx.launch_count()
    for w, p, desc in [(0, 1, good), (129, 1, good), (5, 6, good), (5, 0, good), (5, 1, None)]:
        assert rec.ctx.lib.b2o_crnn_forward_beam_hotword(rec.ctx.handle, xin.data_ptr(), 2, w, p, None, desc,
                                                         labels.data_ptr(), None, None, ws.data_ptr(), nbytes,
                                                         None) == -2
    assert ctx.launch_count() == n0 and rec.ctx.launch_count() == m0
    torch.cuda.synchronize()


def test_a_listed_word_wins_an_ambiguous_image(ctx):
    """'o' and '0' compete at the second character with equal logits: plain beam search keeps the smaller label
    sequence, 'b0ak'; with 'boak' listed the bonus decides, and a list of another word changes nothing."""
    from keras_ocr_b200.recognition import DEFAULT_ALPHABET as A
    k = len(A) + 1
    x = np.full((1, T, k), -8.0, np.float32)
    x[0, :, k - 1] = 6.0
    for j, ch in enumerate("b?ak"):
        t = 6 + 8 * j
        for c in ("0", "o") if ch == "?" else (ch,):
            x[0, t, A.index(c)] = 7.0

    def read(hw):
        return "".join(A[c] for c in _paths(hot_decode(ctx, x, hw, 8, 1)[0][0])[0])

    assert read(Hotwords([], alphabet=A)) == "b0ak"
    assert read(Hotwords(["boak"], alphabet=A)) == "boak"
    # at the end only a listed word keeps its bonus: F_end = A + weight * |a| for "bo", F_end = A for every other reading
    hw = Hotwords(["soak", "bo"], alphabet=A)
    labels, logp, fused = hot_decode(ctx, x, hw, 8, 3)
    for path, a, f in zip(_paths(labels[0]), logp[0], fused[0]):
        text = "".join(A[c] for c in path)
        want = np.float32(a + np.float32(hw.weight * len(text))) if text in hw.words else a
        assert f.view(np.int32) == np.float32(want).view(np.int32), (text, a, f)


# ------------------------------------------------------------------------------------------ 2. every read path
@pytest.fixture(scope="module")
def pipe(cuda_device):
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    return Pipeline(detector=Detector(weights=W.synthetic_craft_weights(3, textlike=True), device=0),
                    recognizer=Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True), device=0), scale=2)


def _page_words(pipe, pages):
    return sorted({t for g in pipe.recognize(pages, recognition_kwargs={"beam_width": 8}) for t, _ in g if t})


@pytest.mark.parametrize("with_model", [False, True])
def test_read_paths_agree(pipe, with_model):
    from keras_ocr_b200 import distributed as D
    from keras_ocr_b200.recognition import labels_to_text
    rec = pipe.recognizer
    pages = _pages()
    words = sorted(set(_page_words(pipe, pages)[::2] + chain_words(9, 300, rec.alphabet)))
    hw = Hotwords(words, weight=2.0, alphabet=rec.alphabet)
    kw = {"beam_width": 8, "hotwords": hw}
    if with_model:
        kw["language_model"] = CharLM.fit(chain_words(5, 3000, rec.alphabet), rec.alphabet, order=5)
    res = pipe.recognize(pages, recognition_kwargs=kw)
    boxes = [[b for _, b in g] for g in res]
    assert [[t for t, _ in g] for g in res] == rec.recognize_from_boxes(list(pages), boxes, **kw)
    crops, x = _crnn_input(rec, 64)
    assert rec.recognize_crops(crops, **kw) == labels_to_text(rec.predict_device(x, **kw).cpu().numpy(), rec.alphabet)
    assert isinstance(rec.recognize(crops[0], **kw), str)
    listed = dict(kw, hotwords=list(hw.words))                      # a plain list, compiled per call, default weight
    assert rec.recognize_crops(crops, **listed) == rec.recognize_crops(crops, **dict(kw, hotwords=hw.weighted()))
    scored = pipe.recognize(pages, recognition_kwargs=kw, return_scores=True)
    assert [[w[0] for w in g] for g in scored] == [[t for t, _ in g] for g in res]
    lines = pipe.recognize(pages, recognition_kwargs=kw, return_lines=True, return_blocks=True)
    assert sorted(w[0] for g in lines for bl in g for ln in bl[2] for w in ln[2]) == sorted(t for g in res for t, _ in g)
    cells = pipe.recognize(pages, recognition_kwargs=kw, return_char_boxes=True, return_char_scores=True,
                           char_alternatives=2)
    assert [[w[0] for w in g] for g in cells] == [[t for t, _ in g] for g in res]
    assert all(len(w[2]) == len(w[0]) == len(w[3][0]) for g in cells for w in g)
    polys = pipe.recognize(pages, recognition_kwargs=kw, return_polygons=True)
    assert [[w[0] for w in g] for g in polys] == [[t for t, _ in g] for g in res]
    top = pipe.recognize(pages, recognition_kwargs=dict(kw, top_paths=3))
    assert [[t[0] for t, _ in g] for g in top] == [[t for t, _ in g] for g in res]
    pipe.inflight = 2
    try:
        assert [[t for t, _ in g] for g in pipe.recognize(pages, recognition_kwargs=kw)] == \
            [[t for t, _ in g] for g in res]
    finally:
        pipe.inflight = 1
    rk = {k: v for k, v in kw.items() if k != "beam_width"}
    records = pipe.recognize_records(pages, beam_width=8, scores=True, **rk)
    decoded = D._decode_blocks([records.cpu()], 128, rec.alphabet, True)
    assert [[w[0] for w in g] for g in decoded] == [[t for t, _ in g] for g in res]
    assert [[np.float32(w[3]) for w in g] for g in decoded] == [[np.float32(w[3]) for w in g] for g in scored]
    sharded = D.recognize_sharded(pipe, pages, beam_width=8, **rk)
    assert [[t for t, _ in g] for g in sharded] == [[t for t, _ in g] for g in res]
    stream = D.ShardedStream(pipe, beam_width=8, **rk)
    assert stream.submit(pages) is None
    assert [[t for t, _ in g] for g in stream.flush()] == [[t for t, _ in g] for g in res]


def test_alignment_and_char_scores_run_after_the_new_forward(pipe):
    """The hotword forward keeps its logits: the character spans and scores of its readings equal those computed for
    the same labels on the logits of a plain forward of the same crops."""
    rec = pipe.recognizer
    crops, x = _crnn_input(rec, 32)
    hw = Hotwords(sorted(set(chain_words(9, 400, rec.alphabet))), weight=3.0, alphabet=rec.alphabet)
    labels, logp, spans, theta, scores = rec._predict_aligned(x, 8, 2, None, char_scores=3, hotwords=hw)
    # the same labels aligned and scored on the logits the greedy forward keeps
    lab2 = torch.empty_like(labels)
    nbytes = rec.ctx.crnn_workspace_bytes(len(crops))
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    rec.ctx.crnn_forward_logits(x.data_ptr(), len(crops), lab2.data_ptr(), None, ws.data_ptr(), nbytes, _stream())
    sp2 = torch.empty_like(spans)
    rec.ctx.crnn_align(len(crops), labels.data_ptr(), 2, sp2.data_ptr(), None,
                       None if theta is None else torch.empty_like(theta).data_ptr(), ws.data_ptr(), nbytes, _stream())
    conf2, al2, po2 = (torch.empty_like(t) for t in scores)
    rec.ctx.crnn_char_scores(len(crops), labels.data_ptr(), 2, 3, conf2.data_ptr(), al2.data_ptr(), po2.data_ptr(),
                             None, ws.data_ptr(), nbytes, _stream())
    assert torch.equal(spans, sp2)
    for a, b in zip(scores, (conf2, al2, po2)):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def test_rotations_vote_on_fused_scores(pipe):
    """Per word, against the decoder's own outputs for every turn: the chosen turn maximises F_end (ties: the turn
    listed first) and the confidence is exp of that turn's acoustic logp."""
    from keras_ocr_b200 import tools
    from keras_ocr_b200.recognition import confidences, labels_to_text
    rec = pipe.recognizer
    pages = _pages(1, seed=1001)
    turned = np.ascontiguousarray(np.rot90(pages, 2, axes=(1, 2)))
    boxes = np.stack([b for _, b in pipe.recognize(turned)[0]]).astype(np.float32)
    flat = torch.from_numpy(tools.rectify_boxes(boxes.copy())).cuda()
    idx = torch.zeros(len(boxes), dtype=torch.int32, device="cuda")
    gray = rec.gray_device(torch.from_numpy(turned).cuda())
    turns, disagree = (0, 1, 2, 3), 0
    # the list: what the sideways turns read, so that a large weight makes the F_end vote and a vote on the acoustic
    # score disagree on some words and the check tells them apart
    side = torch.empty((len(boxes), 1, T), dtype=torch.int32, device="cuda")
    words = set()
    for t in (1, 3):
        crnn_in, _ = rec.warp_device(gray, flat.clone(), idx, turn=t)
        rec._forward(crnn_in, side, None, 8, 1, None)
        words.update(w for w in labels_to_text(side[:, 0].cpu().numpy(), rec.alphabet) if w)
    words = sorted(words)
    for gamma in (0.5, 2.0, 10.0):
        hw = Hotwords(words, weight=gamma, alphabet=rec.alphabet)
        labels = torch.empty((4, len(boxes), 1, T), dtype=torch.int32, device="cuda")
        logp, fused = (torch.empty((4, len(boxes), 1), dtype=torch.float32, device="cuda") for _ in range(2))
        for j, t in enumerate(turns):
            crnn_in, _ = rec.warp_device(gray, flat.clone(), idx, turn=t)
            rec._forward(crnn_in, labels[j], logp[j], 8, 1, None, fused=fused[j], hotwords=hw)
        f, a = fused[:, :, 0].cpu().numpy(), logp[:, :, 0].cpu().numpy()
        pick = np.argmax(f, axis=0)
        disagree += int((pick != np.argmax(a, axis=0)).sum())
        rows = np.arange(len(boxes))
        want_text = labels_to_text(labels[:, :, 0].cpu().numpy()[pick, rows], rec.alphabet)
        want_conf = confidences(a[pick, rows])
        res = rec.recognize_from_boxes([turned[0]], [list(boxes)], return_scores=True, beam_width=8, hotwords=hw,
                                       rotations=turns, rotation_vote="word")[0]
        assert [t for t, _ in res] == want_text
        assert np.array_equal(np.array([c for _, c in res], np.float32).view(np.int32), want_conf.view(np.int32))
    assert disagree > 0


def test_invalid_combinations_raise_before_any_launch(pipe):
    rec = pipe.recognizer
    lm = CharLM.fit(["abc", "abd"], rec.alphabet, order=3)
    hw = Hotwords(["abc"], alphabet=rec.alphabet)
    other = Hotwords(["abc"], alphabet="abcd")
    pages = _pages(1, seed=1002)
    n0 = pipe.detector.ctx.launch_count() + rec.ctx.launch_count()
    bad = [{"hotwords": hw}, {"hotwords": hw, "language_model": lm},
           {"hotwords": hw, "beam_width": 4, "lexicon": ["abc"]}, {"hotwords": hw, "beam_width": 4, "pattern": "a.*"},
           {"hotwords": other, "beam_width": 4}, {"hotwords": hw, "beam_width": 4, "max_windows": 2},
           {"hotwords": "abc", "beam_width": 4}, {"hotwords": hw, "beam_width": 4, "top_paths": 5},
           {"hotwords": ["ab", "ab"], "beam_width": 4}, {"hotwords": ["a!"], "beam_width": 4}]
    for kw in bad:
        with pytest.raises(ValueError):
            pipe.recognize(pages, recognition_kwargs=kw)
        with pytest.raises(ValueError):
            rec.recognize_from_boxes(list(pages), [[np.array([[0, 0], [50, 0], [50, 20], [0, 20]], np.float32)]],
                                     **kw)
        if "max_windows" not in kw:
            with pytest.raises(ValueError):
                rec.recognize_crops(np.zeros((1, 31, 200), np.uint8), **kw)
    with pytest.raises(ValueError, match="hotwords need beam search: pass beam_width"):
        rec.recognize_crops(np.zeros((1, 31, 200), np.uint8), hotwords=hw)
    from keras_ocr_b200 import distributed as D
    for kw in ({"hotwords": hw}, {"hotwords": hw, "beam_width": 4, "top_paths": 2}):
        with pytest.raises(ValueError):
            pipe.recognize_records(pages, **kw)
        with pytest.raises(ValueError):
            D.recognize_sharded(pipe, pages, **kw)
        with pytest.raises(ValueError):
            D.ShardedStream(pipe, **kw)
    assert pipe.detector.ctx.launch_count() + rec.ctx.launch_count() == n0


def test_the_recognize_stage_does_not_wait_for_the_device(pipe, monkeypatch):
    """With hotwords the recognize stage queues its work without a host synchronisation (torch raises on one in
    sync-debug mode "error")."""
    rec = pipe.recognizer
    hw = Hotwords(sorted(set(chain_words(9, 300, rec.alphabet))), alphabet=rec.alphabet)
    lm = CharLM.fit(chain_words(5, 3000, rec.alphabet), rec.alphabet, order=5)
    hw.descriptor(rec.device)                                  # uploaded once, before the checked stage
    lm.descriptor(rec.device)
    pages = _pages()
    pipe.recognize(pages, recognition_kwargs={"beam_width": 8, "hotwords": hw})   # the model of zeros, once
    stage = pipe._stage_recognize
    calls = []

    def strict(*args, **kw):
        torch.cuda.set_sync_debug_mode("error")
        try:
            return stage(*args, **kw)
        finally:
            torch.cuda.set_sync_debug_mode("default")
            calls.append(1)

    monkeypatch.setattr(pipe, "_stage_recognize", strict)
    for kw in ({"beam_width": 8, "hotwords": hw}, {"beam_width": 8, "hotwords": hw, "language_model": lm}):
        pipe.recognize(pages, recognition_kwargs=kw, return_scores=True)
    assert len(calls) == 2


# ------------------------------------------------------------------------------------------ 3. accuracy
UNLISTED_SLACK = 1       # unlisted words read exactly with hotwords >= without - this, on the held-out pages


def test_listed_words_read_better_on_degraded_pages(pipe):
    """On the held-out degraded pages (``test_gpu_lm.TEST_SEEDS`` at ``SEVERITY``) the page words outside the language
    model's corpus are listed as hotwords at the default weight (tuned on seeds 100..103, scripts/bench_hotwords.py).
    Listed words read strictly more exactly, with and without the model; unlisted words lose at most
    ``UNLISTED_SLACK`` exact reads."""
    from keras_ocr_b200.recognition import DEFAULT_ALPHABET as A
    from tests import window_refs as R
    rec = pipe.recognizer
    corpus = pseudo_words(77, 20000, A[10:], sample_seed=1)
    lm = CharLM.fit(corpus, rec.alphabet, order=5)
    pages, items = pseudo_pages(TEST_SEEDS, SEVERITY)
    seen = set(corpus)
    names = sorted({w for it in items for w, _ in it if w not in seen})
    hw = Hotwords(names, alphabet=rec.alphabet)

    def split(kw):
        res = pipe.recognize(pages, recognition_kwargs=kw)
        out = [0, 0]
        for g, it in zip(res, items):
            for listed in (0, 1):
                sub = [(w, c) for w, c in it if (w in hw.words) == bool(listed)]
                out[listed] += R.exact_reads(g, sub)
        return out

    unl_b, lis_b = split({"beam_width": 16})
    unl_h, lis_h = split({"beam_width": 16, "hotwords": hw})
    unl_l, lis_l = split({"beam_width": 16, "language_model": lm})
    unl_lh, lis_lh = split({"beam_width": 16, "language_model": lm, "hotwords": hw})
    print(f"held-out degraded pages: {len(names)} listed names; exact reads (unlisted, listed): beam {unl_b, lis_b}, "
          f"+hotwords {unl_h, lis_h}, +LM {unl_l, lis_l}, +LM+hotwords {unl_lh, lis_lh} (weight {hw.weight})")
    assert lis_h > lis_b and lis_lh > lis_l
    assert unl_h >= unl_b - UNLISTED_SLACK and unl_lh >= unl_l - UNLISTED_SLACK
