"""CTC beam search constrained to a pattern on the GPU (``b2o_ctc_beam_pattern_decode``,
``b2o_crnn_forward_beam_pattern``) against tests/pattern_refs.py, and the ``pattern=`` option on every read path.

Bound.  The search ranks and merges exactly as plain beam search does, so the bound of tests/test_gpu_beam.py holds:
where the reference's prune and rank margins exceed 2 tau the kernel returns the same readings with |A - ref| <= tau;
elsewhere (a near-tie, counted and bounded) every returned reading's A is at most its exact forward log-probability +
tau.  A near-tie may also lead to the same readings along another trajectory, with other scores: it counts as one.
Constrained readings of the peaked crops sit at the 1e-7 floor of lp, where labels tie within a few ulps, so near-ties
are more frequent than for plain beam search: at most half the crops.  Every returned reading matches the pattern in
full, whatever the margins.
"""
import numpy as np
import pytest
import torch

from keras_ocr_b200 import _lib, weights as W
from keras_ocr_b200.recognition import DEFAULT_ALPHABET, Pattern, Recognizer
from tests import beam_refs as BR
from tests import pattern_refs as PR
from tests.test_gpu_beam import T, crafted, decode, tau

pytestmark = pytest.mark.gpu


def _stream():
    return torch.cuda.current_stream().cuda_stream


@pytest.fixture(scope="module")
def ctx(cuda_device):
    return _lib.Context(0)


def alphabet_for(k):
    """k - 1 characters: the default alphabet's, then code points from U+0100."""
    return (DEFAULT_ALPHABET + "".join(chr(0x100 + i) for i in range(200)))[:k - 1]


def patterns_for(k):
    a = alphabet_for(k)
    return {"universal": ".*", "digits": "\\d+", "format": f"{a[1]}[{a[0]}-{a[2]}]{{3}}\\d{{2}}",
            "alternation": f"({a[0]}{a[1]}|{a[2]}+|{a[1]}{a[2]}{a[0]}){a[-1]}?", "empty_ok": f"({a[1]}{a[2]})*",
            "unreachable": f"{a[0]}{{30}}"}


def pat_decode(ctx, logits, pat, w, p, with_logp=True):
    x = torch.from_numpy(np.ascontiguousarray(logits, np.float32)).cuda()
    b, _, k = x.shape
    labels = torch.empty((b, p, T), dtype=torch.int32, device="cuda")
    logp = torch.empty((b, p), dtype=torch.float32, device="cuda")
    ctx.ctc_beam_pattern_decode(x.data_ptr(), b, k, w, p, pat.descriptor("cuda:0"), labels.data_ptr(),
                                logp.data_ptr() if with_logp else None, _stream())
    return labels.cpu().numpy(), logp.cpu().numpy()


def _paths(labels):
    return [tuple(int(c) for c in row if c >= 0) for row in labels]


def check_pattern(logits, labels, logp, pat, w, what):
    taus, lps = tau(logits), BR.log_probs(logits)
    worst, near = 0.0, 0
    for i in range(len(logits)):
        p = labels.shape[1]
        paths, a, info = PR.beam_search_pattern(lps[i], w, *pat.host_tables(), top_paths=p)
        got = _paths(labels[i, :len(paths)])
        for row, v in zip(labels[i], logp[i]):       # a slot past the survivors is -1 with -inf; every reading matches
            if np.isfinite(v) or (row >= 0).any():
                assert pat.fullmatch("".join(pat.alphabet[c] for c in row if c >= 0)), (what, i, row)
        assert np.array_equal(np.sort(logp[i])[::-1], logp[i]), (what, i)             # best first
        same = got == paths
        r = float(np.abs(logp[i, :len(paths)] - a).max() / taus[i]) if same and paths else 0.0
        if min(info["prune_margin"], info["rank_margin"]) > 2 * taus[i]:
            assert same and r <= 1.0, (what, i, info, taus[i], r)
        if same and r <= 1.0:
            worst = max(worst, r)
        else:                                  # a near-tie: another trajectory, to other readings or the same ones
            near += 1
            for s, v in zip(got, logp[i]):
                assert v <= BR.forward_logprob(lps[i], s) + taus[i], (what, i, s)
    return worst, near


# ------------------------------------------------------------------------------------------ 1. the decoder alone
@pytest.mark.parametrize("k", [5, 37, 127])
def test_decoder_vs_reference(ctx, k):
    report = []
    for name, text in patterns_for(k).items():
        pat = Pattern(text, alphabet_for(k))
        for w, n in ((1, 12), (4, 12), (16, 6), (128, 2)):
            logits = crafted(k, n, seed=9000 + k * 10 + w + len(name))
            labels, logp = pat_decode(ctx, logits, pat, w, w)
            worst, near = check_pattern(logits, labels, logp, pat, w, (k, name, w))
            assert near <= max(1, n // 2), (k, name, w, near)
            report.append(f"{name} W={w}: {worst:.3g} tau, near {near}/{n}")
            if name == "unreachable":
                assert (labels == -1).all() and (logp == -np.inf).all()
            for p in sorted({1, 3} & set(range(1, w + 1))):             # top_paths prefixes agree
                lab_p, lp_p = pat_decode(ctx, logits, pat, w, p)
                assert np.array_equal(lab_p, labels[:, :p])
                assert np.array_equal(lp_p.view(np.int32), logp[:, :p].view(np.int32))
            lab_b, lp_b = pat_decode(ctx, logits[:1], pat, w, w)         # alone, in any batch, on every run
            assert np.array_equal(lab_b, labels[:1]) and np.array_equal(lp_b.view(np.int32), logp[:1].view(np.int32))
            big = np.concatenate([logits[::-1], crafted(k, 5, seed=1)])
            lab_c, lp_c = pat_decode(ctx, big, pat, w, w)
            assert np.array_equal(lab_c[:n][::-1], labels)
            assert np.array_equal(lp_c[:n][::-1].view(np.int32), logp.view(np.int32))
            again = pat_decode(ctx, logits, pat, w, w)
            assert np.array_equal(again[0], labels) and np.array_equal(again[1].view(np.int32), logp.view(np.int32))
    print(f"beam+pattern K={k}: " + "; ".join(report))


@pytest.mark.parametrize("k", [5, 37, 127])
def test_universal_pattern_is_plain_beam_search_bit_for_bit(ctx, k):
    pat = Pattern(".*", alphabet_for(k))
    logits = crafted(k, 24, seed=k + 1)
    for w in (1, 4, 16, 128):
        labels, logp = pat_decode(ctx, logits, pat, w, min(w, 3))
        ref_l, ref_p = decode(ctx, logits, w, min(w, 3))
        assert np.array_equal(labels, ref_l) and np.array_equal(logp.view(np.int32), ref_p.view(np.int32))


def test_memory_contract(ctx, golden_dir):
    """Nothing is written outside labels[:, :P] and logp[:, :P] (logp may be NULL), nor outside the CRNN workspace."""
    k, b, w, p = 37, 5, 16, 3
    pat = Pattern("[a-z]{2,4}\\d{2}")
    logits = crafted(k, b, seed=3)
    ref = pat_decode(ctx, logits, pat, w, p)
    x = torch.from_numpy(logits).cuda()
    guard = 1024
    lab = torch.full((b * p * T + 2 * guard,), 0x5A5A5A5A, dtype=torch.int32, device="cuda")
    lp = torch.full((b * p + 2 * guard,), 1234.5, dtype=torch.float32, device="cuda")
    for with_logp in (True, False):
        ctx.ctc_beam_pattern_decode(x.data_ptr(), b, k, w, p, pat.descriptor("cuda:0"), lab[guard:].data_ptr(),
                                    lp[guard:].data_ptr() if with_logp else None, _stream())
        h_lab, h_lp = lab.cpu().numpy(), lp.cpu().numpy()
        assert (h_lab[:guard] == 0x5A5A5A5A).all() and (h_lab[guard + b * p * T:] == 0x5A5A5A5A).all()
        assert np.array_equal(h_lab[guard:guard + b * p * T].reshape(b, p, T), ref[0])
        assert (h_lp[:guard] == 1234.5).all() and (h_lp[guard + b * p:] == 1234.5).all()
        if with_logp:
            assert np.array_equal(h_lp[guard:guard + b * p].reshape(b, p).view(np.int32), ref[1].view(np.int32))
        else:
            assert (h_lp[guard:guard + b * p] == 1234.5).all()
        lp.fill_(1234.5)

    import os
    crops = np.load(os.path.join(golden_dir, "c3_crops.npz"))["crops"][:b]
    rec = Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True))
    t = torch.from_numpy(np.ascontiguousarray(crops)).cuda()
    xin = torch.empty((b, 200, 31), dtype=torch.float16, device="cuda")
    rec.ctx.crops_to_input(t.data_ptr(), b, xin.data_ptr(), _stream())
    want = rec.predict_device(xin, with_scores=True, beam_width=w, top_paths=p, pattern=pat)
    nbytes = rec.ctx.crnn_workspace_bytes(b)
    ws = torch.full((nbytes + 2 * guard,), 0xA5, dtype=torch.uint8, device="cuda")
    lab.fill_(0x5A5A5A5A)
    rec.ctx.crnn_forward_beam_pattern(xin.data_ptr(), b, w, p, pat.descriptor("cuda:0"), lab[guard:].data_ptr(),
                                      lp[guard:].data_ptr(), ws[guard:].data_ptr(), nbytes, _stream())
    h_ws, h_lab, h_lp = ws.cpu().numpy(), lab.cpu().numpy(), lp.cpu().numpy()
    assert (h_ws[:guard] == 0xA5).all() and (h_ws[guard + nbytes:] == 0xA5).all()
    assert (h_lab[:guard] == 0x5A5A5A5A).all() and (h_lab[guard + b * p * T:] == 0x5A5A5A5A).all()
    assert (h_lp[:guard] == 1234.5).all() and (h_lp[guard + b * p:] == 1234.5).all()
    assert np.array_equal(h_lab[guard:guard + b * p * T].reshape(b, p, T), want[0].cpu().numpy())
    assert np.array_equal(h_lp[guard:guard + b * p].reshape(b, p).view(np.int32),
                          want[1].cpu().numpy().view(np.int32))


def test_abi_rejects_out_of_range(ctx):
    pat = Pattern("[0-9]+")
    x = torch.zeros((2, T, 37), dtype=torch.float32, device="cuda")
    labels = torch.empty((2, 128, T), dtype=torch.int32, device="cuda")
    lib, h = ctx.lib, ctx.handle
    good = pat.descriptor("cuda:0")
    n0 = ctx.launch_count()

    def call(b=2, k=37, w=5, p=1, desc=good, logits=x.data_ptr()):
        return lib.b2o_ctc_beam_pattern_decode(h, logits, b, k, w, p, desc, labels.data_ptr(), None, None)

    for kw in ({"w": 0}, {"w": 129}, {"p": 0}, {"p": 6}, {"k": 1}, {"k": 128}, {"b": -1}, {"logits": None}):
        assert call(**kw) == -2 and lib.b2o_last_error(h)
    assert lib.b2o_ctc_beam_pattern_decode(h, x.data_ptr(), 2, 37, 5, 1, None, labels.data_ptr(), None, None) == -2
    for field, value in (("n_states", 0), ("n_states", 4097), ("start", -1), ("start", good.n_states),
                         ("trans_dev", None), ("dist_dev", None)):
        d = _lib.PatternDesc(good.n_states, good.start, good.trans_dev, good.dist_dev)
        setattr(d, field, value)
        assert call(desc=d) == -2 and lib.b2o_last_error(h)
    rec = Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True))
    nbytes = rec.ctx.crnn_workspace_bytes(2)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    xin = torch.zeros((2, 200, 31), dtype=torch.float16, device="cuda")
    m0 = rec.ctx.launch_count()
    for w, p in [(0, 1), (129, 1), (5, 6), (5, 0)]:
        assert rec.ctx.lib.b2o_crnn_forward_beam_pattern(rec.ctx.handle, xin.data_ptr(), 2, w, p, good,
                                                         labels.data_ptr(), None, ws.data_ptr(), nbytes, None) == -2
    assert ctx.launch_count() == n0 and rec.ctx.launch_count() == m0
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------ 2. every read path
@pytest.fixture(scope="module")
def pipe(cuda_device):
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    return Pipeline(detector=Detector(weights=W.synthetic_craft_weights(3, textlike=True), device=0),
                    recognizer=Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True), device=0), scale=2)


def _pages(n=2, seed=1000):
    from oracle import synth
    return synth.text_images(seed=seed, n=n, h=768, w=768, n_words=32)[0]


def _bits(groups):
    return [[np.float32(w[3]).view(np.int32) for w in g] for g in groups]


def test_universal_pattern_through_the_pipeline_is_beam_search(pipe):
    pages = _pages()
    for kw in ({"beam_width": 16}, {"beam_width": 8, "top_paths": 3}):
        a = pipe.recognize(pages, recognition_kwargs=kw, return_scores=True)
        b = pipe.recognize(pages, recognition_kwargs=dict(kw, pattern=".*"), return_scores=True)
        assert [[w[0] for w in g] for g in a] == [[w[0] for w in g] for g in b]
        assert [[np.asarray(w[3], np.float32).tobytes() for w in g] for g in a] == \
               [[np.asarray(w[3], np.float32).tobytes() for w in g] for g in b]


def test_read_paths_agree(pipe):
    from keras_ocr_b200 import distributed as D
    from keras_ocr_b200.recognition import labels_to_text
    rec = pipe.recognizer
    pat = Pattern("[a-z0-9]{1,12}")
    pages = _pages()
    kw = {"beam_width": 8, "pattern": pat}
    res = pipe.recognize(pages, recognition_kwargs=kw)
    texts = [[t for t, _ in g] for g in res]
    assert all(t == "" or pat.fullmatch(t) for g in texts for t in g) and any(t for g in texts for t in g)
    boxes = [[b for _, b in g] for g in res]
    assert rec.recognize_from_boxes(list(pages), boxes, **kw) == texts
    assert rec.recognize_from_boxes(list(pages), boxes, beam_width=8, pattern="[a-z0-9]{1,12}") == texts
    import os
    crops = np.load(os.path.join(os.path.dirname(__file__), "golden", "c3_crops.npz"))["crops"][:64]
    t = torch.from_numpy(np.ascontiguousarray(crops)).cuda()
    x = torch.empty((len(crops), 200, 31), dtype=torch.float16, device="cuda")
    rec.ctx.crops_to_input(t.data_ptr(), len(crops), x.data_ptr(), _stream())
    assert rec.recognize_crops(crops, **kw) == labels_to_text(rec.predict_device(x, **kw).cpu().numpy(), rec.alphabet)
    scored = pipe.recognize(pages, recognition_kwargs=kw, return_scores=True)
    assert [[w[0] for w in g] for g in scored] == texts
    assert all(w[3] == 0.0 for g in scored for w in g if w[0] == "")
    top = pipe.recognize(pages, recognition_kwargs=dict(kw, top_paths=3), return_scores=True)
    assert [[w[0][0] for w in g] for g in top] == texts
    assert all(pat.fullmatch(s) for g in top for w in g for s, c in zip(w[0], w[3]) if c > 0)
    cells = pipe.recognize(pages, recognition_kwargs=kw, return_char_boxes=True)
    assert [[w[0] for w in g] for g in cells] == texts
    assert all(len(w[2]) == len(w[0]) for g in cells for w in g)
    records = pipe.recognize_records(pages, beam_width=8, pattern=pat, scores=True)
    decoded = D._decode_blocks([records.cpu()], 128, rec.alphabet, True)
    assert [[w[0] for w in g] for g in decoded] == texts
    assert _bits(decoded) == _bits(scored)
    sharded = D.recognize_sharded(pipe, pages, beam_width=8, pattern=pat)
    assert [[t for t, _ in g] for g in sharded] == texts
    stream = D.ShardedStream(pipe, beam_width=8, pattern="[a-z0-9]{1,12}")
    assert stream.submit(pages) is None
    assert [[t for t, _ in g] for g in stream.flush()] == texts


def test_rotations_vote_on_the_best_matching_reading(pipe):
    rec = pipe.recognizer
    pat = Pattern("[a-z0-9]{2,8}")
    pages = _pages(1, seed=1001)
    turned = np.ascontiguousarray(np.rot90(pages, 2, axes=(1, 2)))
    from keras_ocr_b200 import tools
    from keras_ocr_b200.recognition import confidences, labels_to_text
    boxes = np.stack([b for _, b in pipe.recognize(turned)[0]]).astype(np.float32)
    flat = torch.from_numpy(tools.rectify_boxes(boxes.copy())).cuda()
    idx = torch.zeros(len(boxes), dtype=torch.int32, device="cuda")
    gray = rec.gray_device(torch.from_numpy(turned).cuda())
    turns = (0, 1, 2, 3)
    labels = torch.empty((4, len(boxes), 1, T), dtype=torch.int32, device="cuda")
    logp = torch.empty((4, len(boxes), 1), dtype=torch.float32, device="cuda")
    for j, t in enumerate(turns):
        crnn_in, _ = rec.warp_device(gray, flat.clone(), idx, turn=t)
        rec._forward(crnn_in, labels[j], logp[j], 8, 1, None, pattern=pat)
    a = logp[:, :, 0].cpu().numpy()
    pick = np.argmax(a, axis=0)                                   # the first of equal values, -inf included
    rows = np.arange(len(boxes))
    res = rec.recognize_from_boxes([turned[0]], [list(boxes)], return_scores=True, beam_width=8, pattern=pat,
                                   rotations=turns, rotation_vote="word")[0]
    assert [t for t, _ in res] == labels_to_text(labels[:, :, 0].cpu().numpy()[pick, rows], rec.alphabet)
    assert np.array_equal(np.array([c for _, c in res], np.float32).view(np.int32), confidences(a[pick, rows]).view(np.int32))
    got = pipe.recognize(turned, recognition_kwargs={"beam_width": 8, "pattern": pat, "rotations": (0, 2),
                                                     "rotation_vote": "page"})
    assert all(t == "" or pat.fullmatch(t) for t, _ in got[0])


def test_invalid_combinations_raise_before_any_launch(pipe):
    from keras_ocr_b200.recognition import CharLM
    rec = pipe.recognizer
    pat = Pattern("[a-z]+")
    pages = _pages(1, seed=1002)
    n0 = pipe.detector.ctx.launch_count() + rec.ctx.launch_count()
    lm = CharLM.fit(["abc", "abd"], rec.alphabet, order=3)
    bad = [{"pattern": pat}, {"pattern": pat, "beam_width": 4, "lexicon": ["abc"]},
           {"pattern": pat, "beam_width": 4, "language_model": lm}, {"pattern": Pattern("a+", "ab"), "beam_width": 4},
           {"pattern": ["[a-z]+"], "beam_width": 4}, {"pattern": pat, "beam_width": 4, "max_windows": 2},
           {"pattern": pat, "beam_width": 4, "top_paths": 5}, {"pattern": "[a-z", "beam_width": 4},
           {"pattern": "a{30}b{30}", "beam_width": 4}]
    for kw in bad:
        with pytest.raises(ValueError):
            pipe.recognize(pages, recognition_kwargs=kw)
        with pytest.raises(ValueError):
            rec.recognize_from_boxes(list(pages), [[np.array([[0, 0], [50, 0], [50, 20], [0, 20]], np.float32)]],
                                     **kw)
    with pytest.raises(ValueError, match="a pattern needs beam search: pass beam_width"):
        rec.recognize_crops(np.zeros((1, 31, 200), np.uint8), pattern=pat)
    with pytest.raises(ValueError):
        pipe.recognize_records(pages, pattern=pat)
    from keras_ocr_b200 import distributed as D
    with pytest.raises(ValueError):
        D.recognize_sharded(pipe, pages, pattern=pat)
    assert pipe.detector.ctx.launch_count() + rec.ctx.launch_count() == n0


def test_the_recognize_stage_does_not_wait_for_the_device(pipe, monkeypatch):
    """With a pattern the recognize stage queues its work without a host synchronisation (torch raises on one in
    sync-debug mode "error")."""
    pat = Pattern("[a-z0-9]{1,8}")
    pat.descriptor(pipe.recognizer.device)                      # uploaded once, before the checked stage
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
    pages = _pages()
    for kw in ({}, {"return_scores": True}):
        pipe.recognize(pages, recognition_kwargs={"beam_width": 8, "pattern": pat}, **kw)
    assert len(calls) == 2


# ------------------------------------------------------------------------------------------ 3. accuracy
FORMATS = {"plate": "[a-z]{3}[0-9]{4}", "invoice": "inv[0-9]{6}",
           "date": "[0-9]{2}(jan|feb|mar|apr|may|jun|jul|aug|sep|oct|nov|dec)[0-9]{4}"}
CODES = "|".join(f"({f})" for f in FORMATS.values())
TEST_SEEDS = (300, 301, 302, 303)   # disjoint from the tuning seeds of scripts/bench_pattern.py (100..103)


def code_words(seed, n):
    """``n`` random codes of the three ``FORMATS``, in turn."""
    import string
    rng = np.random.default_rng(seed)
    lo, dg = string.ascii_lowercase, string.digits
    months = "jan feb mar apr may jun jul aug sep oct nov dec".split()
    out = []
    for i in range(n):
        pick = lambda s, m: "".join(rng.choice(list(s), m))          # noqa: E731
        out.append([pick(lo, 3) + pick(dg, 4), "inv" + pick(dg, 6),
                    pick(dg, 2) + months[int(rng.integers(12))] + pick(dg, 4)][i % 3])
    return out


def code_pages(seeds, severity=None):
    """Degraded pages of codes, rendered and degraded as test_gpu_lm.pseudo_pages renders its words."""
    import cv2
    from tests.test_gpu_lm import SEVERITY, degradation
    severity = SEVERITY if severity is None else severity
    pages, items_all = [], []
    for s in seeds:
        rng = np.random.default_rng(s)
        words = code_words(s, 200)
        page = np.full((768, 768, 3), 255, np.uint8)
        font, scale, thick = cv2.FONT_HERSHEY_SIMPLEX, 0.9, 2
        th = cv2.getTextSize("Ag", font, scale, thick)[0][1]
        items, y, i = [], 30 + th, 0
        while y < 768 - 30:
            x = 30
            while True:
                word = words[i % len(words)]
                wpx = cv2.getTextSize(word, font, scale, thick)[0][0]
                if x + wpx > 768 - 30:
                    break
                cv2.putText(page, word, (x, y), font, scale, (0, 0, 0), thick, cv2.LINE_AA)
                items.append((word, (x + wpx / 2, y - th / 2)))
                x += wpx + 3 * th
                i += 1
            y += int(2.6 * th)
        blur, contrast, noise = degradation(severity)
        page = 255 - (255 - cv2.GaussianBlur(page, (0, 0), blur).astype(np.float32)) * np.float32(contrast)
        page = np.clip(page + rng.normal(0, noise, page.shape), 0, 255).astype(np.uint8)
        pages.append(page)
        items_all.append(items)
    return np.stack(pages), items_all


def test_the_pattern_reads_degraded_code_pages_better(pipe):
    """At ``test_gpu_lm.SEVERITY`` beam search alone misreads codes (0/o, 1/l, 5/s ...); with the alternation of the
    three formats every reading matches one of them, and strictly more codes read exactly, as on the tuning seeds
    (100..103, scripts/bench_pattern.py)."""
    from tests import window_refs as R
    pat = Pattern(CODES)
    pages, items = code_pages(TEST_SEEDS)
    beam = pipe.recognize(pages, recognition_kwargs={"beam_width": 16})
    constrained = pipe.recognize(pages, recognition_kwargs={"beam_width": 16, "pattern": pat})
    n_beam = sum(R.exact_reads(g, it) for g, it in zip(beam, items))
    n_pat = sum(R.exact_reads(g, it) for g, it in zip(constrained, items))
    total = sum(len(it) for it in items)
    empty = sum(t == "" for g in constrained for t, _ in g)
    print(f"degraded code pages: {total} codes; exact reads beam 16 {n_beam}, beam 16 + pattern {n_pat}; "
          f"{empty} words without a matching reading")
    assert all(t == "" or pat.fullmatch(t) for g in constrained for t, _ in g)
    assert n_pat > n_beam                  # strictly more on the tuning seeds too (DESIGN.md section 5)
