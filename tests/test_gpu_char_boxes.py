"""GPU: character positions -- ``b2o_ctc_align`` and ``b2o_char_cells`` alone against tests/align_refs.py, the product
path through the CRNN workspace, the recognizer and pipeline flags, and where the cells fall on the bench pages.

Bound of the alignment.  As in tests/test_gpu_beam.py, the kernel's lp[t,c] is within d_t of the exact value (u = 2^-24,
R_t the step's logit range): d_t = 1.01 (10u + 2u R_t + gamma(K + 8)) + 2u max_c |lp[t,c]|.  A Viterbi score is a sum of
48 such terms along one path, added in fp32 one step at a time (the max over predecessors is exact), each addition
rounding by at most u V with V = sum_t max_c |lp[t,c]| bounding every partial sum.  So every path's fp32 score is
within tau = sum_t d_t + 48 u V of its exact score, the kernel's optimum within tau of the reference's, and the exact
score of the kernel's path at least the reference optimum - 2 tau.  Where every decision on the reference's backtrace
wins by more than 2 tau (``align_refs.viterbi``'s margin), the kernel makes the same decisions: the spans are identical.
"""
import os

import cv2
import numpy as np
import pytest
import torch

import bench
from keras_ocr_b200 import _lib, weights as W
from keras_ocr_b200.detection import Detector
from keras_ocr_b200.pipeline import Pipeline
from keras_ocr_b200.recognition import Lexicon, Recognizer
from tests import align_refs as AR
from tests import beam_refs as BR
from tests import image_refs as IR
from tests import rotation_refs as RR
from tests.test_gpu_beam import crafted
from tests.test_rotation_refs import rot90_points

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
T = 48
N_PAGES = 4


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def tau(logits):
    lg = np.asarray(logits, np.float64)
    lp = BR.log_probs(lg)
    k = lg.shape[-1]
    d = 1.01 * (10 * U + 2 * U * (lg.max(-1) - lg.min(-1)) + (k + 8) * U / (1 - (k + 8) * U)) + 2 * U * np.abs(lp).max(-1)
    v = np.abs(lp).max(-1).sum(-1)
    return d.sum(-1) + T * U * v


@pytest.fixture(scope="module")
def ctx(cuda_device):
    c = _lib.Context(0)
    yield c
    c.close()


def align(ctx, logits, labels):
    b, p = labels.shape[:2]
    spans = torch.full((b, p, T, 2), -7, dtype=torch.int32, device="cuda")
    logp = torch.full((b, p), 3.0, dtype=torch.float32, device="cuda")
    x, lab = _dev(logits.astype(np.float32)), _dev(labels)      # alive until the kernel has run
    ctx.ctc_align(x.data_ptr(), b, logits.shape[2], lab.data_ptr(), p, spans.data_ptr(), logp.data_ptr(), _stream())
    return spans.cpu().numpy(), logp.cpu().numpy()


def readings(logits, p, rng):
    """(b, p, 48) int32: the greedy collapse first, then random readings (doubled letters, empty ones, lengths up to 30),
    one that needs more than 48 steps and one with the blank as a label."""
    b, _, k = logits.shape
    out = np.full((b, p, T), -1, np.int32)
    for i in range(b):
        g, _ = AR.greedy_runs(BR.log_probs(logits[i]))
        out[i, 0, :len(g)] = g
        for j in range(1, p):
            kind = j % 9
            if kind == 1:
                seq = [int(rng.integers(k - 1))] * 25 if i % 2 else []       # unalignable, or empty
            elif kind == 2 and k > 2:
                seq = [k - 1, 0]                                            # the blank is not a label
            elif kind == 3:
                c = int(rng.integers(k - 1))
                seq = [c, c, c]
            else:
                seq = rng.integers(0, k - 1, int(rng.integers(1, 31))).tolist()
            out[i, j, :len(seq)] = seq
    return out


def path_score(lp, labels, spans):
    """Exact score of the alignment that ``spans`` describe: each character on its steps, blank elsewhere."""
    blank = lp.shape[1] - 1
    cls = np.full(T, blank)
    for c, (f, l) in zip(labels, spans):
        cls[f:l + 1] = c
    return float(lp[np.arange(T), cls].sum())


def check_align(logits, labels, spans, logp):
    taus, lps = tau(logits), BR.log_probs(logits)
    worst, near, same = 0.0, 0, 0
    for i in range(len(logits)):
        for j in range(labels.shape[1]):
            seq = [int(c) for c in labels[i, j] if c >= 0]
            ref, ref_spans, margin = AR.viterbi(lps[i], seq)
            if not np.isfinite(ref):
                assert logp[i, j] == -np.inf and (spans[i, j] == -1).all(), (i, j)
                continue
            n = len(seq)
            assert (spans[i, j, n:] == -1).all() and (spans[i, j, :n] >= 0).all()
            assert abs(float(logp[i, j]) - ref) <= taus[i], (i, j, logp[i, j], ref, taus[i])
            if n:
                assert path_score(lps[i], seq, spans[i, j, :n]) >= ref - 2 * taus[i], (i, j)
            worst = max(worst, abs(float(logp[i, j]) - ref) / taus[i])
            if margin > 2 * taus[i]:
                assert np.array_equal(spans[i, j, :n], ref_spans), (i, j, spans[i, j, :n], ref_spans)
                same += 1
            else:
                near += 1
    return worst, near, same


# ------------------------------------------------------------------------------------------ 1. the alignment alone
@pytest.mark.parametrize("k", [3, 37, 301, 1024])
def test_align_vs_fp64(ctx, k):
    rng = np.random.default_rng(k)
    report = []
    for p in (1, 9, 128):
        logits = crafted(k, 17 if p < 128 else 6, seed=k + p)
        labels = readings(logits, p, rng)
        spans, logp = align(ctx, logits, labels)
        worst, near, same = check_align(logits, labels, spans, logp)
        report.append(f"P={p}: worst {worst:.3g} of tau, {same} identical, {near} near-tie readings")
        for b in (1, 7):                                          # a crop aligns alike alone and in any batch
            sb, lb = align(ctx, logits[:b], labels[:b])
            assert np.array_equal(sb, spans[:b]) and np.array_equal(lb.view(np.int32), logp[:b].view(np.int32))
        s2, l2 = align(ctx, logits, labels)                       # and on every run
        assert np.array_equal(s2, spans) and np.array_equal(l2.view(np.int32), logp.view(np.int32))
    print(f"align K={k}: " + "; ".join(report))


def test_align_rejects_bad_arguments(ctx):
    x = torch.zeros((2, T, 37), dtype=torch.float32, device="cuda")
    lab = torch.full((2, 129, T), -1, dtype=torch.int32, device="cuda")
    sp = torch.empty((2, 129, T, 2), dtype=torch.int32, device="cuda")
    for b, k, p in [(2, 1, 1), (2, 1025, 1), (2, 37, 0), (2, 37, 129), (-1, 37, 1)]:
        with pytest.raises(_lib.B2OError):
            ctx.ctc_align(x.data_ptr(), b, k, lab.data_ptr(), p, sp.data_ptr(), None, _stream())


# ------------------------------------------------------------------------------------------ 2. the cells alone
THETAS = {"identity": np.array([1, 0, 0, 0, 1, 0], np.float32), "sheared": np.array([0.9, 0.2, 0.05, 0.1, 0.85, -0.08],
          np.float32), "time_flipped": np.array([1, 0, 0, 0, -1, 0], np.float32), "stn_off": None}


def random_spans(rng, b, p):
    out = np.full((b, p, T, 2), -1, np.int32)
    for i in range(b):
        for j in range(p):
            n = int(rng.integers(0, 13))
            steps = np.sort(rng.choice(T, 2 * n, replace=False)) if n else np.zeros(0, int)
            out[i, j, :n] = steps.reshape(n, 2)
    return out


@pytest.mark.parametrize("theta_name", list(THETAS))
@pytest.mark.parametrize("group", IR.warp_cases(), ids=[g["name"] for g in IR.warp_cases()])
def test_cells_vs_fp64(ctx, group, theta_name):
    rng = np.random.default_rng(len(group["quads"]))
    quads = group["quads"]
    b, p = len(quads), 2
    spans = random_spans(rng, b, p)
    th = THETAS[theta_name]
    theta = None if th is None else np.repeat(th[None], b, 0) + (rng.normal(0, 0.02, (b, 6)).astype(np.float32)
                                                                if theta_name == "sheared" else 0)
    spans_t, quads_t = _dev(spans), _dev(quads)
    theta_t = None if theta is None else _dev(theta.astype(np.float32))
    for turn in range(4):
        turns_t = _dev(np.full(b, turn, np.int32))
        cells = torch.full((b, p, T, 4, 2), 5.0, dtype=torch.float32, device="cuda")
        ctx.char_cells(spans_t.data_ptr(), b, p, None if theta_t is None else theta_t.data_ptr(), quads_t.data_ptr(),
                       turns_t.data_ptr(), cells.data_ptr(), _stream())
        got = cells.cpu().numpy()
        for i in range(b):
            for j in range(p):
                n = int((spans[i, j, :, 0] >= 0).sum())
                ref = AR.cells(spans[i, j, :n], None if theta is None else theta[i], quads[i], turn)
                assert np.isnan(got[i, j, n:]).all()
                if np.isnan(ref).all():
                    assert np.isnan(got[i, j, :n]).all(), (i, j)
                    continue
                ulp = np.spacing(np.abs(ref).astype(np.float32))
                assert (np.abs(got[i, j, :n] - ref) <= ulp).all(), (turn, i, j, got[i, j, :n], ref)
                if n:
                    box = AR.plan(quads[i], turn)[0]
                    assert np.array_equal(got[i, j, 0, [0, 3]], box[[0, 3]])
                    assert np.array_equal(got[i, j, n - 1, [1, 2]], box[[1, 2]])
    # the crop frame: no box
    cells = torch.empty((b, p, T, 4, 2), dtype=torch.float32, device="cuda")
    ctx.char_cells(spans_t.data_ptr(), b, p, None if theta_t is None else theta_t.data_ptr(), None, None,
                   cells.data_ptr(), _stream())
    got = cells.cpu().numpy()
    for i in range(b):
        n = int((spans[i, 0, :, 0] >= 0).sum())
        ref = AR.cells(spans[i, 0, :n], None if theta is None else theta[i])
        assert np.array_equal(got[i, 0, :n], ref)


# ------------------------------------------------------------------------------------------ 3. the product path
def _input(rec, crops):
    t = torch.from_numpy(np.ascontiguousarray(crops)).to(rec.device)
    x = torch.empty((len(crops), 200, 31), dtype=torch.float16, device=rec.device)
    rec.ctx.crops_to_input(t.data_ptr(), len(crops), x.data_ptr(), _stream())
    return x


@pytest.mark.parametrize("decoder", ["greedy", "beam", "lexicon"])
def test_workspace_entry_equals_standalone(cuda_device, ctx, golden_dir, decoder):
    g = np.load(os.path.join(golden_dir, "c3_crops.npz"))
    rec = Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True))
    rec.keep_workspace = True
    x = _input(rec, g["crops"])
    kw = {"greedy": {}, "beam": {"beam_width": 10, "top_paths": 3},
          "lexicon": {"lexicon": Lexicon(["hello", "world", "text", "abc", "zz"] + [f"w{i}" for i in range(50)])}}[decoder]
    labels, logp, spans, theta = rec._predict_aligned(x, kw.get("beam_width"), kw.get("top_paths", 1), kw.get("lexicon"))
    logits = rec.tap("logits", (len(x), T, 37), torch.float32).cpu().numpy()
    theta_tap = rec.tap("theta", (len(x), 6), torch.float32)
    plain = rec.predict_device(x, with_scores=True, **kw)         # the decoder's outputs do not change
    p = labels.shape[1]
    assert np.array_equal(plain[0].cpu().numpy().reshape(labels.shape), labels.cpu().numpy())
    assert np.array_equal(plain[1].cpu().numpy().reshape(logp.shape), logp.cpu().numpy())
    sd, _ = align(ctx, logits, labels.cpu().numpy())
    assert np.array_equal(sd, spans.cpu().numpy()) and torch.equal(theta, theta_tap)
    if decoder == "greedy":                                       # the argmax runs, except at exact ties
        lps, ties = BR.log_probs(logits), 0
        for i in range(len(x)):
            lab, runs = AR.greedy_runs(lps[i])
            assert lab == [int(c) for c in labels[i, 0].cpu().numpy() if c >= 0]
            if not np.array_equal(spans[i, 0, :len(lab)].cpu().numpy(), runs):
                ties += 1
                assert AR.viterbi(lps[i], lab)[2] <= 2 * tau(logits[i:i + 1])[0], i
        print(f"C3 greedy: spans == argmax runs on {len(x) - ties}/{len(x)} crops, {ties} (near-)ties")
    cells = rec.char_cells_device(spans, theta)
    ref = torch.empty_like(cells)
    ctx.char_cells(spans.data_ptr(), len(x), p, theta_tap.data_ptr(), None, None, ref.data_ptr(), _stream())
    assert torch.equal(torch.nan_to_num(cells, 99.0), torch.nan_to_num(ref, 99.0))
    words = rec.recognize_crops(g["crops"][:9], return_scores=True, return_char_boxes=True, **kw)
    for w, text in zip(words, rec.recognize_crops(g["crops"][:9], return_scores=True, **kw)):
        assert w[:2] == text
        texts, boxes = (w[0], w[2]) if p > 1 else ([w[0]], [w[2]])
        assert all(q.shape == (len(t), 4, 2) and q.dtype == np.float32 for t, q in zip(texts, boxes))


@pytest.fixture(scope="module")
def pipe(cuda_device):
    det = Detector(weights=W.synthetic_craft_weights(3, textlike=True), device=0)
    rec = Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True), device=0)
    return Pipeline(detector=det, recognizer=rec, scale=bench.SCALE, max_size=2048)


@pytest.fixture(scope="module")
def pages():
    p, words, rects = bench.make_pages(0, with_layout=True)
    return p[:N_PAGES], words[:N_PAGES], rects[:N_PAGES]


def _bits(result):
    return [[(t, np.asarray(b).view(np.int32).tolist()) + tuple(np.float32(s).view(np.int32).tolist() for s in rest)
             for t, b, *rest in g] for g in result]


KWARGS = {"greedy": {}, "beam10_p3": {"beam_width": 10, "top_paths": 3},
          "lexicon": {"lexicon": None}, "rot0123_word_beam": {"rotations": (0, 1, 2, 3), "rotation_vote": "word",
                                                             "beam_width": 10},
          "rot0123_page_beam": {"rotations": (0, 1, 2, 3), "rotation_vote": "page", "beam_width": 10}}


@pytest.mark.parametrize("name", list(KWARGS))
def test_flag_changes_nothing_else(pipe, pages, name):
    imgs, words, _ = pages
    kw = dict(KWARGS[name])
    if "lexicon" in kw:
        kw["lexicon"] = Lexicon(sorted({w for page in words for w in page}), pipe.recognizer.alphabet)
    plain = pipe.recognize(imgs, recognition_kwargs=kw, return_scores=True)
    with_cells = pipe.recognize(imgs, recognition_kwargs=kw, return_scores=True, return_char_boxes=True)
    assert [len(g) for g in with_cells] == [len(g) for g in plain]
    stripped = [[w[:4] for w in g] for g in with_cells]
    for g, gp in zip(stripped, plain):                           # texts, boxes, detection scores, confidences
        for a, b in zip(g, gp):
            assert a[0] == b[0] and np.array_equal(np.asarray(a[1]).view(np.int32), np.asarray(b[1]).view(np.int32))
            assert np.float32(a[2]) == np.float32(b[2]) and np.array_equal(np.float32(a[3]), np.float32(b[3]))
    for g in with_cells:
        for text, box, _, _, cells in g:
            texts, cl = (text, cells) if isinstance(text, list) else ([text], [cells])
            # outer edges: the corners the word was cut from -- the returned box as it is with rotations (rolled to the
            # chosen turn), else in warpBox's order
            edge = np.asarray(box) if "rotations" in kw else RR.turned_box(np.asarray(box), 0)
            for t, q in zip(texts, cl):
                assert q.shape == (len(t), 4, 2) and q.dtype == np.float32
                if len(t):
                    assert np.array_equal(q[0, [0, 3]], edge[[0, 3]]), (name, t)
                    assert np.array_equal(q[-1, [1, 2]], edge[[1, 2]]), (name, t)
    simple = pipe.recognize(imgs, recognition_kwargs=kw, return_char_boxes=True)
    assert [[w[0] for w in g] for g in simple] == [[w[0] for w in g] for g in plain]


def test_injected_models_raise(pipe):
    class Other:
        def detect(self, images, **kw):
            return [[] for _ in images]
    p = Pipeline(detector=Other(), recognizer=pipe.recognizer)
    with pytest.raises(NotImplementedError):
        p.recognize([np.zeros((64, 64, 3), np.uint8)], return_char_boxes=True)


# ------------------------------------------------------------------------------------------ 4. on the bench pages
def char_intervals(word, rect, h=bench.PAGE_H, w=bench.PAGE_W, n_words=bench.WORDS_PER_PAGE):
    """Every rendered character's x interval: the word's glyph rectangle divided in proportion to the cv2.getTextSize
    advances of the word's prefixes, at the font scale oracle.synth.text_image drew it with."""
    cols = max(1, int(np.floor(np.sqrt(n_words * w / h / 2.0))))
    rows = int(np.ceil(n_words / cols))
    cell_w, cell_h = w / cols, h / rows
    font = cv2.FONT_HERSHEY_SIMPLEX
    (tw, th), _ = cv2.getTextSize(word, font, 0.9, 2)
    scale = 0.9 * min(0.8 * cell_w / tw, 0.45 * cell_h / th)
    adv = [0] + [cv2.getTextSize(word[:i], font, scale, 2)[0][0] for i in range(1, len(word) + 1)]
    x0, _, x1, _ = rect
    edges = x0 + (x1 - x0) * np.asarray(adv, np.float64) / adv[-1]
    return np.stack([edges[:-1], edges[1:]], 1)


def placement(result, words, rects, unturn=None):
    """(characters of correctly read words, cell centres inside their own interval).  ``unturn`` maps page points back
    upright."""
    total = inside = 0
    for group, page_words, page_rects in zip(result, words, rects):
        for text, box, cells in group:
            box, cells = np.asarray(box, np.float64), np.asarray(cells, np.float64)
            if unturn is not None:
                box, cells = unturn(box), unturn(cells.reshape(-1, 2)).reshape(cells.shape)
            c = box.mean(0)
            hits = [k for k, (x0, y0, x1, y1) in enumerate(page_rects) if x0 <= c[0] <= x1 and y0 <= c[1] <= y1]
            if len(hits) != 1 or page_words[hits[0]] != text:
                continue
            iv = char_intervals(text, page_rects[hits[0]])
            cx = cells.mean(1)[:, 0]
            total += len(text)
            inside += int(((cx >= iv[:, 0]) & (cx <= iv[:, 1])).sum())
    return total, inside


# measured on the first 4 bench pages (DESIGN.md section 2: 0.978, 0.979 and 0.988), minus a margin of 0.05
CELL_BOUND_UPRIGHT, CELL_BOUND_TURNED, SPAN_BOUND_UPRIGHT = 0.928, 0.929, 0.938


def test_cells_on_bench_pages(pipe, pages):
    imgs, words, rects = pages
    res = pipe.recognize(imgs, return_char_boxes=True)
    total, inside = placement(res, words, rects)
    frac_up = inside / total
    # emission-span centres: the greedy spans' centres through the forward's own theta and the word's warp
    rec = pipe.recognizer
    rec.keep_workspace = True
    dev = rec.recognize_from_boxes_device
    st = pipe._stage_detect(imgs, None, {})
    bst = st["boxes_state"]
    boxes, counts = pipe.detector.boxes_finish(bst)
    labels, spans, cells = dev(st["batch"], boxes, counts, gray=st["gray"], flat=bst["flat"],
                               image_index=bst["image_index"], char_boxes=True)
    theta = rec.tap("theta", (labels.shape[0], 6), torch.float32).cpu().numpy()
    rec.keep_workspace = False
    flat, spans = bst["flat"][:labels.shape[0]].cpu().numpy(), spans.cpu().numpy()
    span_total = span_inside = 0
    k = 0
    boxes_h = boxes.cpu().numpy()
    for i, (page_words, page_rects) in enumerate(zip(words, rects)):
        for slot in range(int(counts[i])):
            text, _ = res[i][slot][:2]
            box_p = boxes_h[i, slot] / pipe._plans(imgs)[i][0]
            c = box_p.mean(0)
            hits = [j for j, (x0, y0, x1, y1) in enumerate(page_rects) if x0 <= c[0] <= x1 and y0 <= c[1] <= y1]
            if len(hits) == 1 and page_words[hits[0]] == text and len(text):
                iv = char_intervals(text, page_rects[hits[0]])
                _, m, _, sh = AR.plan(flat[k], 0)
                for j in range(len(text)):
                    f, l = spans[k, j]
                    r = 0.5 * (f + l) + 2
                    u = 0.5 * (theta[k, 4] * (-1 + 2 * r / 49) + theta[k, 5] + 1) * 50
                    x, y = 4 * u + 1.5, sh / 2
                    px = ((m[0] * x + m[1] * y + m[2]) / (m[6] * x + m[7] * y + m[8])) / pipe._plans(imgs)[i][0]
                    span_total += 1
                    span_inside += int(iv[j, 0] <= px <= iv[j, 1])
            k += 1
    frac_span = span_inside / span_total
    # the pages turned by np.rot90, read with every turn, mapped back upright
    turned_total = turned_inside = 0
    kw = {"rotations": (0, 1, 2, 3), "rotation_vote": "page", "beam_width": 10}
    h, w = imgs.shape[1:3]
    for kk in (1, 2, 3):
        timgs = np.ascontiguousarray(np.rot90(imgs, kk, axes=(1, 2)))
        res_t = pipe.recognize(timgs, recognition_kwargs=kw, return_char_boxes=True)
        dims = (w, h) if kk % 2 else (h, w)
        t, ins = placement(res_t, words, rects, unturn=lambda q: rot90_points(q, (4 - kk) % 4, *dims).astype(np.float64))
        turned_total += t
        turned_inside += ins
    frac_turned = turned_inside / turned_total
    print(f"bench pages: cell centre inside its character {inside}/{total} = {frac_up:.3f} upright, "
          f"{turned_inside}/{turned_total} = {frac_turned:.3f} turned (rot90 k=1..3, beam 10, page vote); "
          f"emission-span centre {span_inside}/{span_total} = {frac_span:.3f} upright")
    assert total > 100 and turned_total > 300
    assert frac_up >= CELL_BOUND_UPRIGHT and frac_turned >= CELL_BOUND_TURNED and frac_span >= SPAN_BOUND_UPRIGHT
