"""Text lines on the GPU: b2o_group_lines against the fp64 reference (tests/line_refs.py) bit for bit, its memory
contract, and ``Pipeline.recognize(return_lines=True)`` on rendered pages of known lines."""
import math

import cv2
import numpy as np
import pytest
import torch

from keras_ocr_b200 import _lib, weights as W
from tests import line_refs as R
from tests.test_gpu_memory_contract import ERR_ARG, ERR_WORKSPACE, rejected, run

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(cuda_device):
    return _lib.Context(0)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _params(p):
    p = {**R.DEFAULTS, **p}
    ct = p.pop("cos_tol") if "cos_tol" in p else R.cos_tol(p["angle_tolerance"])
    return ct, p["height_ratio"], p["offset_ratio"], p["gap_ratio"]


def table(groups, max_boxes, fill=np.nan):
    """(n, max_boxes, 4, 2) float32 box table (slots past the count hold ``fill``) and (n,) int32 counts."""
    t = np.full((len(groups), max_boxes, 4, 2), fill, np.float32)
    counts = np.zeros(len(groups), np.int32)
    for i, g in enumerate(groups):
        g = np.asarray(g, np.float32).reshape(-1, 4, 2)
        t[i, :min(len(g), max_boxes)] = g[:max_boxes]
        counts[i] = len(g)
    return t, counts


def run_lines(ctx, groups, max_boxes, **params):
    t, counts = table(groups, max_boxes)
    n = len(groups)
    boxes, cnt = torch.from_numpy(t).cuda(), torch.from_numpy(counts).cuda()
    lc = torch.full((n,), -7, dtype=torch.int32, device="cuda")
    wo = torch.full((n, max_boxes), -7, dtype=torch.int32, device="cuda")
    ls = torch.full((n, max_boxes + 1), -7, dtype=torch.int32, device="cuda")
    lb = torch.full((n, max_boxes, 4, 2), -7.0, dtype=torch.float32, device="cuda")
    nbytes = ctx.lines_workspace_bytes(n, max_boxes)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    ctx.group_lines(boxes.data_ptr(), cnt.data_ptr(), n, max_boxes, *_params(params), lc.data_ptr(), wo.data_ptr(),
                    ls.data_ptr(), lb.data_ptr(), ws.data_ptr(), nbytes, _stream())
    torch.cuda.synchronize()
    return [a.cpu().numpy() for a in (lc, wo, ls, lb)]


def check_against_reference(ctx, groups, max_boxes, **params):
    lc, wo, ls, lb = run_lines(ctx, groups, max_boxes, **params)
    rc, ro, rs, rb = R.csr(groups, max_boxes, **params)
    np.testing.assert_array_equal(lc, rc)
    for i, g in enumerate(groups):
        c, L = min(len(g), max_boxes), int(rc[i])
        np.testing.assert_array_equal(wo[i, :c], ro[i])
        np.testing.assert_array_equal(ls[i, :L + 1], rs[i])
        np.testing.assert_array_equal(lb[i, :L].view(np.uint32), rb[i].view(np.uint32))
        assert (wo[i, c:] == -7).all() and (ls[i, L + 1:] == -7).all() and (lb[i, L:] == -7).all()
    return lc, wo, ls, lb


# ------------------------------------------------------------------------------------------- random layouts
def random_page(rng, count):
    """``count`` boxes: lines at random tilts and sizes with jitter, some in two columns, some upside down, and
    degenerate (zero-width, zero-height, single-point) boxes; shuffled."""
    boxes = []
    while len(boxes) < count:
        tilt = float(rng.choice([0.0, rng.uniform(-40, 40), 90.0, 180.0]))
        h = float(rng.uniform(6, 60))
        x0, y0 = rng.uniform(0, 2000, 2)
        cols = int(rng.integers(1, 3))
        for col in range(cols):
            n = int(rng.integers(1, 9))
            widths = rng.uniform(0.5, 6, n) * h
            for b in R.row(x0 + col * (widths.sum() + 4 * h), y0, widths, h, float(rng.uniform(0.2, 1.6)) * h,
                           angle_deg=tilt, origin=(x0, y0), turn=int(rng.choice([0, 0, 0, 2]))):
                boxes.append(b + rng.normal(0, 0.3, (4, 2)).astype(np.float32))
        if rng.uniform() < 0.2:
            q = R.word_box(*rng.uniform(0, 2000, 2), float(rng.uniform(5, 50)), float(rng.uniform(5, 30)))
            boxes.append([q[[0, 0, 2, 3]], q[[0, 1, 1, 0]], q[[0, 0, 0, 0]]][int(rng.integers(0, 3))])
    boxes = np.stack(boxes[:count]).astype(np.float32) if count else np.zeros((0, 4, 2), np.float32)
    return boxes[rng.permutation(count)]


@pytest.mark.parametrize("seed", range(6))
def test_random_layouts_bit_for_bit(ctx, seed):
    rng = np.random.default_rng(seed)
    groups = [random_page(rng, int(rng.integers(0, 200))) for _ in range(8)]
    params = [{}, {"angle_tolerance": 30, "gap_ratio": 3.0}, {"height_ratio": 1.0, "offset_ratio": 0.25},
              {"angle_tolerance": 90, "height_ratio": 0.1, "offset_ratio": 2.0, "gap_ratio": 0.0}][seed % 4]
    check_against_reference(ctx, groups, 256, **params)


@pytest.mark.parametrize("batch", [1, 8, 300])
def test_batches_and_counts(ctx, batch):
    max_boxes = 512                      # a table the detector's overflow re-run has grown past 256
    rng = np.random.default_rng(batch)
    sizes = [0, 1, 2, 255, 256, max_boxes]
    groups = [random_page(rng, sizes[i % len(sizes)] if batch > 1 else 256) for i in range(batch)]
    if batch == 1:
        groups = [random_page(rng, max_boxes + 40)]          # counts past max_boxes: the first max_boxes words
    check_against_reference(ctx, groups, max_boxes)


def test_8192_words_in_one_image(ctx):
    rng = np.random.default_rng(8192)
    check_against_reference(ctx, [random_page(rng, 8192)], 8192)


def test_alone_equals_in_a_batch(ctx):
    rng = np.random.default_rng(11)
    groups = [random_page(rng, c) for c in (37, 0, 256, 5, 180)]
    batch = run_lines(ctx, groups, 256)
    for i, g in enumerate(groups):
        alone = run_lines(ctx, [g], 256)
        for a, b in zip(alone, batch):
            np.testing.assert_array_equal(a[0].view(np.uint32) if a.dtype == np.float32 else a[0],
                                          b[i].view(np.uint32) if b.dtype == np.float32 else b[i])


# ------------------------------------------------------------------------------------------- thresholds
def _nudge(v, k):
    """v moved by k float32 ulps."""
    v = np.float32(v)
    for _ in range(abs(k)):
        v = np.nextafter(v, np.float32(np.inf if k > 0 else -np.inf))
    return v


def threshold_pairs():
    """(name, boxes of two words, params, linked) with the pair exactly on one threshold or one ulp to either side."""
    h = 16.0
    a = R.word_box(100, 100, 40, h)
    out = []
    for k in (-1, 0, 1):
        # gap: |d . u| - (w_a + w_b) / 2 = gap_ratio * h = 24 exactly at k = 0
        b = R.word_box(100 + 40 + 24, 100, 40, h)
        b[:, 0] = [_nudge(v, k) for v in b[:, 0]]
        out.append((f"gap{k:+d}", [a, b], {}, k <= 0))
        # offset: the centres 0.5 * h = 8 apart across the line at k = 0
        b = R.word_box(150, 108, 40, h)
        b[:, 1] = [_nudge(v, k) for v in b[:, 1]]
        out.append((f"offset{k:+d}", [a, b], {}, k <= 0))
        # height: h_b = height_ratio * h_a at k = 0
        b = R.word_box(150, 100, 40, 8.0)
        b[2:, 1] = [_nudge(v, k) for v in b[2:, 1]]
        b[:, 1] += np.float32(4)              # centred on a's centre line
        out.append((f"height{k:+d}", [a, b], {"offset_ratio": 2.0}, k >= 0))
    # angle: cos_tol exactly the dot product of the two directions, and one double ulp to either side
    b = R.word_box(150, 100, 40, h, angle_deg=10.0, origin=(150, 100))
    f = R.features(np.stack([a, b]))
    dot = float(f["ux"][0] * f["ux"][1] + f["uy"][0] * f["uy"][1])
    for k, ct in ((-1, np.nextafter(dot, -np.inf)), (0, dot), (1, np.nextafter(dot, np.inf))):
        out.append((f"angle{k:+d}", [a, b], {"cos_tol": float(ct)}, k <= 0))
    return out


@pytest.mark.parametrize("name,boxes,params,linked", threshold_pairs(), ids=[t[0] for t in threshold_pairs()])
def test_thresholds_exactly(ctx, name, boxes, params, linked):
    assert bool(R.link_matrix(boxes, **params)[0, 1]) == linked
    lc, *_ = check_against_reference(ctx, [boxes, boxes[::-1]], 4, **params)
    assert list(lc) == [1 if linked else 2] * 2


# ------------------------------------------------------------------------------------------- memory contract
def test_memory_contract(ctx):
    rng = np.random.default_rng(5)
    max_boxes, n = 96, 5
    groups = [random_page(rng, c) for c in (0, 1, 40, 96, 130)]      # the last overflows its table
    t, counts = table(groups, max_boxes)
    boxes, cnt = torch.from_numpy(t).cuda(), torch.from_numpy(counts).cuda()
    rc, ro, rs, rb = R.csr(groups, max_boxes)
    nbytes = ctx.lines_workspace_bytes(n, max_boxes)
    c = [min(len(g), max_boxes) for g in groups]
    bufs = {"lc": (4 * n, "i", True),
            "wo": (4 * n * max_boxes, "i", np.concatenate([np.arange(4 * max_boxes) < 4 * c[i] for i in range(n)])),
            "ls": (4 * n * (max_boxes + 1), "i",
                   np.concatenate([np.arange(4 * (max_boxes + 1)) < 4 * (rc[i] + 1) for i in range(n)])),
            "lb": (32 * n * max_boxes, "f", np.concatenate([np.arange(32 * max_boxes) < 32 * rc[i] for i in range(n)])),
            "ws": (nbytes, "i", None)}
    P = _params({})

    def call(g, ws_bytes=nbytes, bx=boxes.data_ptr()):
        return ctx.lib.b2o_group_lines(ctx.handle, bx, cnt.data_ptr(), n, max_boxes, *P, g["lc"].ptr, g["wo"].ptr,
                                       g["ls"].ptr, g["lb"].ptr, g["ws"].ptr, ws_bytes, _stream())

    got = run(ctx, call, bufs, inputs=(boxes, cnt), launches=3)
    wo = got["wo"].view(np.int32).reshape(n, max_boxes)
    ls = got["ls"].view(np.int32).reshape(n, max_boxes + 1)
    np.testing.assert_array_equal(got["lc"].view(np.int32), rc)
    for i in range(n):
        np.testing.assert_array_equal(wo[i, :c[i]], ro[i])
        np.testing.assert_array_equal(ls[i, :rc[i] + 1], rs[i])
    flat = {k: v[:2] for k, v in bufs.items()}
    rejected(ctx, lambda g: call(g, nbytes - 1), flat, ERR_WORKSPACE, inputs=(boxes, cnt))
    rejected(ctx, lambda g: call(g, bx=None), flat, ERR_ARG, inputs=(boxes, cnt))
    bad = (math.nan,) + P[1:]
    rejected(ctx, lambda g: ctx.lib.b2o_group_lines(ctx.handle, boxes.data_ptr(), cnt.data_ptr(), n, max_boxes, *bad,
                                                    g["lc"].ptr, g["wo"].ptr, g["ls"].ptr, g["lb"].ptr, g["ws"].ptr,
                                                    nbytes, _stream()), flat, ERR_ARG, inputs=(boxes, cnt))
    rejected(ctx, lambda g: ctx.lib.b2o_group_lines(ctx.handle, boxes.data_ptr(), cnt.data_ptr(), 0, max_boxes, *P,
                                                    g["lc"].ptr, g["wo"].ptr, g["ls"].ptr, g["lb"].ptr, g["ws"].ptr,
                                                    nbytes, _stream()), flat, 0, inputs=(boxes, cnt))


# ------------------------------------------------------------------------------------------- the pipeline
@pytest.fixture(scope="module")
def pipe(cuda_device):
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    from keras_ocr_b200.recognition import Recognizer
    return Pipeline(detector=Detector(weights=W.synthetic_craft_weights(3, textlike=True), device=0),
                    recognizer=Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True), device=0), scale=2)


ALPHABET = list("abcdefghijklmnopqrstuvwxyz")


def render_page(seed, layout="column", angle=0, h=512, w=512, scale=0.9, thick=2):
    """A white page of cv2.putText Hershey lines, rotated by ``angle`` degrees (counter-clockwise, cv2's sense) about
    its centre.  Returns (page, words, lines, centres): lines as lists of word indices, in page order; centres (n,2)
    every word's centre in the page's pixels.  Words are 1.4 glyph heights apart: one detector box each, and within
    the gap limit of one line; lines are 3.2 glyph heights apart."""
    rng = np.random.default_rng(seed)
    page = np.full((h, w, 3), 255, np.uint8)
    font = cv2.FONT_HERSHEY_SIMPLEX
    words, lines, centres = [], [], []
    th = cv2.getTextSize("Ag", font, scale, thick)[0][1]

    def line_at(x, y, n, sc, right):
        idx = []
        for _ in range(n):
            word = "".join(rng.choice(ALPHABET, int(rng.integers(6, 9))))
            (tw, t_h), _ = cv2.getTextSize(word, font, sc, thick)
            if x + tw > right:
                break
            cv2.putText(page, word, (int(x), int(y)), font, sc, (0, 0, 0), thick, cv2.LINE_AA)
            idx.append(len(words))
            words.append(word)
            centres.append((x + tw / 2, y - t_h / 2))
            x += tw + int(1.4 * t_h)
        return idx

    pitch = int(3.2 * th)
    y = 40 + th
    if layout == "title":
        lines.append(line_at(40, 40 + 2 * th, 2, 2 * scale, w - 40))
        y = 40 + 2 * th + int(3.5 * th)
    while y < h - 40:
        if layout == "columns":                   # a gutter of 150 px, wider than 1.5 box heights
            lines.append(line_at(30, y, 2, scale, w // 2 - 75))
            lines.append(line_at(w // 2 + 75, y, 2, scale, w - 30))
        else:
            lines.append(line_at(40, y, 4, scale, w - 40))
        y += pitch
    centres = np.array(centres, np.float64)
    if angle % 90 == 0 and angle:
        assert h == w
        page = np.ascontiguousarray(np.rot90(page, angle // 90))
        for _ in range(angle // 90 % 4):          # np.rot90 (counter-clockwise): (x, y) -> (y, w - 1 - x)
            centres = np.stack([centres[:, 1], w - 1 - centres[:, 0]], 1)
    elif angle:                                   # padded first, so that no word leaves the page
        pad = 96
        page = cv2.copyMakeBorder(page, pad, pad, pad, pad, cv2.BORDER_CONSTANT, value=(255, 255, 255))
        centres = centres + pad
        m = cv2.getRotationMatrix2D((w / 2 + pad, h / 2 + pad), angle, 1.0)
        page = cv2.warpAffine(page, m, (w + 2 * pad, h + 2 * pad), flags=cv2.INTER_LINEAR, borderValue=(255, 255, 255))
        centres = centres @ m[:, :2].T + m[:, 2]
    return page, words, [l for l in lines if l], centres


def _inside(box, p):
    return cv2.pointPolygonTest(np.asarray(box, np.float32).reshape(-1, 1, 2), (float(p[0]), float(p[1])), False) >= 0


def word_of_box(result, centres):
    """Rendered word index of every returned word (its box holds exactly one rendered centre), asserting that every
    rendered word is found as exactly one box."""
    found = []
    for w in result:
        inside = [k for k, p in enumerate(centres) if _inside(w[1], p)]
        assert len(inside) == 1, ("a box holds", len(inside), "rendered words")
        found.append(inside[0])
    assert sorted(found) == list(range(len(centres))), "not every rendered word is one box"
    return found


PAGES = {"column": ("column", 0), "columns": ("columns", 0), "title": ("title", 0), "tilt+8": ("column", 8),
         "tilt-8": ("column", -8), "tilt+20": ("column", 20), "tilt-20": ("column", -20)}
TURNED = {"turn180": (180, {"rotations": (0, 2), "rotation_vote": "page", "beam_width": 8}),
          "turn90": (90, {"rotations": (0, 1, 2, 3), "rotation_vote": "page", "beam_width": 8})}
# lines whose text equals the rendered line, per page (of 7 on each, 14 on the two-column page), by the first H100 run
EXPECTED_EXACT = {"column": 7, "columns": 14, "title": 7, "tilt+8": 7, "tilt-8": 6, "tilt+20": 7, "tilt-20": 7,
                  "turn180": 7, "turn90": 7}


def check_page(pipe, page, words, lines, centres, single_column, rec=None):
    plain = pipe.recognize(page[None], recognition_kwargs=rec)[0]
    ids = word_of_box(plain, centres)
    got = pipe.recognize(page[None], recognition_kwargs=rec, return_lines=True)[0]
    # the words of all lines together are the default call's tuples, permuted
    flat = [w for _, _, ws in got for w in ws]
    assert len(flat) == len(plain)
    keyed = {np.asarray(w[1]).tobytes(): w for w in plain}
    for w in flat:
        ref = keyed[np.asarray(w[1]).tobytes()]
        assert w[0] == ref[0]
    rendered_line = {k: li for li, l in enumerate(lines) for k in l}
    got_ids = [[ids[[np.asarray(p[1]).tobytes() for p in plain].index(np.asarray(w[1]).tobytes())] for w in ws]
               for _, _, ws in got]
    # exact membership and word order
    assert sorted(got_ids) == sorted(lines), (got_ids, lines)
    if single_column:
        assert got_ids == lines
    else:
        for l in got_ids:
            assert len({rendered_line[k] for k in l}) == 1
    exact = sum(text == " ".join(words[k] for k in l) for (text, _, _), l in zip(got, got_ids))
    return exact


@pytest.mark.parametrize("name", list(PAGES) + list(TURNED))
def test_rendered_pages(pipe, name):
    if name in PAGES:
        layout, angle = PAGES[name]
        rec = None
    else:
        angle, rec = TURNED[name]
        layout = "column"
    page, words, lines, centres = render_page(sum(map(ord, name)), layout, angle, w=800 if layout == "columns" else 512)
    exact = check_page(pipe, page, words, lines, centres, layout != "columns", rec)
    print(f"{name}: {exact} of {len(lines)} lines read exactly")
    assert exact == EXPECTED_EXACT[name]


def _same_words(a, b):
    """Word tuples equal bit for bit (arrays by bytes)."""
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert len(x) == len(y)
        for u, v in zip(x, y):
            if isinstance(u, np.ndarray):
                assert u.dtype == v.dtype and u.tobytes() == v.tobytes()
            elif isinstance(u, list) and u and isinstance(u[0], np.ndarray):
                assert all(p.tobytes() == q.tobytes() for p, q in zip(u, v))
            else:
                assert u == v or (u != u and v != v)


COMBOS = {"scores": {"return_scores": True},
          "beam": {"recognition_kwargs": {"beam_width": 8, "top_paths": 2}},
          "lexicon": {"recognition_kwargs": {"lexicon": "WORDS"}},
          "rotations": {"recognition_kwargs": {"rotations": (0, 2), "beam_width": 4}},
          "char_boxes": {"return_char_boxes": True, "return_scores": True},
          "polygons": {"return_polygons": True, "return_scores": True}}


@pytest.mark.parametrize("combo", list(COMBOS) + ["inflight"])
def test_lines_permute_the_default_words(pipe, combo):
    pages = [render_page(s, "column", a)[0] for s, a in ((1, 0), (2, 8), (3, -20), (4, 0))]   # 512² and 704²
    kw = dict(COMBOS.get(combo, {}))
    if combo == "lexicon":
        kw["recognition_kwargs"] = {"lexicon": sorted({w for s in (1, 2, 3, 4) for w in render_page(s)[1]})}
    if combo == "inflight":
        pages = pages * 2
        pipe.inflight = 2
    try:
        plain = pipe.recognize(pages, **kw)
        got = pipe.recognize(pages, return_lines=True, **kw)
    finally:
        pipe.inflight = 1
    assert len(got) == len(plain)
    for g, p in zip(got, plain):
        flat = [w for _, _, ws in g for w in ws]
        order = {np.asarray(w[1]).tobytes(): k for k, w in enumerate(p)}
        perm = [order[np.asarray(w[1]).tobytes()] for w in flat]
        assert sorted(perm) == list(range(len(p)))
        _same_words(flat, [p[k] for k in perm])
        for text, box, ws in g:
            assert text == " ".join(w[0][0] if isinstance(w[0], list) else w[0] for w in ws)
            assert box.shape == (4, 2) and box.dtype == np.float32


def test_group_lines_on_host_groups(pipe):
    page, _, lines, centres = render_page(21, "column", 0)
    padded, _ = pipe.prepare_device(page[None])
    batch = padded.cpu().numpy()
    groups = pipe.detector.detect(np.concatenate([batch, np.full_like(batch, 255)]))
    got = pipe.detector.group_lines(groups)
    assert got[1] == []
    ref = R.group_lines(groups[0])
    assert [w.tolist() for _, w in got[0]] == [w.tolist() for _, w in ref]
    for (b, _), (rb, _) in zip(got[0], ref):
        assert b.tobytes() == rb.tobytes()
    assert pipe.detector.group_lines([]) == []


def test_invalid_calls_raise_before_any_launch(pipe):
    from keras_ocr_b200.pipeline import Pipeline

    page = render_page(1)[0][None]
    n0 = pipe.detector.ctx.launch_count() + pipe.recognizer.ctx.launch_count()
    for kw in ({"gap": 1}, {"angle_tolerance": 0}, {"height_ratio": float("nan")}):
        with pytest.raises(ValueError):
            pipe.recognize(page, return_lines=True, line_kwargs=kw)
        with pytest.raises(ValueError):
            pipe.detector.group_lines([np.zeros((1, 4, 2), np.float32)], **kw)

    class Injected:
        def detect(self, images, **kw):
            raise AssertionError("must not run")

        def recognize_from_boxes(self, images, box_groups, **kw):
            raise AssertionError("must not run")

    for other in (Pipeline(detector=Injected(), recognizer=pipe.recognizer, scale=2),
                  Pipeline(detector=pipe.detector, recognizer=Injected(), scale=2)):
        with pytest.raises(NotImplementedError):
            other.recognize(page, return_lines=True)
    assert pipe.detector.ctx.launch_count() + pipe.recognizer.ctx.launch_count() == n0
