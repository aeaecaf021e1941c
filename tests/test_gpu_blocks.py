"""Text blocks on the GPU: b2o_group_blocks against the fp64 reference (tests/block_refs.py) bit for bit, its memory
contract, and ``Pipeline.recognize(return_blocks=True)`` on rendered multi-column pages of known blocks."""
import math

import cv2
import numpy as np
import pytest
import torch

from keras_ocr_b200 import _lib
from tests import block_refs as R
from tests.test_gpu_lines import ALPHABET, COMBOS, _same_words, pipe, word_of_box  # noqa: F401 (pipe: fixture)
from tests.test_gpu_memory_contract import ERR_ARG, ERR_WORKSPACE, rejected, run

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx(cuda_device):
    return _lib.Context(0)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _params(p):
    p = {**R.DEFAULTS, **p}
    return p["row_gap"], p["col_gap"]


def table(pages, max_boxes):
    """The line tables b2o_group_lines would write for ``pages`` (each (boxes (L,4,2), word counts (L,))): (n,)
    line counts, (n, max_boxes + 1) starts and (n, max_boxes, 4, 2) boxes; slots past a count hold NaN / -1."""
    n = len(pages)
    counts = np.zeros(n, np.int32)
    starts = np.full((n, max_boxes + 1), -1, np.int32)
    boxes = np.full((n, max_boxes, 4, 2), np.nan, np.float32)
    for i, (b, s) in enumerate(pages):
        L = min(len(b), max_boxes)
        counts[i] = len(b)
        boxes[i, :L] = b[:L]
        starts[i, :L + 1] = np.concatenate([[0], np.cumsum(s[:L])])
    return counts, starts, boxes


def run_blocks(ctx, pages, max_boxes, **params):
    counts, starts, boxes = (torch.from_numpy(a).cuda() for a in table(pages, max_boxes))
    n = len(pages)
    bc = torch.full((n,), -7, dtype=torch.int32, device="cuda")
    lo = torch.full((n, max_boxes), -7, dtype=torch.int32, device="cuda")
    bs = torch.full((n, max_boxes + 1), -7, dtype=torch.int32, device="cuda")
    bb = torch.full((n, max_boxes, 4, 2), -7.0, dtype=torch.float32, device="cuda")
    nbytes = ctx.blocks_workspace_bytes(n, max_boxes)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    ctx.group_blocks(counts.data_ptr(), starts.data_ptr(), boxes.data_ptr(), n, max_boxes, *_params(params),
                     bc.data_ptr(), lo.data_ptr(), bs.data_ptr(), bb.data_ptr(), ws.data_ptr(), nbytes, _stream())
    torch.cuda.synchronize()
    return [a.cpu().numpy() for a in (bc, lo, bs, bb)]


def check_against_reference(ctx, pages, max_boxes, **params):
    bc, lo, bs, bb = run_blocks(ctx, pages, max_boxes, **params)
    rc, ro, rs, rb = R.csr(pages, max_boxes, **params)
    np.testing.assert_array_equal(bc, rc)
    for i, (b, _) in enumerate(pages):
        L, B = min(len(b), max_boxes), int(rc[i])
        np.testing.assert_array_equal(lo[i, :L], ro[i])
        np.testing.assert_array_equal(bs[i, :B + 1], rs[i])
        np.testing.assert_array_equal(bb[i, :B].view(np.uint32), rb[i].view(np.uint32))
        assert (lo[i, L:] == -7).all() and (bs[i, B + 1:] == -7).all() and (bb[i, B:] == -7).all()
    return bc, lo, bs, bb


# ------------------------------------------------------------------------------------------- random layouts
@pytest.mark.parametrize("seed", range(6))
def test_random_layouts_bit_for_bit(ctx, seed):
    rng = np.random.default_rng(seed)
    pages = [R.random_page(rng, int(rng.integers(0, 200))) for _ in range(8)]
    params = [{}, {"row_gap": 0.5}, {"col_gap": 3.0}, {"row_gap": 4.0, "col_gap": 0.2}][seed % 4]
    check_against_reference(ctx, pages, 256, **params)


@pytest.mark.parametrize("batch", [1, 8, 300])
def test_batches_and_counts(ctx, batch):
    max_boxes = 512
    rng = np.random.default_rng(batch)
    sizes = [0, 1, 2, 255, 256, max_boxes]
    pages = [R.random_page(rng, sizes[i % len(sizes)] if batch > 1 else 256) for i in range(batch)]
    if batch == 1:
        pages = [R.random_page(rng, max_boxes + 40)]        # counts past max_boxes: the first max_boxes lines
    check_against_reference(ctx, pages, max_boxes)


@pytest.mark.parametrize("count", [512, 8192])
def test_many_lines_in_one_image(ctx, count):
    rng = np.random.default_rng(count)
    check_against_reference(ctx, [R.random_page(rng, count, tilt=3.0)], count)


def test_spiral_of_1024_levels(ctx):
    b, s = R.spiral(1030)
    bc, *_ = check_against_reference(ctx, [(b, s)], 1030)
    assert bc[0] == 1030


def test_alone_equals_in_a_batch(ctx):
    rng = np.random.default_rng(11)
    pages = [R.random_page(rng, c) for c in (37, 0, 256, 5, 180)]
    batch = run_blocks(ctx, pages, 256)
    for i, p in enumerate(pages):
        alone = run_blocks(ctx, [p], 256)
        for a, b in zip(alone, batch):
            np.testing.assert_array_equal(a[0].view(np.uint32) if a.dtype == np.float32 else a[0],
                                          b[i].view(np.uint32) if b.dtype == np.float32 else b[i])


# ------------------------------------------------------------------------------------------- memory contract
def test_memory_contract(ctx):
    rng = np.random.default_rng(5)
    max_boxes, n = 96, 5
    pages = [R.random_page(rng, c) for c in (0, 1, 40, 96, 130)]      # the last overflows its table
    counts, starts, boxes = (torch.from_numpy(a).cuda() for a in table(pages, max_boxes))
    rc, ro, rs, rb = R.csr(pages, max_boxes)
    nbytes = ctx.blocks_workspace_bytes(n, max_boxes)
    L = [min(len(b), max_boxes) for b, _ in pages]
    bufs = {"bc": (4 * n, "i", True),
            "lo": (4 * n * max_boxes, "i", np.concatenate([np.arange(4 * max_boxes) < 4 * L[i] for i in range(n)])),
            "bs": (4 * n * (max_boxes + 1), "i",
                   np.concatenate([np.arange(4 * (max_boxes + 1)) < 4 * (rc[i] + 1) for i in range(n)])),
            "bb": (32 * n * max_boxes, "f", np.concatenate([np.arange(32 * max_boxes) < 32 * rc[i] for i in range(n)])),
            "ws": (nbytes, "i", None)}
    P = _params({})
    inputs = (counts, starts, boxes)

    def call(g, ws_bytes=nbytes, lb=boxes.data_ptr(), p=P, nn=n):
        return ctx.lib.b2o_group_blocks(ctx.handle, counts.data_ptr(), starts.data_ptr(), lb, nn, max_boxes, *p,
                                        g["bc"].ptr, g["lo"].ptr, g["bs"].ptr, g["bb"].ptr, g["ws"].ptr, ws_bytes,
                                        _stream())

    got = run(ctx, call, bufs, inputs=inputs, launches=1)
    lo = got["lo"].view(np.int32).reshape(n, max_boxes)
    bs = got["bs"].view(np.int32).reshape(n, max_boxes + 1)
    bb = got["bb"].view(np.uint32).reshape(n, max_boxes, 4, 2)
    np.testing.assert_array_equal(got["bc"].view(np.int32), rc)
    for i in range(n):
        np.testing.assert_array_equal(lo[i, :L[i]], ro[i])
        np.testing.assert_array_equal(bs[i, :rc[i] + 1], rs[i])
        np.testing.assert_array_equal(bb[i, :rc[i]], rb[i].view(np.uint32))
    flat = {k: v[:2] for k, v in bufs.items()}
    rejected(ctx, lambda g: call(g, nbytes - 1), flat, ERR_WORKSPACE, inputs=inputs)
    rejected(ctx, lambda g: call(g, lb=None), flat, ERR_ARG, inputs=inputs)
    for bad in ((math.nan, 1.0), (1.5, math.inf), (0.0, 1.0), (1.5, -1.0)):
        rejected(ctx, lambda g: call(g, p=bad), flat, ERR_ARG, inputs=inputs)
    rejected(ctx, lambda g: call(g, nn=0), flat, 0, inputs=inputs)


# ------------------------------------------------------------------------------------------- the pipeline
# cv2.getTextSize("Ag", FONT_HERSHEY_SIMPLEX, 0.9, 2) is 20 px high, and the detector's word boxes are taller than the
# glyphs, so s is more than a glyph height and a row cut needs a box gap of more than 1.5 of them.  A pitch of 3.5
# glyph heights (70 px) leaves box gaps below that inside a column while every word stays one box (2.6 glyph heights
# merged words of adjacent lines into one box); 10 glyph heights (200 px) from the last baseline of a section to the
# first of the next leave a gap that cuts.
TH = 20
PITCH = 70
SECTION = 200


def render_blocks_page(seed, layout, turn180=False):
    """A white page of cv2.putText Hershey lines in known blocks.  ``layout``: "columns2", "columns3", "title" (a
    title at twice the size over two columns) or "footer" (two columns over a full-width line).  Columns are 280 px
    wide with 150 px gutters, wider than the line linking gap.  Returns (page, words, blocks, centres): blocks in
    reading order, each a list of lines (lists of word indices) in page order; centres (n,2) every word's centre."""
    rng = np.random.default_rng(seed)
    cols = 3 if layout == "columns3" else 2
    colw, gutter, margin = 280, 150, 30
    w = 2 * margin + cols * colw + (cols - 1) * gutter
    rows = 6
    h = 40 + 2 * TH + (rows - 1) * PITCH + SECTION * ((layout == "title") + (layout == "footer")) + 80
    page = np.full((h, w, 3), 255, np.uint8)
    font = cv2.FONT_HERSHEY_SIMPLEX
    words, centres = [], []

    def line_at(x, y, n, sc, right):
        idx = []
        for _ in range(n):
            word = "".join(rng.choice(ALPHABET, int(rng.integers(6, 9))))
            (tw, t_h), _ = cv2.getTextSize(word, font, sc, 2)
            if x + tw > right:
                break
            cv2.putText(page, word, (int(x), int(y)), font, sc, (0, 0, 0), 2, cv2.LINE_AA)
            idx.append(len(words))
            words.append(word)
            centres.append((x + tw / 2, y - t_h / 2))
            x += tw + int(1.4 * t_h)
        return idx

    blocks = []
    y = 40 + 2 * TH
    if layout == "title":
        blocks.append([line_at(margin, y, 2, 1.8, w - margin)])
        y += SECTION
    body = [[] for _ in range(cols)]
    for r in range(rows):
        for c in range(cols):
            x = margin + c * (colw + gutter)
            body[c].append(line_at(x, y + r * PITCH, 2, 0.9, x + colw))
    blocks += [[l for l in col if l] for col in body]
    if layout == "footer":
        blocks.append([line_at(margin, y + (rows - 1) * PITCH + SECTION, 5, 0.9, w - margin)])
    centres = np.array(centres, np.float64)
    if turn180:
        page = np.ascontiguousarray(page[::-1, ::-1])
        centres = np.stack([w - 1 - centres[:, 0], h - 1 - centres[:, 1]], 1)
    return page, words, [[l for l in b if l] for b in blocks if any(b)], centres


PAGES = {"columns2": ("columns2", None), "columns3": ("columns3", None), "title": ("title", None),
         "footer": ("footer", None),
         "columns2-turn180": ("columns2", {"rotations": (0, 2), "rotation_vote": "page", "beam_width": 8})}


def _key(w):
    return np.asarray(w[1]).tobytes()


@pytest.mark.parametrize("name", list(PAGES))
def test_rendered_pages(pipe, name):
    layout, rec = PAGES[name]
    page, words, blocks, centres = render_blocks_page(sum(map(ord, name)), layout, turn180=rec is not None)
    plain = pipe.recognize(page[None], recognition_kwargs=rec)[0]
    ids = word_of_box(plain, centres)
    of_box = {_key(w): ids[k] for k, w in enumerate(plain)}
    got = pipe.recognize(page[None], recognition_kwargs=rec, return_blocks=True)[0]
    # the words of all blocks together are the default call's tuples, permuted
    flat = [w for _, _, ls in got for _, _, ws in ls for w in ws]
    by_key = {_key(w): w for w in plain}
    assert sorted(_key(w) for w in flat) == sorted(by_key)
    _same_words(flat, [by_key[_key(w)] for w in flat])
    # exact blocks, lines and words, in reading order
    got_ids = [[[of_box[_key(w)] for w in ws] for _, _, ws in ls] for _, _, ls in got]
    assert got_ids == blocks, (got_ids, blocks)
    for text, box, ls in got:
        assert text == "\n".join(t for t, _, _ in ls)
        assert box.shape == (4, 2) and box.dtype == np.float32


@pytest.mark.parametrize("combo", list(COMBOS) + ["inflight"])
def test_blocks_partition_the_lines(pipe, combo):
    pages = [render_blocks_page(s, l)[0] for s, l in ((1, "columns2"), (2, "title"), (3, "footer"), (4, "columns2"))]
    kw = dict(COMBOS.get(combo, {}))
    if combo == "lexicon":
        kw["recognition_kwargs"] = {"lexicon": sorted({w for s, l in ((1, "columns2"), (2, "title"), (3, "footer"),
                                                                       (4, "columns2"))
                                                       for w in render_blocks_page(s, l)[1]})}
    if combo == "inflight":
        pages = pages * 2
        pipe.inflight = 2
    try:
        lines = pipe.recognize(pages, return_lines=True, **kw)
        got = pipe.recognize(pages, return_blocks=True, **kw)
    finally:
        pipe.inflight = 1
    assert len(got) == len(lines)
    for g, ls in zip(got, lines):
        index = {_key(l): k for k, l in enumerate(ls)}
        seen = []
        for text, box, members in g:
            idx = [index[_key(l)] for l in members]
            assert idx == sorted(idx)                             # page order inside a block
            for l in members:
                ref = ls[index[_key(l)]]
                assert l[0] == ref[0]
                _same_words(l[2], ref[2])
            assert text == "\n".join(l[0] for l in members)
            assert box.shape == (4, 2) and box.dtype == np.float32
            seen += idx
        assert sorted(seen) == list(range(len(ls)))
        assert len(g) >= 2


def test_group_blocks_on_host_lines(pipe):
    page = render_blocks_page(21, "title")[0]
    padded, _ = pipe.prepare_device(page[None])
    batch = padded.cpu().numpy()
    groups = pipe.detector.detect(np.concatenate([batch, np.full_like(batch, 255)]))
    lines = pipe.detector.group_lines(groups)
    got = pipe.detector.group_blocks(lines)
    assert got[1] == []
    ref = R.group_blocks(np.stack([b for b, _ in lines[0]]), np.array([len(w) for _, w in lines[0]]))
    assert [w.tolist() for _, w in got[0]] == [w.tolist() for _, w in ref]
    for (b, _), (rb, _) in zip(got[0], ref):
        assert b.tobytes() == rb.tobytes()
    assert len(got[0]) == 3
    assert pipe.detector.group_blocks([]) == []


def test_invalid_calls_raise_before_any_launch(pipe):
    from keras_ocr_b200.pipeline import Pipeline

    page = render_blocks_page(1, "columns2")[0][None]
    n0 = pipe.detector.ctx.launch_count() + pipe.recognizer.ctx.launch_count()
    for kw in ({"gap": 1}, {"row_gap": 0}, {"col_gap": float("nan")}, {"row_gap": -1.0}):
        with pytest.raises(ValueError):
            pipe.recognize(page, return_blocks=True, block_kwargs=kw)
        with pytest.raises(ValueError):
            pipe.detector.group_blocks([[(np.zeros((4, 2), np.float32), np.zeros(1, np.int32))]], **kw)
    with pytest.raises(ValueError):
        pipe.recognize(page, return_blocks=True, line_kwargs={"gap_ratio": -1})

    class Injected:
        def detect(self, images, **kw):
            raise AssertionError("must not run")

        def recognize_from_boxes(self, images, box_groups, **kw):
            raise AssertionError("must not run")

    for other in (Pipeline(detector=Injected(), recognizer=pipe.recognizer, scale=2),
                  Pipeline(detector=pipe.detector, recognizer=Injected(), scale=2)):
        with pytest.raises(NotImplementedError):
            other.recognize(page, return_blocks=True)
    assert pipe.detector.ctx.launch_count() + pipe.recognizer.ctx.launch_count() == n0
