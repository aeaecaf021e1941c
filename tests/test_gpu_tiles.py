"""Tiled detection (DESIGN.md section 1, "Tiles") on the GPU.

* b2o_cut_tiles and b2o_stitch_tiles equal tests/tile_refs.py bit for bit, chunk by chunk, and keep their memory
  contracts (tests/test_gpu_memory_contract.py's ``run`` / ``rejected``);
* ``predict_device(tile_size=...)`` equals the NumPy stitch of CRAFT run on the NumPy-cut tiles, whatever the chunk;
* a batch that fits takes the whole-page path: the same results and launches;
* getBoxes on maps taller than 1024 rows against the oracle (tests/test_gpu_boxes.py's checks);
* tile_size is validated before any launch, the detect stage waits on nothing, ``inflight`` changes nothing;
* end to end, large pages read more words tiled than shrunk to 2048, and a word across a seam is one box.
"""
import collections

import cv2
import numpy as np
import pytest
import torch

from keras_ocr_b200 import _lib, detection, weights as W
from oracle import synth
from tests import tile_refs as TR
from tests.test_gpu_boxes import check_image, run_boxes
from tests.test_gpu_memory_contract import ERR_ARG, rejected, rows, run

pytestmark = pytest.mark.gpu

TILE = 512


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _plan(hp, wp, t=TILE, m=detection.TILE_MARGIN):
    return _lib.tile_plan(hp, wp, t, m), TR.plan(hp, wp, t, m)


@pytest.fixture(scope="module")
def ctx(cuda_device):
    return _lib.Context(0)


@pytest.fixture(scope="module")
def det(cuda_device):
    return detection.Detector(weights=W.synthetic_craft_weights(3, textlike=True), device=0)


@pytest.fixture(scope="module")
def rec(cuda_device):
    from keras_ocr_b200.recognition import Recognizer
    return Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True), device=0)


def _pipe(det, rec, **kw):
    from keras_ocr_b200.pipeline import Pipeline
    return Pipeline(detector=det, recognizer=rec, scale=kw.pop("scale", 2), **kw)


# ------------------------------------------------------------------------------------------ cut and stitch kernels
@pytest.mark.parametrize("shape", [(2, 1100, 700), (1, 1536, 1536), (3, 520, 1300), (1, 1001, 613)])
def test_cut_matches_reference_in_chunks(ctx, shape):
    n, hp, wp = shape
    plan, ref = _plan(hp, wp)
    img = np.random.default_rng(hp).integers(0, 255, (n, hp, wp, 3), dtype=np.uint8)
    dev = torch.from_numpy(img).cuda()
    total = n * plan.n_h * plan.n_w
    tile_bytes = plan.t_h * plan.t_w * 3
    expect = TR.cut(img, ref).reshape(-1)
    for first, count in ((0, total), (0, 1), (1, min(3, total - 1)), (total - 1, 1)):
        if count < 1:
            continue
        keep = [first <= j < first + count for j in range(total)]
        out = run(ctx, lambda g: ctx.lib.b2o_cut_tiles(ctx.handle, dev.data_ptr(), n, plan, first, count,
                                                        g["tiles"].ptr + first * tile_bytes, _stream()),
                  {"tiles": (total * tile_bytes, "i", rows(total, tile_bytes, keep))}, [dev], float_runs=False)
        sl = slice(first * tile_bytes, (first + count) * tile_bytes)
        assert np.array_equal(out["tiles"][sl], expect[sl])


def test_stitch_matches_reference_in_chunks(ctx):
    n, hp, wp = 2, 1100, 700
    plan, ref = _plan(hp, wp)
    total = n * plan.n_h * plan.n_w
    ts = np.random.default_rng(5).standard_normal((total, plan.t_h // 2, plan.t_w // 2, 2)).astype(np.float32)
    dev = torch.from_numpy(ts).cuda()
    page = n * (hp // 2) * (wp // 2) * 8
    tsz = (plan.t_h // 2) * (plan.t_w // 2) * 2
    whole = TR.stitch(ts, ref, n)
    assert not np.isnan(whole).any()                       # the cores cover every score of the page

    def chunks(g, size):
        for first in range(0, total, size):
            k = min(size, total - first)
            rc = ctx.lib.b2o_stitch_tiles(ctx.handle, dev.data_ptr() + first * tsz * 4, n, plan, first, k, g["s"].ptr,
                                          _stream())
            if rc:
                return rc
        return 0

    for size in (1, 3, total):
        out = run(ctx, lambda g: chunks(g, size), {"s": (page, "f", True)}, [dev])
        assert np.array_equal(out["s"].view(np.float32).reshape(whole.shape), whole)
    # one chunk writes exactly its tiles' cores and nothing else
    first, k = 2, 3
    mask = ~np.isnan(TR.stitch(ts[first:first + k], ref, n, first=first))
    out = run(ctx, lambda g: ctx.lib.b2o_stitch_tiles(ctx.handle, dev.data_ptr() + first * tsz * 4, n, plan, first, k,
                                                      g["s"].ptr, _stream()),
              {"s": (page, "f", np.repeat(mask.reshape(-1), 4))}, [dev])
    assert np.array_equal(out["s"].view(np.float32).reshape(whole.shape)[mask], whole[mask])


def test_cut_and_stitch_reject_bad_arguments(ctx):
    n, hp, wp = 1, 1100, 700
    plan, _ = _plan(hp, wp)
    img = torch.zeros((n, hp, wp, 3), dtype=torch.uint8, device="cuda")
    total = n * plan.n_h * plan.n_w
    tb = plan.t_h * plan.t_w * 3
    sb = (plan.t_h // 2) * (plan.t_w // 2) * 8
    ts = torch.zeros(total * sb, dtype=torch.uint8, device="cuda")
    bad = _lib.TilePlan.from_buffer_copy(plan)
    bad.n_w += 1
    cases = [(plan, 0, 0, 0), (plan, total, 1, 0), (plan, -1, 1, 0), (plan, 0, total + 1, 0), (bad, 0, 1, 0),
             (plan, 0, 1, 1)]                                # the last: a misaligned output
    for p, first, k, skew in cases:
        rejected(ctx, lambda g: ctx.lib.b2o_cut_tiles(ctx.handle, img.data_ptr(), n, p, first, k, g["t"].ptr + skew,
                                                      _stream()), {"t": (total * tb + 16, "i")}, ERR_ARG, [img])
        rejected(ctx, lambda g: ctx.lib.b2o_stitch_tiles(ctx.handle, ts.data_ptr(), n, p, first, k, g["s"].ptr + skew,
                                                         _stream()), {"s": (n * (hp // 2) * (wp // 2) * 8 + 16, "f")},
                 ERR_ARG, [ts])
    rejected(ctx, lambda g: ctx.lib.b2o_cut_tiles(ctx.handle, img.data_ptr(), 0, plan, 0, 1, g["t"].ptr, _stream()),
             {"t": (tb, "i")}, ERR_ARG, [img])


# ------------------------------------------------------------------------------------------ the tiled forward
def test_tiled_forward_equals_stitch_of_tile_forwards(det, monkeypatch):
    n, hp, wp = 2, 1100, 700
    pages = np.random.default_rng(3).integers(0, 255, (n, hp, wp, 3), dtype=np.uint8)
    pages[:, 200:600, 100:500] = 255
    dev = torch.from_numpy(pages).cuda()
    plan, ref = _plan(hp, wp)
    tiles = TR.cut(pages, ref)
    per_tile = det.predict_device(torch.from_numpy(tiles).cuda()).cpu().numpy()
    expect = TR.stitch(per_tile, ref, n)
    got = det.predict_device(dev, tile_size=TILE).cpu().numpy()
    assert np.array_equal(got, expect)
    total = tiles.shape[0]
    for chunk in (1, 3, total):
        monkeypatch.setattr(detection, "TILE_CHUNK_PIXELS", chunk * plan.t_h * plan.t_w)
        assert np.array_equal(det.predict_device(dev, tile_size=TILE).cpu().numpy(), expect), chunk
    # a batch that fits one tile is the whole-page forward
    small = dev[:, :TILE, :TILE].contiguous()
    assert np.array_equal(det.predict_device(small, tile_size=TILE).cpu().numpy(), det.predict_device(small).cpu().numpy())


def _launches(pipe):
    return pipe.detector.ctx.launch_count() + pipe.recognizer.ctx.launch_count()


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert len(x) == len(y)
        for u, v in zip(x, y):
            assert repr(u) == repr(v)


@pytest.mark.parametrize("size,max_size", [((768, 768), 2048), ((1675, 2048), 2048), ((1024, 3072), 3072)])
def test_pages_that_fit_take_the_whole_page_path(det, rec, monkeypatch, size, max_size):
    h, w = size
    pages, _ = synth.text_images(seed=h, n=2, h=h, w=w, n_words=24)
    pipe = _pipe(det, rec, max_size=max_size)
    for kw in ({"return_scores": True}, {"return_lines": True}, {"recognition_kwargs": {"max_windows": 4}}):
        n0 = _launches(pipe)
        got = pipe.recognize(pages, **kw)
        n_got = _launches(pipe) - n0
        with monkeypatch.context() as m:
            orig = det.predict_device
            m.setattr(det, "predict_device", lambda b, tile_size=None, margin=None: orig(b, tile_size=None))
            n0 = _launches(pipe)
            ref = pipe.recognize(pages, **kw)
            n_ref = _launches(pipe) - n0
        _same(got, ref)
        assert n_got == n_ref


# ------------------------------------------------------------------------------------------ getBoxes on tall maps
def _bar(scores, y0, y1, x0, width, slant):
    """A slanted text bar from row y0 to y1 (x0 + slant * (y - y0) its left edge), text 0.95, no link."""
    for y in range(y0, y1):
        x = int(x0 + slant * (y - y0))
        scores[y, x:x + width, 0] = 0.95


def _tall_maps():
    cases = []
    s = np.zeros((1025, 192, 2), np.float32)
    _bar(s, 2, 1022, 40, 14, 0.05)                           # ROI of all 1025 rows
    _bar(s, 100, 140, 120, 40, 0.0)
    cases.append(("rows1025", s[None], 16))
    s = np.zeros((1536, 320, 2), np.float32)
    _bar(s, 10, 1400, 20, 12, 0.1)                           # > 1024 ROI rows
    _bar(s, 30, 1300, 200, 10, -0.05)
    _bar(s, 1450, 1500, 100, 80, 0.0)
    cases.append(("rows1536", s[None], 16))
    s = np.zeros((2, 4096, 256, 2), np.float32)
    for i in range(2):
        _bar(s[i], 5, 4000, 10, 10, 0.04)                    # > 1754 rows: the hull stack leaves shared memory
        _bar(s[i], 50, 2100, 120, 12, -0.03 * (i + 1))
        _bar(s[i], 2200, 3900, 200, 8, 0.0)
        _bar(s[i], 1200, 2600, 80, 6, 0.01)                  # four big components per image share the lock
        for k in range(6):
            s[i, 100 + 600 * k:120 + 600 * k, 160:220] = (0.9, 0.0)
    cases.append(("rows4096", s, 16))
    return cases


@pytest.mark.parametrize("case", _tall_maps(), ids=lambda c: c[0])
def test_get_boxes_on_tall_maps(ctx, case):
    name, scores, max_boxes = case
    got = run_boxes(ctx, scores, max_boxes)
    for i in range(scores.shape[0]):
        check_image(got, i, scores[i], max_boxes)
    # the polygon stage on the same maps: the same boxes
    n, hs, ws, _ = scores.shape
    t = torch.from_numpy(np.ascontiguousarray(scores)).cuda()
    nbytes = ctx.boxes_workspace_bytes(n, hs, ws, max_boxes)
    wsp = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    boxes = torch.zeros((n, max_boxes, 4, 2), dtype=torch.float32, device="cuda")
    counts = torch.zeros((n,), dtype=torch.int32, device="cuda")
    polys = torch.zeros((n, max_boxes, _lib.POLY_POINTS, 2), dtype=torch.float32, device="cuda")
    points = torch.zeros((n, max_boxes), dtype=torch.int32, device="cuda")
    from tests.test_gpu_boxes import THR
    ctx.get_boxes_poly(t.data_ptr(), n, hs, ws, THR["detection_threshold"], THR["text_threshold"],
                       THR["link_threshold"], THR["size_threshold"], boxes.data_ptr(), counts.data_ptr(), None,
                       polys.data_ptr(), points.data_ptr(), max_boxes, wsp.data_ptr(), nbytes, _stream())
    torch.cuda.synchronize()
    c = counts.cpu().numpy()
    assert np.array_equal(c, got["counts"])
    for i in range(n):
        k = min(int(c[i]), max_boxes)
        assert np.array_equal(boxes.cpu().numpy()[i, :k], got["boxes"][i, :k])
        assert ((points.cpu().numpy()[i, :k] >= 4)).all()


def test_boxes_workspace_grows_only_for_tall_maps(ctx):
    small = ctx.boxes_workspace_bytes(2, 1024, 768, 256)
    assert ctx.boxes_workspace_bytes(2, 1025, 768, 256) > small + 2 * 64 * 1025


# ------------------------------------------------------------------------------------------ Python surface
@pytest.mark.parametrize("bad", [True, 500, 4096, 256.0, "512"])
def test_invalid_tile_size_raises_before_any_launch(det, rec, bad):
    pipe = _pipe(det, rec)
    pages, _ = synth.text_images(seed=1, n=1, h=96, w=128, n_words=2)
    n0 = _launches(pipe)
    with pytest.raises(ValueError):
        pipe.recognize(pages, detection_kwargs={"tile_size": bad})
    with pytest.raises(ValueError):
        pipe.recognize_records(pages, detection_kwargs={"tile_size": bad})
    with pytest.raises(ValueError):
        det.detect(pages, tile_size=bad)
    torch.cuda.synchronize()
    assert _launches(pipe) == n0


def test_craft_refuses_pages_over_the_indexing_bound(det):
    h, w = 2048, (_lib.CRAFT_MAX_PIXELS // 2048) + 32
    img = torch.full((1, h, w, 3), 255, dtype=torch.uint8, device="cuda")
    with pytest.raises(_lib.B2OError, match="tile_size"):
        det.ctx.craft_forward(img.data_ptr(), 1, h, w, img.data_ptr(), img.data_ptr(), 1 << 40, _stream())


def test_tiled_detect_stage_waits_on_nothing(det, rec, monkeypatch):
    pipe = _pipe(det, rec)
    stage = pipe._stage_detect
    calls = []

    def strict(*args, **kw):
        torch.cuda.set_sync_debug_mode("error")
        try:
            return stage(*args, **kw)
        finally:
            torch.cuda.set_sync_debug_mode("default")
            calls.append(1)

    monkeypatch.setattr(pipe, "_stage_detect", strict)
    pages, _ = synth.text_images(seed=1000, n=2, h=768, w=768, n_words=32)
    pipe.recognize(pages, detection_kwargs={"tile_size": TILE})
    pipe.recognize(pages, detection_kwargs={"tile_size": TILE}, return_scores=True)
    assert len(calls) == 2


def test_inflight_changes_nothing_on_tiled_pages(det, rec):
    pages, _ = synth.text_images(seed=7, n=8, h=768, w=768, n_words=32)
    kw = {"detection_kwargs": {"tile_size": TILE}, "return_scores": True}
    _same(_pipe(det, rec, inflight=2).recognize(pages, **kw), _pipe(det, rec).recognize(pages, **kw))


# ------------------------------------------------------------------------------------------ end to end
def _exact(results, truth):
    got = 0
    for words, true in zip(results, truth):
        got += sum((collections.Counter(w[0] for w in words) & collections.Counter(true)).values())
    return got


def test_large_pages_read_more_words_tiled(det, rec):
    pages, truth = synth.text_images(seed=31, n=2, h=3072, w=3072, n_words=512)
    tiled = _exact(_pipe(det, rec, max_size=6144).recognize(pages), truth)
    capped = _exact(_pipe(det, rec).recognize(pages), truth)
    print(f"exact reads on 2 pages of 3072^2 with 512 words: tiled (max_size=6144) {tiled}, capped at 2048 {capped}")
    assert tiled > capped


def test_word_across_every_seam_is_one_box(det):
    # 1408^2 detector input, tiles of 512: three seams on each axis where the cores meet
    page = np.full((1408, 1408, 3), 255, np.uint8)
    rects = []
    _, ref = _plan(1408, 1408)
    seams = [hi for _, hi in TR.cores(1408, ref["t_w"], ref["s_w"], ref["n_w"], ref["margin"])[:-1]]
    assert len(seams) == 3
    for k, s in enumerate(seams):                            # glyphs of the size bench.py's pages have at scale 2
        for orient in (0, 1):
            word = "SEAM" + "ABC"[k] + "XY"[orient]
            (tw, th), _ = cv2.getTextSize(word, cv2.FONT_HERSHEY_SIMPLEX, 1.8, 3)
            if orient == 0:                                  # across the vertical seam x = s
                x, y = s - tw // 2, (100, 250, 500)[k] + th // 2
            else:                                            # across the horizontal seam y = s
                x, y = (60, 360, 700)[k], s + th // 2
            cv2.putText(page, word, (x, y), cv2.FONT_HERSHEY_SIMPLEX, 1.8, (0, 0, 0), 3, cv2.LINE_AA)
            rects.append((x, y - th, x + tw, y))
    for tile in (None, TILE):
        boxes = det.detect([page], tile_size=tile)[0]
        assert len(boxes) >= len(rects)
        for x0, y0, x1, y1 in rects:
            centres = boxes.reshape(-1, 4, 2).mean(1)
            inside = ((centres[:, 0] > x0 - 4) & (centres[:, 0] < x1 + 4) & (centres[:, 1] > y0 - 4) &
                      (centres[:, 1] < y1 + 4))
            assert int(inside.sum()) == 1, (tile, (x0, y0, x1, y1), boxes)
