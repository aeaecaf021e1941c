"""Wide words on the GPU: b2o_window_plan_test, b2o_window_counts, b2o_warp_windows and b2o_stitch_windows against the
NumPy reference (tests/window_refs.py), their memory contract, and ``max_windows`` through the recognizer and
``Pipeline.recognize`` on rendered pages."""
import numpy as np
import pytest
import torch

from keras_ocr_b200 import _lib, weights as W
from tests import window_refs as R
from tests.test_gpu_memory_contract import ERR_ARG, rejected, run
from tests.test_window_refs import window_cases

pytestmark = pytest.mark.gpu
C = 37


@pytest.fixture(scope="module")
def ctx(cuda_device):
    return _lib.Context(0)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("m", [1, 2, 4, 16])
def test_window_plans_bit_for_bit(ctx, m):
    _, quads = window_cases()
    quads = np.concatenate([quads, R.random_boxes(1, 300)])
    plans = torch.zeros(len(quads) * m * _lib.WINDOW_PLAN_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    ctx.window_plan_test(_dev(quads).data_ptr(), len(quads), m, plans.data_ptr(), _stream())
    got = plans.cpu().numpy().view(_lib.WINDOW_PLAN_DTYPE).reshape(len(quads), m)
    for i, q in enumerate(quads):
        for k in range(m):
            ref, g = R.plan(q, m, k), got[i, k]
            for f in ("k", "dw", "dh", "valid"):
                assert int(g[f]) == ref[f], (i, k, f)
            for f in ("a", "wc", "sh"):
                assert np.float64(g[f]).tobytes() == np.float64(ref[f]).tobytes(), (i, k, f)
            if ref["valid"]:
                assert g["m"].tobytes() == ref["m"].tobytes(), (i, k)


def test_window_counts_table_and_memory_contract(ctx):
    quads = R.random_boxes(2, 6 * 40).reshape(6, 40, 4, 2)
    counts = np.array([0, 40, 7, 1, 39, 13], np.int32)
    boxes, cnt = _dev(quads), _dev(counts)
    n, mb = quads.shape[:2]

    def written(_):
        mask = np.zeros((n, mb), bool)
        for i, c in enumerate(counts):
            mask[i, :c] = True
        return np.repeat(mask.reshape(-1), 4)

    first = run(ctx, lambda g: ctx.lib.b2o_window_counts(ctx.handle, boxes.data_ptr(), cnt.data_ptr(), n, mb, 4,
                                                         g["w"].ptr, _stream()),
                {"w": (n * mb * 4, "i", written)}, inputs=(boxes, cnt), launches=1)
    got = first["w"].view(np.int32).reshape(n, mb)
    for i, c in enumerate(counts):
        assert got[i, :c].tolist() == [R.extent(q, 4)[3] for q in quads[i, :c]]
    for bad in (0, 17):
        rejected(ctx, lambda g: ctx.lib.b2o_window_counts(ctx.handle, boxes.data_ptr(), cnt.data_ptr(), n, mb, bad,
                                                          g["w"].ptr, _stream()), {"w": (n * mb * 4, "i")}, ERR_ARG,
                 inputs=(boxes, cnt))


@pytest.mark.parametrize("channels", [1, 3])
def test_warp_windows_bit_for_bit_and_in_chunks(ctx, channels):
    rng = np.random.default_rng(channels)
    img, _ = window_cases()
    imgs = np.stack([img, img[::-1]]) if channels == 1 else np.stack([np.stack([img, 255 - img, img[::-1]], -1)] * 2)
    quads = R.random_boxes(3, 120)
    index = rng.integers(0, 2, len(quads)).astype(np.int32)
    words, start = R.wide_list(quads, 4)
    total = int(start[-1])
    args = [_dev(a) for a in (imgs, quads, index, words, start)]
    ptrs = [a.data_ptr() for a in args]
    shape = (total, 31, 200) + ((3,) if channels == 3 else ())
    crops = torch.full(shape, 7, dtype=torch.uint8, device="cuda")
    x = torch.empty((total, 200, 31) + shape[3:], dtype=torch.float16, device="cuda")
    h, w = img.shape
    ctx.warp_windows(ptrs[0], channels, 2, h, w, ptrs[1], ptrs[2], ptrs[3], ptrs[4], len(words), 4, 0, total,
                     crops.data_ptr(), x.data_ptr(), _stream())
    got = crops.cpu().numpy()
    for i, b in enumerate(words):
        for k in range(start[i + 1] - start[i]):
            assert np.array_equal(got[start[i] + k], R.crop(imgs[index[b]], quads[b], 4, k)), (i, k)
    from tests import image_refs as I
    assert np.array_equal(x.cpu().numpy(), I.crops_to_input(got))
    # in two chunks, into slots 0.. of each call's outputs: the same windows
    part = torch.full(shape, 7, dtype=torch.uint8, device="cuda")
    cut = total // 3
    ctx.warp_windows(ptrs[0], channels, 2, h, w, ptrs[1], ptrs[2], ptrs[3], ptrs[4], len(words), 4, cut, total - cut,
                     part.data_ptr(), None, _stream())
    assert torch.equal(part[:total - cut], crops[cut:]) and bool((part[total - cut:] == 7).all())


def run_stitch(ctx, quads, m, words, start, lg, th, rows=None):
    rows = len(quads) if rows is None else rows
    labels = torch.full((rows, 48 * m), -7, dtype=torch.int32, device="cuda")
    logp = torch.full((rows,), 7.0, dtype=torch.float32, device="cuda")
    keep = [_dev(a) for a in (lg, quads, words, start)] + ([_dev(th)] if th is not None else [None])
    ctx.stitch_windows(keep[0].data_ptr(), C, None if th is None else keep[4].data_ptr(), keep[1].data_ptr(),
                       keep[2].data_ptr(), keep[3].data_ptr(), len(words), m, labels.data_ptr(), logp.data_ptr(),
                       _stream())
    return labels.cpu().numpy(), logp.cpu().numpy()


@pytest.mark.parametrize("n_words, theta", [(1, True), (8, True), (8, False), (300, True)])
def test_stitch_bit_for_bit(ctx, n_words, theta):
    quads, m, words, start, lg, th = R.stitch_case(n_words, n_words, theta)
    labels, logp = run_stitch(ctx, quads, m, words, start, lg, th)
    untouched = np.setdiff1d(np.arange(len(quads)), words)
    assert (labels[untouched] == -7).all() and (logp[untouched] == 7.0).all()
    for i, b in enumerate(words):
        s, e = start[i], start[i + 1]
        a = R.starts(e - s, R.extent(quads[b], m)[1])
        row, ref_s, _, _ = R.stitch(lg[s:e], None if th is None else th[s:e], a, m)
        assert labels[b].tolist() == row.tolist(), (i, b)
        assert abs(float(logp[b]) - float(ref_s)) <= 1e-5 * max(1.0, abs(float(ref_s))), (i, float(logp[b]), ref_s)


def test_stitch_alone_equals_in_a_batch(ctx):
    quads, m, words, start, lg, th = R.stitch_case(11, 64)
    labels, logp = run_stitch(ctx, quads, m, words, start, lg, th)
    for i in (0, 5, len(words) - 1):
        s, e = start[i], start[i + 1]
        one_l, one_p = run_stitch(ctx, quads[words[i]][None], m, np.zeros(1, np.int32), np.array([0, e - s], np.int32),
                                  lg[s:e], th[s:e])
        assert one_l[0].tobytes() == labels[words[i]].tobytes() and one_p[0].tobytes() == logp[words[i]].tobytes()


def test_stitch_memory_contract(ctx):
    quads, m, words, start, lg, th = R.stitch_case(12, 40)
    n = len(quads)
    ins = [_dev(a) for a in (lg, th, quads, words, start)]
    row_bytes = 48 * m * 4
    keep = np.isin(np.arange(n), words)

    def call(g, mw=m):
        return ctx.lib.b2o_stitch_windows(ctx.handle, ins[0].data_ptr(), C, ins[1].data_ptr(), ins[2].data_ptr(),
                                          ins[3].data_ptr(), ins[4].data_ptr(), len(words), mw, g["l"].ptr,
                                          g["p"].ptr, _stream())

    bufs = {"l": (n * row_bytes, "i", np.repeat(keep, row_bytes)), "p": (n * 4, "f", np.repeat(keep, 4))}
    run(ctx, call, bufs, inputs=tuple(ins), launches=1)
    rejected(ctx, lambda g: call(g, 0), {k: v[:2] for k, v in bufs.items()}, ERR_ARG, inputs=tuple(ins))


# ------------------------------------------------------------------------------------------- the pipeline
@pytest.fixture(scope="module")
def pipe(cuda_device):
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    from keras_ocr_b200.recognition import Recognizer
    return Pipeline(detector=Detector(weights=W.synthetic_craft_weights(3, textlike=True), device=0),
                    recognizer=Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True), device=0), scale=2)


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        if isinstance(x, (list, tuple)) and not isinstance(x, str):
            _same(x, y)
        elif isinstance(x, np.ndarray):
            assert x.dtype == y.dtype and x.tobytes() == y.tobytes()
        else:
            assert x == y or (x != x and y != y)


COMBOS = {"plain": {}, "scores": {"return_scores": True}, "lines": {"return_lines": True, "return_scores": True},
          "blocks": {"return_blocks": True}, "inflight": {}}


@pytest.mark.parametrize("combo", list(COMBOS))
def test_pages_without_wide_boxes_read_as_the_default(pipe, combo):
    from oracle import synth
    pages, _ = synth.text_images(seed=1000, n=8, h=768, w=768, n_words=32)      # bench.py's pages
    kw = COMBOS[combo]
    pipe.inflight = 2 if combo == "inflight" else 1
    try:
        plain = pipe.recognize(pages, **kw)
        for m in (1, 4):
            _same(pipe.recognize(pages, recognition_kwargs={"max_windows": m}, **kw), plain)
    finally:
        pipe.inflight = 1
    words = [w for page in plain for w in page]
    for _ in ("lines", "blocks")[:("lines", "blocks").index(combo) + 1] if combo in ("lines", "blocks") else ():
        words = [w for _, _, ws in words for w in ws]              # (text, box, members) -> members
    assert len(words) > 200
    assert all(R.extent(w[1] * 2, 4)[3] == 1 for w in words)      # no box is wide in the detector's pixels (scale 2)


def test_the_recognize_stage_does_not_wait_for_the_device(pipe, monkeypatch):
    """With max_windows > 1 the recognize stage queues its work without a host synchronisation (torch raises on one in
    sync-debug mode "error"), on pages with wide words and on pages without."""
    from oracle import synth
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
    long_pages = np.stack([R.long_word_page(s)[0] for s in range(2)])
    bench_pages, _ = synth.text_images(seed=1000, n=2, h=768, w=768, n_words=32)
    for pages in (long_pages, bench_pages):
        for kw in ({}, {"return_scores": True}, {"return_lines": True}):
            pipe.recognize(pages, recognition_kwargs={"max_windows": 4}, **kw)
    assert len(calls) == 6


def test_long_words_read_better_in_windows(pipe):
    pages = [R.long_word_page(s) for s in range(4)]
    images = np.stack([p for p, _ in pages])
    plain = pipe.recognize(images, return_scores=True)
    wide = pipe.recognize(images, recognition_kwargs={"max_windows": 4}, return_scores=True)
    a = sum(R.exact_reads(r, items) for r, (_, items) in zip(plain, pages))
    b = sum(R.exact_reads(r, items) for r, (_, items) in zip(wide, pages))
    items = sum(len(i) for _, i in pages)
    print(f"long-word pages: {a} of {items} items read exactly by default, {b} with max_windows=4")
    for p, q in zip(plain, wide):                     # the same boxes and detection scores, word for word
        assert len(p) == len(q)
        for x, y in zip(p, q):
            assert x[1].tobytes() == y[1].tobytes() and x[2] == y[2]
            if R.extent(x[1] * 2, 4)[3] == 1:         # boxes in the detector's pixels (scale 2) that fit: as today
                assert x[0] == y[0] and x[3] == y[3]
    assert b > a
    # the recognizer's own entry point reads the same words from host box groups
    padded, _ = pipe.prepare_device(images[:1])
    groups = [np.stack([w[1] for w in wide[0]]) * 2]
    got = pipe.recognizer.recognize_from_boxes(padded.cpu().numpy(), groups, max_windows=4)
    assert got[0] == [w[0] for w in wide[0]]


def test_invalid_values_and_combinations_raise_before_any_launch(pipe):
    page = R.long_word_page(9)[0][None]
    rec = pipe.recognizer
    n0 = pipe.detector.ctx.launch_count() + rec.ctx.launch_count()
    for m in (0, 17, True, 2.0, "4", None):
        with pytest.raises(ValueError):
            pipe.recognize(page, recognition_kwargs={"max_windows": m})
    for kw in ({"recognition_kwargs": {"max_windows": 4, "beam_width": 4}},
               {"recognition_kwargs": {"max_windows": 4, "lexicon": ["abc"]}},
               {"recognition_kwargs": {"max_windows": 4, "rotations": (0, 2)}},
               {"recognition_kwargs": {"max_windows": 4}, "return_char_boxes": True},
               {"recognition_kwargs": {"max_windows": 4}, "return_polygons": True}):
        with pytest.raises(ValueError):
            pipe.recognize(page, **kw)
    box = np.array([[[0, 0], [300, 0], [300, 20], [0, 20]]], np.float32)
    with pytest.raises(ValueError):
        rec.recognize_from_boxes(page, [box], max_windows=4, beam_width=2)
    with pytest.raises(ValueError):
        rec.recognize_from_boxes(page, [box], max_windows=False)
    images_t = torch.from_numpy(page).cuda()
    table = torch.from_numpy(np.stack([box, box], 1)).cuda()                 # (1, 2, 4, 2), two boxes
    for windows in (np.array([2]), np.array([2, 1, 1]), np.array([0, 2]), np.array([2, 5]), np.array([1.0, 2.0])):
        with pytest.raises(ValueError):
            rec.recognize_from_boxes_device(images_t, table, np.array([2]), max_windows=4, windows=windows)
    assert pipe.detector.ctx.launch_count() + rec.ctx.launch_count() == n0
