"""GPU: reading words in quarter turns -- ``b2o_warp_boxes_turned`` and ``b2o_select_rotation`` bit for bit against
tests/rotation_refs.py, the recognizer's turn loop against separate single-turn runs, and the whole pipeline on bench
pages turned by np.rot90."""
import numpy as np
import pytest
import torch

import bench
from keras_ocr_b200 import _lib, distributed, recognition, weights as W
from keras_ocr_b200.detection import Detector
from keras_ocr_b200.pipeline import Pipeline
from keras_ocr_b200.recognition import Lexicon, Recognizer
from oracle import imageops
from tests import image_refs as IR
from tests import rotation_refs as RR
from tests.test_rotation_refs import rot90_points

pytestmark = pytest.mark.gpu

GROUPS = IR.warp_cases()
N_PAGES = 4


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _dev(a, device):
    return torch.from_numpy(np.ascontiguousarray(a)).to(device)


@pytest.fixture(scope="module")
def ctx(cuda_device):
    c = _lib.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def pipe(cuda_device):
    det = Detector(weights=W.synthetic_craft_weights(3, textlike=True), device=0)
    rec = Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True), device=0)
    return Pipeline(detector=det, recognizer=rec, scale=bench.SCALE, max_size=2048)


@pytest.fixture(scope="module")
def pages():
    p, words, rects = bench.make_pages(0, with_layout=True)
    return p[:N_PAGES], words[:N_PAGES], rects[:N_PAGES]


# ------------------------------------------------------------------------------------------------ 1. turned warp
@pytest.mark.parametrize("color", [False, True], ids=["gray", "color"])
@pytest.mark.parametrize("group", GROUPS, ids=[g["name"] for g in GROUPS])
def test_turned_warp_bit_exact(ctx, cuda_device, group, color):
    """Every turn: crops == rotation_refs.turned_warp (degenerate boxes all zero) and the CRNN input == those crops
    transposed; turn 0 == b2o_warp_boxes(_color)."""
    img = group["rgb"] if color else group["gray"]
    quads, index = group["quads"], group["image_index"]
    b, ch = len(quads), 3 if color else 1
    n, h, w = img.shape[:3]
    tail = (3,) if color else ()
    img_t, quads_t, index_t = _dev(img, cuda_device), _dev(quads, cuda_device), _dev(index, cuda_device)
    plain = torch.full((b, IR.CROP_H, IR.CROP_W) + tail, 0x5A, dtype=torch.uint8, device=cuda_device)
    ctx.warp_boxes(img_t.data_ptr(), n, h, w, quads_t.data_ptr(), index_t.data_ptr(), b, plain.data_ptr(), None,
                   _stream(), color=color)
    for r in range(4):
        crops = torch.full((b, IR.CROP_H, IR.CROP_W) + tail, 0x5A, dtype=torch.uint8, device=cuda_device)
        crnn_in = torch.full((b, IR.CROP_W, IR.CROP_H) + tail, float("nan"), dtype=torch.float16, device=cuda_device)
        ctx.warp_boxes_turned(img_t.data_ptr(), ch, n, h, w, quads_t.data_ptr(), index_t.data_ptr(), b, r,
                              crops.data_ptr(), crnn_in.data_ptr(), _stream())
        got = crops.cpu().numpy()
        bad = []
        for k, (q, i) in enumerate(zip(quads, index)):
            ref, plan = RR.turned_warp(img[i], q, r)
            if not np.array_equal(got[k], ref):
                bad.append((r, k, q.tolist(), None if plan is None else plan[1:], int((got[k] != ref).sum())))
        assert not bad, bad
        assert np.array_equal(crnn_in.cpu().numpy(), IR.crops_to_input(got))
        if r == 0:
            assert torch.equal(crops, plain)


def test_turned_warp_rejects_bad_arguments(ctx, cuda_device):
    img = torch.zeros((1, 8, 8), dtype=torch.uint8, device=cuda_device)
    box = _dev(IR._axis(1, 1, 6, 4)[None], cuda_device)
    idx = torch.zeros((1,), dtype=torch.int32, device=cuda_device)
    out = torch.empty((1, 31, 200), dtype=torch.uint8, device=cuda_device)
    for ch, turn in ((1, 4), (1, -1), (2, 0)):
        with pytest.raises(_lib.B2OError):
            ctx.warp_boxes_turned(img.data_ptr(), ch, 1, 8, 8, box.data_ptr(), idx.data_ptr(), 1, turn, out.data_ptr(),
                                  None, _stream())


# ------------------------------------------------------------------------------------------------ 2. select kernel
def _table(flat, index, n_images):
    counts = np.bincount(index, minlength=n_images)
    m = max(1, int(counts.max()) if len(counts) else 1)
    table = np.full((n_images, m, 4, 2), 7.25, np.float32)
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
    for k, i in enumerate(index):
        table[i, k - starts[i]] = flat[k]
    return table, starts


def run_select(ctx, device, labels, logp, index, n_images, turns, vote, boxes):
    r, b, p = logp.shape
    lab_t, lp_t, idx_t = _dev(labels, device), _dev(logp, device), _dev(index, device)
    table, _ = _table(boxes, index, n_images)
    flat_t, table_t = _dev(boxes, device), _dev(table, device)
    out_l = torch.full((b, p, 48), -7, dtype=torch.int32, device=device)
    out_p = torch.full((b, p), 3.0, dtype=torch.float32, device=device)
    out_t = torch.full((b,), -7, dtype=torch.int32, device=device)
    ctx.select_rotation(lab_t.data_ptr(), lp_t.data_ptr(), idx_t.data_ptr(), n_images, b, p, turns,
                        recognition.ROTATION_VOTES[vote], out_l.data_ptr(), out_p.data_ptr(), out_t.data_ptr(),
                        flat_t.data_ptr(), table_t.data_ptr(), table.shape[1], _stream())
    return out_l.cpu().numpy(), out_p.cpu().numpy(), out_t.cpu().numpy(), flat_t.cpu().numpy(), table_t.cpu().numpy()


CASES = RR.select_cases()


@pytest.mark.parametrize("vote", ["word", "page"])
@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_select_kernel_bit_exact(ctx, cuda_device, case, vote):
    """labels, logp, turns, the rolled flat boxes and the rolled table == rotation_refs.select in every bit; table slots
    past an image's words are untouched."""
    want = RR.select(case["labels"], case["logp"], case["image_index"], case["turns"], vote, case["boxes"])
    lab, lp, turns, flat, table = run_select(ctx, cuda_device, case["labels"], case["logp"], case["image_index"],
                                             case["n_images"], case["turns"], vote, case["boxes"])
    assert np.array_equal(lab, want[0]) and np.array_equal(turns, want[2])
    assert np.array_equal(lp.view(np.uint32), want[1].view(np.uint32))
    assert np.array_equal(flat.view(np.uint32), want[3].view(np.uint32))
    want_table, _ = _table(want[3], case["image_index"], case["n_images"])
    assert np.array_equal(table.view(np.uint32), want_table.view(np.uint32))


@pytest.mark.parametrize("case", [c for c in CASES if c["name"] in ("R4_P1", "R3_P3_order_2_0_3", "R4_P1_long_page")],
                         ids=lambda c: c["name"])
def test_select_kernel_batch_invariant(ctx, cuda_device, case):
    """A word's result is the same alone, in a batch of 7 and in a batch of 17 ("word" vote), and an image's words are
    the same with the image alone ("page" vote)."""
    for vote in ("word", "page"):
        full = run_select(ctx, cuda_device, case["labels"], case["logp"], case["image_index"], case["n_images"],
                          case["turns"], vote, case["boxes"])
        b = len(case["image_index"])
        if vote == "word":
            chunks = [np.arange(k, min(k + size, b)) for size in (1, 7, 17) for k in range(0, b, size)]
        else:
            chunks = [np.flatnonzero(case["image_index"] == i) for i in np.unique(case["image_index"])]
        for ks in chunks:
            part = run_select(ctx, cuda_device, case["labels"][:, ks], case["logp"][:, ks],
                              np.zeros(len(ks), np.int32), 1, case["turns"], vote, case["boxes"][ks])
            for a, f in zip(part[:4], full[:4]):               # labels, logp, turns, rolled boxes: every bit
                assert a.tobytes() == np.ascontiguousarray(f[ks]).tobytes(), (vote, ks.tolist())


def test_select_rejects_bad_arguments(ctx, cuda_device):
    z = torch.zeros((64,), dtype=torch.int32, device=cuda_device)
    p = z.data_ptr()
    for turns, vote in (((0, 0), 0), ((4,), 0), ((), 0), ((0, 1, 2, 3, 0), 0), ((0,), 2)):
        with pytest.raises(_lib.B2OError):
            ctx.select_rotation(p, p, p, 1, 1, 1, turns, vote, p, p, p, None, None, 0, _stream())


# ------------------------------------------------------------------------------------------------ helpers: pages
def rotated_batch(pages, k_of_page):
    return np.stack([np.ascontiguousarray(np.rot90(p, k)) for p, k in zip(pages, k_of_page)])


def rect_boxes(rects):
    return np.array([[[x0, y0], [x1, y0], [x1, y1], [x0, y1]] for x0, y0, x1, y1 in rects], np.float32)


def table_of(groups):
    counts = np.array([len(g) for g in groups])
    m = max(1, int(counts.max()))
    table = np.zeros((len(groups), m, 4, 2), np.float32)
    for i, g in enumerate(groups):
        table[i, :len(g)] = g
    return table, counts


def lexicon_of(words, rec):
    vocab = list(dict.fromkeys(w for page in words for w in page))
    return Lexicon(vocab + ["zzq", "qqq", "sos", "noon"], rec.alphabet)


# ------------------------------------------------------------------------------------------------ 3. fused vs separate
@pytest.mark.parametrize("decoder", ["greedy", "beam", "lexicon"])
def test_fused_turns_equal_separate_runs(pipe, pages, cuda_device, decoder):
    """recognize_from_boxes_device(rotations=(0,1,2,3)) == the host vote (rotation_refs.select) over four separate
    single-turn runs (b2o_warp_boxes_turned + predict_device): labels, logp, turns and rolled boxes, both votes."""
    rec = pipe.recognizer
    imgs, words, rects = pages
    ks = [0, 1, 2, 3]
    batch = rotated_batch(imgs, ks)
    groups = [rot90_points(rect_boxes(r).reshape(-1, 2), k, *imgs[0].shape[:2]).reshape(-1, 4, 2)
              for r, k in zip(rects, ks)]
    table, counts = table_of(groups)
    flat = np.concatenate(groups)
    index = np.repeat(np.arange(len(groups), dtype=np.int32), counts)
    beam = {"greedy": {}, "beam": {"beam_width": 10, "top_paths": 3},
            "lexicon": {"lexicon": lexicon_of(words, rec), "top_paths": 2}}[decoder]
    images_t = _dev(batch, cuda_device)
    gray = rec.gray_device(images_t)
    flat_t, idx_t = _dev(flat, cuda_device), _dev(index, cuda_device)
    per_turn = []
    for r in range(4):
        crnn_in, _ = rec.warp_device(gray, flat_t, idx_t, turn=r)
        lab, lp = rec.predict_device(crnn_in, with_scores=True, **beam)
        p = beam.get("top_paths", 1)
        per_turn.append((lab.cpu().numpy().reshape(len(flat), p, 48), lp.cpu().numpy().reshape(len(flat), p)))
    labels_all = np.stack([a for a, _ in per_turn])
    logp_all = np.stack([b for _, b in per_turn])
    for vote in ("word", "page"):
        want = RR.select(labels_all, logp_all, index, (0, 1, 2, 3), vote, flat)
        table_t = _dev(table, cuda_device)
        lab, lp, turns = rec.recognize_from_boxes_device(images_t, table_t, counts, with_scores=True,
                                                         rotations=(0, 1, 2, 3), rotation_vote=vote, **beam)
        p = beam.get("top_paths", 1)
        assert np.array_equal(lab.cpu().numpy().reshape(len(flat), p, 48), want[0])
        assert np.array_equal(lp.cpu().numpy().reshape(len(flat), p).view(np.uint32), want[1].view(np.uint32))
        assert np.array_equal(turns.cpu().numpy(), want[2])
        got_table = table_t.cpu().numpy()
        got_flat = np.concatenate([got_table[i, :c] for i, c in enumerate(counts)])
        assert np.array_equal(got_flat, want[3])
        if vote == "page":
            print(f"{decoder}: page turns {[int(want[2][index == i][0]) for i in range(len(ks))]} for k = {ks}")


# ------------------------------------------------------------------------------------------------ 4. rotations=(0,)
def test_turn_zero_equals_default(pipe, pages):
    """rotations=(0,): texts and confidences equal the default call's bit for bit, each box the same corners up to a
    cyclic shift."""
    imgs = pages[0]
    base = pipe.recognize(imgs, return_scores=True)
    got = pipe.recognize(imgs, return_scores=True, recognition_kwargs={"rotations": (0,)})
    assert [len(g) for g in got] == [len(g) for g in base]
    for g, b in zip(got, base):
        for (t, box, ds, c), (t0, box0, ds0, c0) in zip(g, b):
            assert t == t0 and np.float32(c).view(np.uint32) == np.float32(c0).view(np.uint32) and ds == ds0
            assert any(np.array_equal(box, np.roll(box0, -s, axis=0)) for s in range(4)), (box, box0)


# ------------------------------------------------------------------------------------------------ 5. turned pages
ISOLATED = [("beam10", {"beam_width": 10}, (0, 1, 2, 3), (1, 2, 3), True),
            ("greedy", {}, (0, 2), (2,), True),
            ("greedy", {}, (0, 1, 2, 3), (1, 2, 3), False)]


@pytest.mark.parametrize("name,beam,rotations,ks,decisive", ISOLATED,
                         ids=[f"{n}-{''.join(map(str, r))}" for n, _, r, _, _ in ISOLATED])
def test_turned_pages_recognition_isolated(pipe, pages, cuda_device, name, beam, rotations, ks, decisive):
    """The upright call's boxes mapped onto np.rot90(page, k): the page vote chooses turn (4 - k) % 4 on every page
    and every word reads the upright text; the word vote's other choices are counted and printed.

    The greedy score S does not tell quarter turns apart (DESIGN.md section 1): the odd turns of a word cut its box
    across, into a crop a few pixels wide, which the recognizer reads as an all-blank path about as certain as a
    word.  So greedy decoding is held to the upright / upside-down choice (0, 2) and its four-turn vote is printed."""
    rec = pipe.recognizer
    imgs = pages[0]
    H, Wd = imgs.shape[1:3]
    found = pipe.recognize(imgs)
    groups = [np.array([b for _, b in g], np.float32).reshape(-1, 4, 2) for g in found]
    table, counts = table_of(groups)
    up = rec.recognize_from_boxes_device(_dev(imgs, cuda_device), _dev(table, cuda_device), counts, **beam)
    up_text = recognition.labels_to_text(up.cpu().numpy(), rec.alphabet)
    differ_total = 0
    for k in ks:
        turned = rotated_batch(imgs, [k] * len(imgs))
        t_groups = [rot90_points(g.reshape(-1, 2), k, H, Wd).reshape(-1, 4, 2) for g in groups]
        t_table, _ = table_of(t_groups)
        want = (4 - k) % 4
        for vote in ("page", "word"):
            lab, turns = rec.recognize_from_boxes_device(_dev(turned, cuda_device), _dev(t_table, cuda_device), counts,
                                                         rotations=rotations, rotation_vote=vote, **beam)
            text = recognition.labels_to_text(lab.cpu().numpy(), rec.alphabet)
            turns = turns.cpu().numpy()
            if vote == "page":
                page_turns = [int(t) for t in turns[np.cumsum(counts) - 1]]
                print(f"{name} {rotations} k={k}: page turns {page_turns} (upright: {want})")
                if not decisive:
                    continue
                assert (turns == want).all(), (k, turns)
                differ = [(i, a, b) for i, (a, b) in enumerate(zip(text, up_text)) if a != b]
                differ_total += len(differ)
                for i, a, b in differ:
                    print(f"k={k} word {i}: turned reads {a!r}, upright {b!r}")
            else:
                other = [(text[i], int(turns[i])) for i in np.flatnonzero(turns != want)]
                print(f"{name} {rotations} k={k} word vote: {len(other)} of {len(turns)} words picked another turn: "
                      f"{other[:8]}")
    print(f"{name} {rotations} page vote: {differ_total} words differ from the upright reading")
    assert differ_total == 0


# ------------------------------------------------------------------------------------------------ 6. end to end
@pytest.mark.parametrize("decoder", ["beam10", "greedy"])
def test_turned_pages_end_to_end(pipe, pages, decoder):
    """Pipeline.recognize on turned pages with rotations=(0,1,2,3), vote "page", against the default call on the same
    pages (bench.words_read against the turned rectangles, printed).  With beam search, for every k, every word found
    upright and in the turned call has its returned box[0], mapped back upright, within 2 px of the upright word's
    top-left corner (k = 2: horizontal boxes; k = 1 / 3: the detector has to find vertical words first).  Greedy
    decoding (whose four-turn vote is not decisive, see test_turned_pages_recognition_isolated) is only reported."""
    imgs, words, rects = pages
    H, Wd = imgs.shape[1:3]
    upright = pipe.recognize(imgs)
    kw = {"rotations": (0, 1, 2, 3), "rotation_vote": "page"}
    if decoder == "beam10":
        kw["beam_width"] = 10
    for k in (1, 2, 3):
        turned = rotated_batch(imgs, [k] * len(imgs))
        t_rects = []
        for page_rects in rects:
            pts = rot90_points(rect_boxes(page_rects).reshape(-1, 2), k, H, Wd).reshape(-1, 4, 2)
            t_rects.append([(q[:, 0].min(), q[:, 1].min(), q[:, 0].max(), q[:, 1].max()) for q in pts])
        plain = pipe.recognize(turned)
        rot = pipe.recognize(turned, recognition_kwargs=kw)
        hit_plain, total = bench.words_read(plain, words, t_rects)
        hit_rot, _ = bench.words_read(rot, words, t_rects)
        print(f"{decoder} k={k}: words_read default {hit_plain}/{total}, rotations {hit_rot}/{total}, boxes found "
              f"{sum(len(g) for g in rot)} (upright {sum(len(g) for g in upright)})")
        back_k = (4 - k) % 4
        matched, far = 0, []
        for g_up, g_rot in zip(upright, rot):
            if not g_rot:
                continue
            up_boxes = np.array([b for _, b in g_up], np.float32).reshape(-1, 4, 2)
            up_centres = up_boxes.mean(1)
            for t, box in g_rot:
                back = rot90_points(np.asarray(box), back_k, *turned.shape[1:3])
                d = np.abs(up_centres - back.mean(0)).max(1)
                j = int(np.argmin(d)) if len(d) else -1
                if j < 0 or d[j] > 2:
                    continue                               # no upright word at this place
                matched += 1
                tl = imageops.order_corners(up_boxes[j])[0]
                if np.abs(back[0] - tl).max() > 2:
                    far.append((t, g_up[j][0], back[0].tolist(), tl.tolist()))
        print(f"{decoder} k={k}: {matched} words found in both calls, {len(far)} with box[0] off the upright top-left: "
              f"{far[:3]}")
        if decoder == "beam10":
            assert not far
            if k == 2:
                assert matched >= 0.9 * sum(len(g) for g in upright)


# ------------------------------------------------------------------------------------------------ 7. records
def test_records_with_rotations(pipe, pages):
    """recognize_records(rotations, scores=True) decoded by distributed.unpack_blocks == recognize(return_scores=True)
    with the same kwargs: words, rolled boxes, detection scores and confidences; bad arguments raise before launch."""
    imgs = rotated_batch(pages[0], [2, 2, 0, 1])
    for vote in ("word", "page"):
        kw = {"rotations": (0, 2, 1, 3), "rotation_vote": vote}
        ref = pipe.recognize(imgs, return_scores=True, recognition_kwargs=kw)
        records = pipe.recognize_records(imgs, rec_boxes=64, scores=True, **kw)
        counts, boxes, labels, box_scores, logp = distributed.unpack_blocks([records], 64, scores=True)
        texts = recognition.labels_to_text(labels.astype(np.int32), pipe.recognizer.alphabet)
        conf = recognition.confidences(logp)
        flat = [w for g in ref for w in g]
        assert counts.tolist() == [len(g) for g in ref]
        assert texts == [w[0] for w in flat]
        assert np.array_equal(boxes, np.array([w[1] for w in flat], np.float32).reshape(-1, 4, 2))
        assert np.array_equal(box_scores, np.array([w[2] for w in flat], np.float32))
        assert np.array_equal(conf, np.array([w[3] for w in flat], np.float32))
    launches = pipe.detector.ctx.launch_count() + pipe.recognizer.ctx.launch_count()
    for bad in ({"rotations": (0, 4)}, {"rotations": ()}, {"rotations": (1,), "rotation_vote": "line"}):
        with pytest.raises(ValueError):
            pipe.recognize_records(imgs, **bad)
        with pytest.raises(ValueError):
            pipe.recognize(imgs, recognition_kwargs=bad)
        with pytest.raises(ValueError):
            distributed.recognize_sharded(pipe, imgs, **bad)
    assert pipe.detector.ctx.launch_count() + pipe.recognizer.ctx.launch_count() == launches
