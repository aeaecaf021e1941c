"""CPU: the quarter-turn references of tests/rotation_refs.py against cv2 and on crafted votes, and the validation of
``recognition.check_rotations``."""
import cv2
import numpy as np
import pytest

from keras_ocr_b200 import recognition
from tests import image_refs as IR
from tests import rotation_refs as RR

GROUPS = IR.warp_cases()


def _cv2_turned(img, quad, r):
    """cv2.getPerspectiveTransform + cv2.warpPerspective of the turned box pasted into a zero 31x200 crop, i.e.
    tools.warpBox(image, np.roll(c, -r, axis=0), 31, 200, skip_rotate=True)."""
    from oracle import imageops
    box = RR.turned_box(quad, r)
    w, h = imageops.rotated_width_height(box)
    scale = min(IR.CROP_W / w, IR.CROP_H / h)
    dst = np.array([[0, 0], [scale * w, 0], [scale * w, scale * h], [0, scale * h]]).astype("float32")
    crop = cv2.warpPerspective(img, cv2.getPerspectiveTransform(src=box, dst=dst), dsize=(int(scale * w), int(scale * h)))
    full = np.zeros((IR.CROP_H, IR.CROP_W) + img.shape[2:], np.uint8)
    full[:crop.shape[0], :crop.shape[1]] = crop
    return full


@pytest.mark.parametrize("group", GROUPS, ids=[g["name"] for g in GROUPS])
def test_turned_warp_equals_cv2(group):
    """Every turn of every case, gray and colour, bit for bit against cv2; turn 0 is image_refs.warp_box."""
    compared = 0
    for q, i in zip(group["quads"], group["image_index"]):
        for img in (group["gray"][i], group["rgb"][i]):
            assert np.array_equal(RR.turned_warp(img, q, 0)[0], IR.warp_box(img, q)[0])
            for r in range(4):
                crop, plan = RR.turned_warp(img, q, r)
                if plan is None:
                    assert not crop.any()
                    with pytest.raises(ZeroDivisionError):
                        _cv2_turned(img, q, r)
                    continue
                if min(plan[1:]) == 0:                  # cv2's dsize fallback: unpinned, as for turn 0
                    assert not crop.any()
                    continue
                assert np.array_equal(crop, _cv2_turned(img, q, r)), (q.tolist(), r, plan[1:])
                compared += 1
    assert compared >= 4 * len(group["quads"])


def test_turns_swap_width_and_height():
    """Odd turns measure the box after the roll: a 150 x 28 box is cut 200 x 37 -> 31 tall in turns 0 / 2 and as a
    28 x 150 box, 5 px wide, in turns 1 / 3; turn 2 is turn 0 upside down."""
    img = np.random.default_rng(1).integers(0, 256, (60, 200), dtype=np.uint8)
    quad = IR._axis(10, 20, 160, 48)
    dims = [RR.turned_warp(img, quad, r)[1][1:] for r in range(4)]
    assert dims[0] == dims[2] and dims[1] == dims[3] and dims[0][0] > dims[0][1] and dims[1][0] < dims[1][1]
    assert dims[1][1] == 31
    c = RR.turned_box(quad, 0)
    assert np.array_equal(RR.turned_box(quad, 2), c[[2, 3, 0, 1]])


def rot90_points(q, k, h, w):
    """Points of an (h, w) page on np.rot90(page, k): (x, y) -> (y, w - 1 - x), applied k times."""
    q = np.asarray(q, np.float64)
    for _ in range(k):
        q = np.stack([q[:, 1], w - 1 - q[:, 0]], 1)
        h, w = w, h
    return q.astype(np.float32)


def test_rot90_page_reads_upright_in_turn():
    """A box on np.rot90(page, k), cut in turn (4 - k) % 4, starts at the upright box's top-left corner and gives the
    upright crop up to the 1/32-pixel rounding of the homography (a smooth page keeps that rounding below 2 levels)."""
    yy, xx = np.mgrid[0:90, 0:130]
    page = (127 + 60 * np.sin(xx / 5.0) + 60 * np.cos(yy / 4.0)).astype(np.uint8)
    for quad in (IR._axis(12, 30, 112, 50), IR._axis(20.5, 10, 60, 80.25)):
        upright = RR.turned_warp(page, quad, 0)[0]
        for k in (1, 2, 3):
            q = rot90_points(quad, k, *page.shape)
            r = (4 - k) % 4
            assert np.array_equal(RR.turned_box(q, r), rot90_points(RR.turned_box(quad, 0), k, *page.shape))
            got = RR.turned_warp(np.ascontiguousarray(np.rot90(page, k)), q, r)[0]
            assert np.abs(got.astype(int) - upright.astype(int)).max() <= 2, k


def _check_select_semantics(case, vote, out):
    labels, logp, turns_out, rolled = out
    best = case["logp"][:, :, 0]
    r, b = best.shape
    for k in range(b):
        j = case["turns"].index(int(turns_out[k]))
        assert np.array_equal(labels[k], case["labels"][j, k]) and np.array_equal(logp[k], case["logp"][j, k])
        if vote == "word":
            first_max = next(i for i in range(r) if not (best[:, k] > best[i, k]).any())
            assert j == first_max if np.isfinite(best[:, k]).any() else j == 0
        assert np.array_equal(rolled[k], RR.turned_box(case["boxes"][k], turns_out[k]))


@pytest.mark.parametrize("vote", ["word", "page"])
@pytest.mark.parametrize("case", RR.select_cases(), ids=[c["name"] for c in RR.select_cases()])
def test_select_reference(case, vote):
    """The reference on crafted arrays: the chosen turn's readings, ties and all -inf to the turn listed first, one
    turn per image for "page", and a word's (an image's) result independent of the other words (images)."""
    out = RR.select(case["labels"], case["logp"], case["image_index"], case["turns"], vote, case["boxes"])
    _check_select_semantics(case, vote, out)
    if vote == "page":
        for img in np.unique(case["image_index"]):
            assert len(set(out[2][case["image_index"] == img].tolist())) == 1
    # one image alone gives the same result
    for img in np.unique(case["image_index"])[:3]:
        ks = np.flatnonzero(case["image_index"] == img)
        alone = RR.select(case["labels"][:, ks], case["logp"][:, ks], case["image_index"][ks], case["turns"], vote,
                          case["boxes"][ks])
        for a, full in zip(alone, out):
            assert np.array_equal(a, full[ks])


def test_select_hand_cases():
    turns = (2, 0, 1)
    lab = np.arange(3 * 4 * 1 * 48, dtype=np.int32).reshape(3, 4, 1, 48)
    lp = np.array([[-1, -3, -np.inf, -2], [-1, -2, -np.inf, -9], [-0.5, -3, -np.inf, -9]], np.float32)[..., None]
    idx = np.array([0, 0, 1, 1], np.int32)
    _, _, t, _ = RR.select(lab, lp, idx, turns, "word")
    assert t.tolist() == [1, 0, 2, 2]                   # -0.5 wins; -2 beats -3; all -inf -> first listed; -2 first
    _, _, t, _ = RR.select(lab, lp, idx, turns, "page")
    # image 0: sums -4, -3, -3.5 -> turn 0 (listed second); image 1: every sum -inf -> turn 2 (listed first)
    assert t.tolist() == [0, 0, 2, 2]


# ----------------------------------------------------------------------------------------------- check_rotations
@pytest.mark.parametrize("rotations,vote,want", [
    (None, "word", None), (None, "page", None), ((0,), "word", (0,)), ([0, 2], "page", (0, 2)),
    ((0, 1, 2, 3), "word", (0, 1, 2, 3)), ((3, 1), "page", (3, 1)), ((np.int64(2), 0), "word", (2, 0)),
    ([np.int32(1)], "word", (1,)),
])
def test_check_rotations_accepts(rotations, vote, want):
    got = recognition.check_rotations(rotations, vote)
    assert got == want and (got is None or all(type(r) is int for r in got))


@pytest.mark.parametrize("rotations,vote", [
    ((), "word"), ([], "word"), ((True,), "word"), ((0, False), "word"), ((0, 0), "word"), ([1, 2, 1], "page"),
    ((4,), "word"), ((-1,), "word"), ((0, 1.0), "word"), (("0",), "word"), ("02", "word"), (0, "word"),
    ({0, 1}, "word"), (np.array([0, 1]), "word"), ((0,), "words"), ((0,), "Page"), ((0,), None), (None, "any"),
    ((np.bool_(True),), "word"), ((0,), 1),
])
def test_check_rotations_rejects(rotations, vote):
    with pytest.raises(ValueError):
        recognition.check_rotations(rotations, vote)
