"""CPU: the image-stage references of tests/image_refs.py equal cv2 on every case the GPU tests run."""
import cv2
import numpy as np
import pytest

from oracle import imageops
from tests import cvmodels as M
from tests import image_refs as R

GROUPS = R.warp_cases()


def _zero_side(plan):
    return plan is not None and min(plan[1:]) == 0


@pytest.mark.parametrize("group", GROUPS, ids=[g["name"] for g in GROUPS])
def test_warp_reference_equals_cv2(group):
    """Every crop, gray and colour, equal to imageops.warp_box (cv2.getPerspectiveTransform + warpPerspective), and the
    reference plan invalid exactly where warpBox raises ZeroDivisionError."""
    compared = 0
    for q, i in zip(group["quads"], group["image_index"]):
        for img in (group["gray"][i], group["rgb"][i]):
            crop, plan = R.warp_box(img, q)
            if _zero_side(plan):
                continue                                    # test_zero_side_dsize_is_unpinned
            if plan is None:
                with pytest.raises(ZeroDivisionError):
                    imageops.warp_box(img, q)
                assert not crop.any()
                continue
            assert np.array_equal(crop, imageops.warp_box(img, q)), (q.tolist(), plan[1:])
            compared += 1
    assert compared >= len(group["quads"])


def test_cases_are_rectangles_kept_by_get_rotated_box():
    """The kernel implements get_rotated_box's rectangle branch (the host rectifies other quads first): every case is a
    rectangle whose corners order_corners keeps, or a degenerate box with no rotated rectangle at all."""
    for g in GROUPS:
        for k, q in enumerate(g["quads"]):
            rect = imageops.min_rotated_rectangle(q)
            if rect is not None:
                near = np.abs(rect[:, None, :] - q[None].astype(np.float64)).max(-1).min(-1).max()
                assert near <= 1e-3, (g["name"], k, q.tolist())


def test_cases_cover_the_edges():
    """The case set reaches what it is meant to: both block layouts, re-basing at x = 64 and at x = 146, dw = 200,
    dh = 31, dh = 1, dw <= 3, sources beyond the short saturation, and degenerate boxes."""
    dims, far, invalid = set(), 0, 0
    for g in GROUPS:
        for q in g["quads"]:
            try:
                m, dw, dh = R.warp_plan(q)
            except ZeroDivisionError:
                invalid += 1
                continue
            dims.add((dw, dh))
            far += bool(np.abs(q).max(0).min() > 33000 or np.abs(q).max() > 1e7)
    assert invalid >= 3 and far >= 4
    assert any(dh >= 16 and dw > 64 for dw, dh in dims) and any(dh == 7 and dw > 146 for dw, dh in dims)
    assert any(dw == 200 for dw, _ in dims) and any(dh == 31 for _, dh in dims)
    assert any(dh == 1 for _, dh in dims) and {1, 2, 3} <= {dw for dw, _ in dims}
    assert any(dw == 199 and dh > 1 for dw, dh in dims)               # (200 / w) * w just below 200


def test_zero_side_dsize_is_unpinned():
    """Where int(scale * w) or int(scale * h) is 0, cv2.warpPerspective falls back to the source size and warpBox's
    paste into the 31x200 crop fails; the kernel writes an all-zero crop (DESIGN.md).  The case set has such boxes."""
    seen = 0
    for g in GROUPS:
        for q, i in zip(g["quads"], g["image_index"]):
            crop, plan = R.warp_box(g["gray"][i], q)
            if _zero_side(plan):
                assert not crop.any()
                with pytest.raises(ValueError):
                    imageops.warp_box(g["gray"][i], q)
                seen += 1
    assert seen >= 3


def test_vectorised_sampler_equals_loop_model():
    """warp_sample == cvmodels.warp_model (the per-pixel loop) on a subset: both block layouts, boxes across every
    edge, the 1-row and 1-column images and the distant boxes."""
    checked = 0
    for g in GROUPS:
        step = 7 if g["name"] == "page" else 3
        for k in range(0, len(g["quads"]), step):
            q, img = g["quads"][k], g["gray"][g["image_index"][k]]
            try:
                fwd, dw, dh = R.warp_transform(q)
            except ZeroDivisionError:
                continue
            if min(dw, dh) == 0:
                continue
            full = np.zeros((R.CROP_H, R.CROP_W), np.uint8)
            full[:dh, :dw] = M.warp_model(img, fwd, dw, dh)
            assert np.array_equal(R.warp_sample(img, M.inv3(fwd).reshape(-1), dw, dh), full), (g["name"], k)
            checked += 1
    assert checked >= 20


def test_crops_to_input_layout():
    crops = np.random.default_rng(0).integers(0, 256, (2, 31, 200, 3), dtype=np.uint8)
    x = R.crops_to_input(crops)
    assert x.shape == (2, 200, 31, 3) and x.dtype == np.float16
    assert x[1, 17, 4, 2] == np.float16(np.float32(crops[1, 26, 17, 2]) / np.float32(255))
    assert np.array_equal(R.crops_to_input(crops[..., 0]), x[..., 0])


@pytest.mark.parametrize("case", R.resize_cases(), ids=[c[0] for c in R.resize_cases()])
def test_resize_model_equals_cv2(case):
    _, hs, ws, hr, wr = case
    src = np.random.default_rng(hs * 7919 + ws).integers(0, 256, (hs, ws, 3), dtype=np.uint8)
    assert np.array_equal(M.resize_model(src, wr, hr), cv2.resize(src, dsize=(wr, hr)))


def test_gray_reference_equals_cv2_on_every_triplet():
    img = R.all_rgb_triplets()
    assert np.array_equal(R.gray_of(img), cv2.cvtColor(img, cv2.COLOR_RGB2GRAY))
