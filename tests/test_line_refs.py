"""The text-line definition (DESIGN.md section 1, "Text lines") on hand-built layouts whose answers are written out, and
its properties, through the fp64 reference (tests/line_refs.py) that the GPU test holds b2o_group_lines to."""
import math

import cv2
import numpy as np
import pytest

from tests import line_refs as R

H = 20.0


def words(groups):
    return [w.tolist() for _, w in groups]


def test_one_line():
    boxes = R.row(10, 10, [40, 60, 30], H, 12)
    g = R.group_lines([boxes[k] for k in (2, 0, 1)])
    assert words(g) == [[1, 2, 0]]
    np.testing.assert_array_equal(g[0][0], [[10, 10], [164, 10], [164, 30], [10, 30]])


def test_two_close_lines_stay_apart():
    # line pitch 1.2 h: the centres are 1.2 h apart across the line, beyond offset_ratio * h
    boxes = R.row(10, 10, [40, 60, 30], H, 12) + R.row(10, 10 + 1.2 * H, [50, 30, 30], H, 12)
    assert words(R.group_lines(boxes)) == [[0, 1, 2], [3, 4, 5]]
    assert words(R.group_lines(boxes[3:] + boxes[:3])) == [[3, 4, 5], [0, 1, 2]]


@pytest.mark.parametrize("angle", [30, -30])
def test_tilted_lines(angle):
    boxes = (R.row(300, 300, [40, 60, 30], H, 12, angle_deg=angle, origin=(300, 300))
             + R.row(300, 330, [40, 60, 30], H, 12, angle_deg=angle, origin=(300, 300)))
    perm = [4, 0, 5, 2, 1, 3]
    g = R.group_lines([boxes[k] for k in perm])
    assert [[perm[k] for k in w] for w in words(g)] == [[0, 1, 2], [3, 4, 5]]
    u = g[0][0][1].astype(np.float64) - g[0][0][0]
    assert math.degrees(math.atan2(u[1], u[0])) == pytest.approx(angle, abs=1e-4)


def test_quarter_turned_page_with_rolled_corners():
    # text reading downwards, box[0] at each word's own top-left (what rotations return): the first line is the one
    # furthest in -N = +x
    boxes = (R.row(100, 100, [40, 60, 30], H, 12, angle_deg=90, origin=(100, 100))
             + R.row(100, 130, [40, 60, 30], H, 12, angle_deg=90, origin=(100, 100)))
    g = R.group_lines(boxes[::-1])
    assert words(g) == [[5, 4, 3], [2, 1, 0]]
    np.testing.assert_array_equal(g[0][0], [[100, 100], [100, 254], [80, 254], [80, 100]])


def test_upside_down_words_do_not_join_upright_ones():
    up = R.row(10, 10, [40, 40], H, 12)
    down = [R.word_box(10 + 2 * 52, 10, 40, H, turn=2)]          # same row, read right to left
    assert not R.link_matrix(up + down)[1, 2]
    assert words(R.group_lines(up + down)) == [[0, 1], [2]]


def test_two_columns_with_a_gutter_wider_than_the_gap():
    gutter = 1.5 * H + 1
    left = R.row(10, 10, [40, 60], H, 12) + R.row(10, 40, [50, 50], H, 12)
    right = R.row(10 + 112 + gutter, 10, [40, 50], H, 12) + R.row(10 + 112 + gutter, 40, [30, 30], H, 12)
    g = R.group_lines(left + right)
    # lines of the two columns at one height tie on m . N_D and go left to right by m . D; the documented limit:
    # columns interleave
    assert words(g) == [[0, 1], [4, 5], [2, 3], [6, 7]]
    assert words(R.group_lines(R.row(10, 10, [40, 60], H, 12) + R.row(10 + 112 + 1.5 * H - 0.5, 10, [40], H, 12))) \
        == [[0, 1, 2]]


def test_title_twice_the_body_height():
    title = R.row(10, 10, [120, 160], 2 * H, 24)
    body = R.row(10, 70, [40, 60, 30, 50], H, 12) + R.row(10, 100, [60, 30], H, 12)
    g = R.group_lines(body + title)
    assert words(g) == [[6, 7], [0, 1, 2, 3], [4, 5]]


def test_chain_links_through_the_middle_word():
    boxes = R.row(10, 10, [40, 40, 40], H, 25)           # gaps 25 <= 30 pairwise, A..C 90 apart
    m = R.link_matrix(boxes)
    assert m[0, 1] and m[1, 2] and not m[0, 2]
    assert words(R.group_lines(boxes[::-1])) == [[2, 1, 0]]


def test_zero_width_and_zero_height_boxes_stand_alone():
    boxes = R.row(10, 10, [40, 40], H, 12)
    zero_w = R.word_box(55, 10, 0, H)
    zero_h = R.word_box(60, 10, 20, 0)
    g = R.group_lines(boxes + [zero_w, zero_h])
    assert not R.link_matrix(boxes + [zero_w, zero_h])[:, 2:].any()
    assert sorted(words(g)) == [[0, 1], [2], [3]]
    for box, w in g:
        if w.tolist() == [2]:
            np.testing.assert_array_equal(box, zero_w)       # U = (1, 0) for a zero-width word


def test_exact_key_ties():
    a = R.word_box(10, 10, 40, H)
    b = R.word_box(62, 10, 40, H)
    # a duplicate word ties on c . U: word index decides
    assert words(R.group_lines([b, a, b])) == [[1, 0, 2]]
    # zero-width words never link; two at one place tie on both line keys: lowest word index first
    z = R.word_box(500, 500, 0, H)
    assert words(R.group_lines([z, a, z, b])) == [[1, 3], [0], [2]]
    # -0.0 and +0.0 keys are one tie
    za, zb = R.word_box(-20, -10, 40, H), R.word_box(-20, -10, 40, H)
    zb[:, 0] = np.where(zb[:, 0] == 0, -0.0, zb[:, 0])
    assert words(R.group_lines([zb, za])) == [[0, 1]]


# ---------------------------------------------------------------------------------------------- properties
def random_layout(seed, n_lines=6, tilt=0.0, turn=0):
    rng = np.random.default_rng(seed)
    boxes = []
    for l in range(n_lines):
        widths = rng.uniform(20, 80, rng.integers(1, 7))
        boxes += R.row(40 + rng.uniform(0, 30), 40 + 40 * l + rng.uniform(-2, 2), widths, rng.uniform(16, 22),
                       rng.uniform(6, 20), angle_deg=tilt, origin=(200, 200), turn=turn)
    return np.stack(boxes)


def line_sets(groups, perm=None):
    perm = np.arange(10 ** 6) if perm is None else np.asarray(perm)
    return sorted(sorted(perm[w].tolist()) for _, w in groups)


@pytest.mark.parametrize("seed", range(6))
def test_link_relation_is_symmetric(seed):
    b = random_layout(seed, tilt=[0, 7, -12, 30, 88, 180][seed])
    b[::5] = b[::5][:, [0, 0, 2, 3]]                   # zero-width words among them
    m = R.link_matrix(b)
    assert np.array_equal(m, m.T) and m.any()


@pytest.mark.parametrize("seed", range(4))
def test_lines_do_not_depend_on_input_order(seed):
    b = random_layout(seed, tilt=5.0 * seed)
    perm = np.random.default_rng(seed).permutation(len(b))
    assert line_sets(R.group_lines(b[perm]), perm) == line_sets(R.group_lines(b))


@pytest.mark.parametrize("factor", [2.0, 0.5])
def test_power_of_two_scale_gives_identical_lines(factor):
    b = random_layout(7, tilt=11.0)
    g, s = R.group_lines(b), R.group_lines((b * np.float32(factor)).astype(np.float32))
    assert words(g) == words(s)
    for (box, _), (box2, _) in zip(g, s):
        np.testing.assert_array_equal(box * np.float32(factor), box2)


def test_quarter_turn_with_rolled_corners_gives_the_same_lines():
    b = random_layout(8, tilt=3.0)
    turned = np.stack([b[..., 1] * -1, b[..., 0]], -1).astype(np.float32)     # (x, y) -> (-y, x), exact
    g, t = R.group_lines(b), R.group_lines(turned)
    assert words(g) == words(t)
    for (box, _), (box2, _) in zip(g, t):
        np.testing.assert_array_equal(np.stack([-box[:, 1], box[:, 0]], -1), box2)


@pytest.mark.parametrize("seed", range(4))
def test_member_corners_lie_inside_the_line_box(seed):
    b = random_layout(seed, tilt=[0, 9, -21, 44][seed])
    for box, w in R.group_lines(b):
        q = box.astype(np.float64)
        ulp = float(np.spacing(np.float32(np.abs(q).max())))
        for k in range(4):                              # signed distance to each edge, positive inside (clockwise)
            e = q[(k + 1) % 4] - q[k]
            d = (e[0] * (b[w].reshape(-1, 2)[:, 1] - q[k][1]) - e[1] * (b[w].reshape(-1, 2)[:, 0] - q[k][0]))
            assert (d / np.linalg.norm(e) >= -ulp).all(), (k, d.min() / np.linalg.norm(e), ulp)


@pytest.mark.parametrize("tilt", [0.0, 10.0, -25.0])
def test_collinear_line_box_is_the_min_area_rectangle(tilt):
    rng = np.random.default_rng(int(tilt) + 40)
    b = np.stack(R.row(100, 100, rng.uniform(20, 80, 5), H, 10, angle_deg=tilt, origin=(150, 110)))
    (box, w), = R.group_lines(b)
    # tools.combine_line's point set: the top edges left to right, then the bottom edges right to left
    pts = np.concatenate([b[k][:2] for k in w] + [b[k][[3, 2]] for k in w[::-1]]).astype(np.float32)
    (_, (rw, rh), _) = cv2.minAreaRect(pts)
    area = np.linalg.norm(box[1] - box[0]) * np.linalg.norm(box[3] - box[0])
    assert area == pytest.approx(rw * rh, rel=0.02)


def test_check_lines_validates_and_normalises():
    from keras_ocr_b200 import detection

    assert detection.check_lines() == R.DEFAULTS
    assert detection.check_lines(angle_tolerance=90, gap_ratio=0) == {**R.DEFAULTS, "angle_tolerance": 90.0,
                                                                       "gap_ratio": 0.0}
    bad = [{"angle": 10}, {"angle_tolerance": 0}, {"angle_tolerance": 91}, {"height_ratio": 0},
           {"height_ratio": 1.5}, {"offset_ratio": 0}, {"gap_ratio": -1}, {"gap_ratio": float("nan")},
           {"offset_ratio": float("inf")}, {"height_ratio": "0.5"}, {"angle_tolerance": True}]
    for kw in bad:
        with pytest.raises(ValueError):
            detection.check_lines(**kw)
