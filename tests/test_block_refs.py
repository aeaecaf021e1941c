"""The text-block definition (DESIGN.md section 1, "Text blocks") on hand-built layouts whose answers are written out,
and its properties, through the fp64 reference (tests/block_refs.py) that the GPU test holds b2o_group_blocks to.

Lines are 20 high unless said otherwise, so s = 20, a row cut needs a gap of 1.5 * 20 = 30 and a column cut one of
1.0 * 20 = 20.  Line pitch 30 (a gap of 10) keeps a column's lines in one block."""
import numpy as np
import pytest

from tests import block_refs as R

H = 20.0


def blocks(lines, sizes=None, **params):
    sizes = np.full(len(lines), 3, np.int32) if sizes is None else np.asarray(sizes, np.int32)
    return [b.tolist() for _, b in R.group_blocks(np.stack(lines), sizes, **params)]


def interleave(*cols):
    """Lines of side-by-side columns in page order as b2o_group_lines returns them: by height, then left to right."""
    out = []
    for row in zip(*cols):
        out += list(row)
    return out


def test_one_column():
    g = R.group_blocks(np.stack(R.column(10, 10, 200, H, 30, 5)), np.full(5, 3))
    assert [b.tolist() for _, b in g] == [[0, 1, 2, 3, 4]]
    np.testing.assert_array_equal(g[0][0], [[10, 10], [210, 10], [210, 150], [10, 150]])


def test_two_columns():
    lines = interleave(R.column(0, 0, 200, H, 30, 4), R.column(240, 0, 200, H, 30, 4))
    assert blocks(lines) == [[0, 2, 4, 6], [1, 3, 5, 7]]


def test_three_columns():
    lines = interleave(R.column(0, 0, 150, H, 30, 3), R.column(180, 0, 150, H, 30, 3), R.column(360, 0, 150, H, 30, 3))
    assert blocks(lines) == [[0, 3, 6], [1, 4, 7], [2, 5, 8]]


def test_title_over_two_columns():
    title = R.line_box(0, 0, 440, 2 * H)                    # 40 high; the body starts 40 below it
    lines = [title] + interleave(R.column(0, 80, 200, H, 30, 4), R.column(240, 80, 200, H, 30, 4))
    assert blocks(lines) == [[0], [1, 3, 5, 7], [2, 4, 6, 8]]


def test_two_columns_with_a_full_width_footer():
    lines = interleave(R.column(0, 0, 200, H, 30, 4), R.column(240, 0, 200, H, 30, 4)) + [R.line_box(0, 150, 440, H)]
    assert blocks(lines) == [[0, 2, 4, 6], [1, 3, 5, 7], [8]]


@pytest.mark.parametrize("gap,split", [(31.0, True), (29.0, False)])
def test_paragraph_break(gap, split):
    lines = R.column(0, 0, 200, H, 30, 3) + R.column(0, 80 + gap, 200, H, 30, 3)     # line 2 ends at 80
    assert blocks(lines) == ([[0, 1, 2], [3, 4, 5]] if split else [[0, 1, 2, 3, 4, 5]])


def test_label_value_rows():
    labels = R.column(0, 0, 60, H, 30, 3)
    values = R.column(300, 0, 100, H, 30, 3)
    assert blocks(interleave(labels, values)) == [[0, 2, 4], [1, 3, 5]]
    assert blocks([labels[0], values[0]]) == [[0], [1]]      # a single "label ... value" row: two blocks


def test_aligned_paragraph_breaks_split_the_page_into_bands():
    # both columns break at the same height: the row cut runs across the page first, each band is read left, right
    left = R.column(0, 0, 200, H, 30, 2) + R.column(0, 100, 200, H, 30, 2)
    right = R.column(240, 0, 200, H, 30, 2) + R.column(240, 100, 200, H, 30, 2)
    assert blocks(interleave(left, right)) == [[0, 2], [1, 3], [4, 6], [5, 7]]


def _nudge(v, k):
    v = np.float32(v)
    for _ in range(abs(k)):
        v = np.nextafter(v, np.float32(np.inf if k > 0 else -np.inf))
    return v


@pytest.mark.parametrize("k", [-1, 0, 1])
def test_row_gap_exactly_at_the_threshold(k):
    # line 1's top edge at 20 + 30 = 50 exactly at k = 0; line 2 beside line 0 keeps the median height at 20
    top, beside = R.line_box(0, 0, 200, H), R.line_box(210, 0, 100, H)
    low = R.line_box(0, 50, 200, H)
    low[:2, 1] = _nudge(50, k)
    assert blocks([top, low, beside], sizes=[3, 1, 1]) == ([[0, 2], [1]] if k >= 0 else [[0, 1, 2]])


@pytest.mark.parametrize("k", [-1, 0, 1])
def test_col_gap_exactly_at_the_threshold(k):
    # line 1's left edge at 200 + 20 = 220 exactly at k = 0
    left, right = R.line_box(0, 0, 200, H), R.line_box(220, 0, 100, H)
    right[[0, 3], 0] = _nudge(220, k)
    below = R.line_box(0, 30, 200, H)
    assert blocks([left, right, below], sizes=[3, 1, 1]) == ([[0, 2], [1]] if k >= 0 else [[0, 1, 2]])


def test_page_frame_and_parameters():
    # the page frame is the line with the most words: read as a quarter-turned page, the two columns are rows
    lines = interleave(R.column(0, 0, 200, H, 30, 2), R.column(240, 0, 200, H, 30, 2))
    assert blocks(lines, row_gap=0.5) == [[0], [1], [2], [3]]   # a gap of 10 >= 0.5 * 20 cuts rows, then columns
    assert blocks(lines, col_gap=2.01) == [[0, 1, 2, 3]]     # the gutter of 40 < 2.01 * 20
    turned = [np.stack([q[:, 1], -q[:, 0]], -1).astype(np.float32) for q in lines]   # read downwards, box[0] rolled
    assert blocks(turned) == [[0, 2], [1, 3]]


def test_spiral_cuts_one_line_per_level():
    b, s = R.spiral(12)
    assert [w.tolist() for _, w in R.group_blocks(b, s)] == [[0], [3], [4], [7], [8], [11], [10], [9], [6], [5], [2],
                                                               [1]]


# ---------------------------------------------------------------------------------------------- properties
def page(seed, count=60, tilt=0.0):
    return R.random_page(np.random.default_rng(seed), count, tilt=tilt)


def block_lists(g):
    return [w.tolist() for _, w in g]


@pytest.mark.parametrize("factor", [2.0, 0.5, 0.25])
def test_power_of_two_scale_gives_identical_blocks(factor):
    b, s = page(3, tilt=7.0)
    g, t = R.group_blocks(b, s), R.group_blocks((b * np.float32(factor)).astype(np.float32), s)
    assert block_lists(g) == block_lists(t)
    for (box, _), (box2, _) in zip(g, t):
        np.testing.assert_array_equal(box * np.float32(factor), box2)


@pytest.mark.parametrize("seed", range(3))
def test_integer_translation_of_an_integer_layout_gives_identical_blocks(seed):
    b, s = page(seed)
    lo, hi = np.round(b.min(1)), np.round(b.max(1))            # axis-aligned integer boxes around the random lines
    b = np.stack([lo, np.stack([hi[:, 0], lo[:, 1]], 1), hi, np.stack([lo[:, 0], hi[:, 1]], 1)], 1).astype(np.float32)
    g, t = R.group_blocks(b, s), R.group_blocks(b + np.float32([137, -59]), s)
    assert block_lists(g) == block_lists(t)
    for (box, _), (box2, _) in zip(g, t):
        np.testing.assert_array_equal(box + np.float32([137, -59]), box2)


@pytest.mark.parametrize("turns", [1, 2, 3])
def test_quarter_turns_give_identical_blocks(turns):
    b, s = page(4, tilt=5.0)
    t = b
    for _ in range(turns):                                   # (x, y) -> (-y, x), exact; corners keep their roles
        t = np.stack([-t[..., 1], t[..., 0]], -1).astype(np.float32)
    g, r = R.group_blocks(b, s), R.group_blocks(t, s)
    assert block_lists(g) == block_lists(r)
    for (box, _), (box2, _) in zip(g, r):
        for _ in range(turns):
            box = np.stack([-box[:, 1], box[:, 0]], -1)
        np.testing.assert_array_equal(box, box2)


@pytest.mark.parametrize("seed", range(6))
def test_blocks_partition_the_lines_and_contain_them(seed):
    b, s = page(seed + 10, count=80, tilt=[0, 4, -9, 90, 180, 2][seed])
    g = R.group_blocks(b, s)
    got = sorted(l for _, w in g for l in w.tolist())
    assert got == list(range(len(b)))
    for box, w in g:
        assert w.tolist() == sorted(w.tolist())
        q = box.astype(np.float64)
        ulp = float(np.spacing(np.float32(np.abs(q).max())))
        pts = b[w].reshape(-1, 2).astype(np.float64)
        for k in range(4):                                   # signed distance to each edge, positive inside
            e = q[(k + 1) % 4] - q[k]
            d = e[0] * (pts[:, 1] - q[k][1]) - e[1] * (pts[:, 0] - q[k][0])
            assert (d / np.linalg.norm(e) >= -2 * ulp).all()


def test_empty_and_single_line():
    assert R.group_blocks(np.zeros((0, 4, 2), np.float32), np.zeros(0, np.int32)) == []
    (box, w), = R.group_blocks(R.line_box(5, 5, 0, 0)[None], [0])     # a degenerate box: D = (1, 0)
    assert w.tolist() == [0]
    np.testing.assert_array_equal(box, [[5, 5]] * 4)


def test_check_blocks_validates_and_normalises():
    from keras_ocr_b200 import detection

    assert detection.check_blocks() == R.DEFAULTS
    assert detection.check_blocks(row_gap=2, col_gap=0.5) == {"row_gap": 2.0, "col_gap": 0.5}
    for kw in ({"gap": 1}, {"row_gap": 0}, {"col_gap": -1}, {"row_gap": float("nan")}, {"col_gap": float("inf")},
               {"row_gap": "1"}, {"col_gap": True}):
        with pytest.raises(ValueError):
            detection.check_blocks(**kw)


def test_blocks_from_csr():
    from keras_ocr_b200 import detection

    boxes = np.arange(3 * 8, dtype=np.float32).reshape(3, 4, 2)
    got = detection.blocks_from_csr(2, np.array([2, 0, 1, 9], np.int32), np.array([0, 1, 3, 9], np.int32), boxes)
    assert [w.tolist() for _, w in got] == [[2], [0, 1]]
    np.testing.assert_array_equal(got[1][0], boxes[1])
