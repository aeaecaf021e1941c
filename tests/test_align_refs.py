"""CPU: the character-position references of tests/align_refs.py -- Viterbi against brute force, the greedy runs, and
the cell geometry against cv2.getPerspectiveTransform / cv2.perspectiveTransform."""
import numpy as np
import pytest

from tests import align_refs as AR
from tests import image_refs as IR
from tests import rotation_refs as RR
from tests.test_rotation_refs import rot90_points


def _dyadic(rng, t, k):
    """lp with values on a coarse dyadic grid: sums are exact in fp64, so equal-scoring alignments tie exactly."""
    return -rng.integers(0, 6, (t, k)).astype(np.float64) / 4.0


@pytest.mark.parametrize("t,k", [(4, 3), (5, 3), (6, 3), (5, 4)])
def test_viterbi_equals_brute_force(t, k):
    rng = np.random.default_rng(t * 10 + k)
    seqs = [(), (0,), (1,), (0, 0), (0, 1), (1, 0, 1), (0, 0, 0), (1, 1, 0), (0, 1, 0, 1), (0, 0, 1, 1), (k - 1,),
            (0, 0, 0, 0), tuple(range(min(k - 1, 3)))]
    ties = unalignable = 0
    for trial in range(12):
        lp = _dyadic(rng, t, k) if trial % 2 else np.log(rng.dirichlet(np.ones(k), t) + 1e-7)
        for seq in seqs:
            score, spans, margin = AR.viterbi(lp, seq)
            ref_score, ref_spans = AR.brute_force(lp, seq)
            if ref_score == -np.inf:
                unalignable += 1
                assert score == -np.inf and (spans == -1).all(), seq
                continue
            assert np.isclose(score, ref_score, rtol=0, atol=1e-12), (seq, score, ref_score)
            assert np.array_equal(spans, ref_spans), (trial, seq, spans, ref_spans)
            ties += margin == 0
    assert ties > 0 and unalignable > 0          # the tie rule and -inf were exercised


def test_viterbi_spans_follow_states():
    """Doubled letters need a blank between their copies; leading and trailing blanks are allowed."""
    k, blank = 3, 2
    lp = np.full((6, k), -5.0)
    for t, c in enumerate([blank, 0, blank, 0, 0, blank]):
        lp[t, c] = 0.0
    score, spans, _ = AR.viterbi(lp, (0, 0))
    assert score == 0.0 and spans.tolist() == [[1, 1], [3, 4]]
    assert AR.viterbi(lp[:2], (0, 0))[0] == -np.inf          # 2 steps cannot hold "aa"


def test_greedy_runs_are_viterbi_spans():
    """Without ties, the argmax path is the best alignment of its own collapse: the spans are its runs."""
    rng = np.random.default_rng(7)
    checked = 0
    for i in range(40):
        k = [3, 5, 37][i % 3]
        x = rng.normal(size=(AR.STEPS, k)) * 3
        x[:, k - 1] += rng.uniform(0, 4)
        lp = np.log(np.exp(x) / np.exp(x).sum(1, keepdims=True) + 1e-7)
        labels, runs = AR.greedy_runs(lp)
        score, spans, margin = AR.viterbi(lp, labels)
        assert margin > 0
        assert np.isclose(score, lp.max(1).sum(), rtol=0, atol=1e-9)
        assert np.array_equal(spans, runs), i
        checked += len(labels)
    assert checked > 100


def _cv2_cells(quad, turn, cuts_x):
    """Crop points (x, 0) / (x, sh) mapped by cv2: getPerspectiveTransform of the rolled box onto its crop, inverted by
    perspectiveTransform with the inverse matrix."""
    import cv2
    from oracle import imageops
    box = RR.turned_box(quad, turn)
    w, h = imageops.rotated_width_height(box)
    scale = min(200 / w, 31 / h)
    dst = np.array([[0, 0], [scale * w, 0], [scale * w, scale * h], [0, scale * h]]).astype("float32")
    inv = np.linalg.inv(cv2.getPerspectiveTransform(box, dst))
    sh = float(dst[2, 1])
    pts = np.array([[[x, y] for x in cuts_x for y in (0.0, sh)]], np.float64)
    return cv2.perspectiveTransform(pts, inv)[0].reshape(len(cuts_x), 2, 2), box, float(dst[1, 0])


QUADS = [IR._rect(120, 80, 150, 30, 12), IR._rect(60, 200, 90, 22, -35, 2, True), IR._axis(10.5, 20, 150.5, 48, 1),
         IR._rect(300, 150, 40, 120, 80)]


@pytest.mark.parametrize("turn", [0, 1, 2, 3])
@pytest.mark.parametrize("qi", range(len(QUADS)))
def test_cells_geometry_against_cv2(qi, turn):
    quad = QUADS[qi]
    spans = np.array([[1, 3], [6, 6], [9, 14], [20, 22], [30, 40]], np.int32)
    for theta in (None, np.array([1, 0, 0, 0, 1, 0], np.float32), np.array([0.9, 0.1, 0.0, 0.05, 0.8, -0.1], np.float32),
                  np.array([1, 0, 0, 0, -1, 0], np.float32)):
        got = AR.cells(spans, theta, quad, turn)
        cuts = [AR.cut_x(spans, j, theta) for j in range(1, len(spans))]
        _, box, sw = _cv2_cells(quad, turn, [0.0])
        # closed forms of the cut: identity theta u = 50 r / 49, stn=False u = r
        r = np.array([0.5 * (spans[j - 1, 1] + spans[j, 0]) + 2 for j in range(1, len(spans))])
        if theta is None:
            assert np.allclose(cuts, 4 * r + 1.5, rtol=0, atol=1e-12)
        elif theta[4] == 1 and theta[3] == 0 and theta[5] == 0:
            assert np.allclose(cuts, 4 * (50 * r / 49) + 1.5, rtol=0, atol=1e-12)
        # outer edges are the rolled box's corners, bit for bit; the cells tile the box in reading order
        assert np.array_equal(got[0, [0, 3]], box[[0, 3]]) and np.array_equal(got[-1, [1, 2]], box[[1, 2]])
        assert np.array_equal(got[1:, 0], got[:-1, 1]) and np.array_equal(got[1:, 3], got[:-1, 2])
        # cuts are clamped and non-decreasing (a time-flipping theta collapses them at one edge)
        xs = [0.0]
        for c in cuts:
            xs.append(max(xs[-1], min(max(c, 0.0), sw)))
        assert all(a <= b for a, b in zip(xs, xs[1:]))
        ref_pts, _, _ = _cv2_cells(quad, turn, xs[1:])
        assert np.allclose(got[1:, 0], ref_pts[:, 0], rtol=0, atol=1e-3)
        assert np.allclose(got[1:, 3], ref_pts[:, 1], rtol=0, atol=1e-3)


def test_one_character_is_the_word_box():
    for quad in QUADS:
        for turn in range(4):
            got = AR.cells(np.array([[0, 47]], np.int32), np.array([1, 0, 0, 0, 1, 0], np.float32), quad, turn)
            assert np.array_equal(got[0], RR.turned_box(quad, turn))


def test_crop_frame_cells():
    spans = np.array([[2, 4], [10, 12], [30, 31]], np.int32)
    got = AR.cells(spans)
    assert got[0, 0].tolist() == [0, 0] and got[-1, 2].tolist() == [200, 31]
    assert np.isclose(got[0, 1, 0], 4 * ((4 + 10) / 2 + 2) + 1.5) and got[1, 2, 1] == 31


def test_degenerate_box_gives_nan():
    assert np.isnan(AR.cells(np.array([[0, 3]], np.int32), None, IR._axis(50, 50, 50.6, 80))).all()


@pytest.mark.parametrize("k", [1, 2, 3])
def test_cells_on_turned_page_map_back_upright(k):
    """An upright box on np.rot90(page, k), read in turn (4 - k) % 4, has the cells of the upright box, rotated.  (Boxes
    tilted away from the axes may order their corners one place further round after the turn; the axis-parallel ones
    here do not.)"""
    h, w = 300, 400
    spans = np.array([[0, 2], [5, 9], [12, 12], [20, 30]], np.int32)
    theta = np.array([0.95, 0.05, 0.0, 0.02, 0.9, 0.03], np.float32)
    for quad in (IR._axis(10.5, 20, 150.5, 48, 1), IR._axis(200, 100, 390.25, 131), IR._axis(3, 250, 97, 290.5, 3)):
        up = AR.cells(spans, theta, quad, 0)
        turned = AR.cells(spans, theta, rot90_points(quad, k, h, w), (4 - k) % 4)
        back = rot90_points(turned.reshape(-1, 2), (4 - k) % 4, *((w, h) if k % 2 else (h, w))).reshape(up.shape)
        assert np.allclose(back, up, rtol=0, atol=2e-3), (k, np.abs(back - up).max())
