"""CPU: the polygon reference (tests/polygon_refs.py) on shapes with a known centre line, the piecewise warp reference
against warpBox, and the host validation of polygons."""
import numpy as np
import pytest

from tests import image_refs, polygon_refs as P


def _poly_of(seg):
    blob, contour = P.filled_blob(seg)
    box = P.box_of(contour)
    return blob, box, P.polygon(blob, box, centre=True)


@pytest.mark.parametrize("angle", range(0, 180, 15))
def test_straight_bands_keep_their_rectangle(angle):
    blob, box, (poly, points, line) = _poly_of(P.straight_band(angle))
    assert points == 4 and line is None
    np.testing.assert_array_equal(poly[:4], 2 * box)
    assert np.isnan(poly[4:]).all()


def _check_curve(seg, dist, cover, interior, ends):
    """The polygon covers ``cover`` of the blob; its centre line q_1 .. q_S-1 lies within ``interior`` score-map px of
    the analytic curve and its ends q_0, q_S within ``ends``.  The centre line chords the curve: its interior points sit
    inside a bend by about a band's sagitta, and the ends extend the end chords, so the bounds grow with the bend."""
    blob, box, (poly, points, line) = _poly_of(seg)
    assert points >= 8, points                     # at least 3 segments
    assert np.isnan(poly[points:]).all() and np.isfinite(poly[:points]).all()
    assert P.covered(poly, points, blob) >= cover
    d = dist(line)
    assert d[1:-1].max() <= interior, d
    assert max(d[0], d[-1]) <= ends, d
    return points


# (sweep, radius, interior bound, end bound) in score-map px, thickness 9.  Measured (worst of both rotations,
# interior / ends): 30/200 0.53 / 0.50; 60/80 0.28 / 1.02; 90/80 0.6 / 1.74; 120/80 1.0 / 3.12; 150/80 1.93 / 5.16;
# 180/80 3.53 / 8.94.  Up to 90 degrees the centre line stays within 1 px of the arc; beyond, it does not.
ARCS = [(30, 200, 1.0, 1.0), (60, 80, 1.0, 1.5), (90, 80, 1.0, 2.0), (120, 80, 1.5, 3.5), (150, 80, 2.0, 5.5),
        (180, 80, 4.0, 9.5)]


@pytest.mark.parametrize("sweep, radius, interior, ends", ARCS)
@pytest.mark.parametrize("rotate", [0.0, 35.0])
def test_arcs_give_polygons_along_the_arc(sweep, radius, interior, ends, rotate):
    seg, dist = P.arc_band(sweep, radius=radius, rotate_deg=rotate)
    _check_curve(seg, dist, 0.99, interior, ends)


def test_a_slight_bend_keeps_its_rectangle():
    """A 30 degree arc of radius 80 bends its centroids by less than a quarter of its thickness: straight enough."""
    seg, _ = P.arc_band(30, radius=80)
    assert _poly_of(seg)[2][1] == 4


@pytest.mark.parametrize("amplitude", [6, 10, 14])
def test_sine_bands_give_polygons_along_the_curve(amplitude):
    """An S-curve's bands are not arcs of one circle: the polygon covers 98.8 % of the blob (measured 98.85 % at the
    largest amplitude), its interior points lie within 4 px of the curve (measured 1.72, 2.75, 3.79) and its ends within
    6 px (4.23, 4.92, 5.69)."""
    seg, dist = P.sine_band(amplitude)
    _check_curve(seg, dist, 0.988, 4.0, 6.0)


def test_polygon_is_clockwise_from_the_top_left():
    seg, _ = P.arc_band(120)
    _, _, (poly, points, _) = _poly_of(seg)
    p = poly[:points].astype(np.float64)
    area = 0.5 * (np.dot(p[:, 0], np.roll(p[:, 1], -1)) - np.dot(p[:, 1], np.roll(p[:, 0], -1)))
    assert area > 0                                  # clockwise in image coordinates (y down)
    s = points // 2 - 1
    assert p[0, 0] < p[s, 0]                         # the top edge runs left to right


def _rect(x0, y0, w, h, deg):
    return image_refs._rect(x0, y0, w, h, deg)


@pytest.mark.parametrize("deg", [0.0, 12.0, -27.0, 45.0])
def test_one_segment_warp_is_warpbox(deg):
    rng = np.random.default_rng(1)
    img = rng.integers(0, 256, (90, 130), dtype=np.uint8)
    from oracle import imageops
    box = imageops.order_corners(_rect(60, 45, 80, 20, deg)).astype(np.float32)
    # the piecewise rule with s = 1: (t_0, t_1) = (tl, tr), (b_1, b_0) = (br, bl)
    poly = np.full((P.POLY_POINTS, 2), np.nan, np.float32)
    poly[:4] = box
    lay = P.warp_layout(np.concatenate([box[:2], box[2:]]), 4)
    assert lay is not None
    import cv2
    s, dw, dh, X, sh = lay
    src = np.array([box[0], box[1], box[2], box[3]], np.float32)
    dst = np.array([[X[0], 0], [X[1], 0], [X[1], sh], [X[0], sh]], np.float32)
    full = cv2.warpPerspective(img, cv2.getPerspectiveTransform(src, dst), (dw, dh), flags=cv2.INTER_LINEAR,
                               borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    got = np.zeros((31, 200), np.uint8)
    got[:min(dh, 31), :min(dw, 200)] = full[:31, :200]
    want, plan = image_refs.warp_box(img, box)
    assert plan is not None and (plan[1], plan[2]) == (dw, dh)
    np.testing.assert_array_equal(got, want)


def test_piecewise_warp_of_a_straight_polygon_matches_the_box_width():
    rng = np.random.default_rng(2)
    img = rng.integers(0, 256, (80, 160), dtype=np.uint8)
    top = np.stack([np.linspace(10, 150, 5), np.full(5, 20.0)], -1)
    bot = np.stack([np.linspace(10, 150, 5), np.full(5, 44.0)], -1)
    poly = np.concatenate([top, bot[::-1]]).astype(np.float32)
    crop = P.warp_poly(img, poly, 10)
    want, _ = image_refs.warp_box(img, np.array([[10, 20], [150, 20], [150, 44], [10, 44]], np.float32))
    s, dw, dh, X, sh = P.warp_layout(poly, 10)
    assert (dw, dh) == (int(want.any(0).sum()) or dw, dh)
    assert np.abs(crop.astype(int) - want.astype(int)).max() <= 1      # equal segments of one affine map


@pytest.mark.parametrize("entry, what", [
    (np.zeros((5, 2)), "odd"),
    (np.zeros((20, 2)), "points"),
    (np.zeros((2, 2)), "points"),
    (np.array([[0, 0], [10, 0], [20, 0], [20, 5], [10, np.nan], [0, 5]], np.float32), "non-finite"),
    (np.array([[0, 0], [10, 0], [20, 0], [20, 5], [10, 0], [0, 5]], np.float32), "degenerate"),
    (np.array([[0, 0], [0, 0], [20, 0], [20, 5], [0, 5], [0, 5]], np.float32), "degenerate"),
    (np.zeros((4, 3)), "shape"),
])
def test_check_polygons_rejects_malformed_entries(entry, what):
    from keras_ocr_b200 import recognition
    good = np.array([[0, 0], [10, 0], [20, 2], [20, 8], [10, 6], [0, 6]], np.float32)
    with pytest.raises(ValueError, match=f"entry 1 .*{what}|entry 1 has.*{what}"):
        recognition.check_polygons([good, entry, good])


def test_check_polygons_lays_out_the_dense_table():
    from keras_ocr_b200 import recognition
    box = np.array([[0, 0], [10, 0], [10, 5], [0, 5]], np.float32)
    poly = np.array([[0, 0], [10, 0], [20, 2], [20, 8], [10, 6], [0, 6]], np.float32)
    polys, points = recognition.check_polygons([box, poly])
    assert polys.shape == (2, P.POLY_POINTS, 2) and polys.dtype == np.float32
    np.testing.assert_array_equal(points, [4, 6])
    np.testing.assert_array_equal(polys[0, :4], box)
    np.testing.assert_array_equal(polys[1, :6], poly)
    assert np.isnan(polys[0, 4:]).all() and np.isnan(polys[1, 6:]).all()
