"""CPU references for the polygons of curved words (keras-ocr_b200/csrc/boxes.cu ``poly_of_blob`` and image.cu
``warp_polys_kernel``), and the seeded shapes the tests run.

``polygon`` restates the polygon stage in fp64 NumPy with the kernel's operation order (separate roundings, no fused
multiply-add) and its order-independent reductions (int64 sums, maxima), so its float32 output equals the kernel's bit
for bit when it is given the kernel's blob and box.  ``component_blobs`` builds that blob with cv2 as getBoxes does
(dilation, findContours(RETR_TREE)[0]) and fills it (drawContours, thickness -1).  ``warp_poly`` is the piecewise
warpBox: cv2.getPerspectiveTransform + cv2.warpPerspective per segment over the full dsize, each segment keeping its
own columns of the crop -- with cv2 itself, or with the pinned models of those two calls that the kernel restates.
"""
import math

import numpy as np

S_MAX = 8                   # B2O_MAX_POLY_SEGMENTS
POLY_POINTS = 2 * (S_MAX + 1)
STRAIGHTNESS = 0.25         # kStraightness: max |v(c_j) - mean v| <= 0.25 t keeps the rectangle
CROP_H, CROP_W = 31, 200


def _unit(du, dv):
    n = math.sqrt(du * du + dv * dv)
    if not n > 0.0:
        return None
    return du / n, dv / n


def polygon(blob, box, centre=False):
    """The polygon of one component: blob (H,W) bool, the filled blob in score-map pixels; box (4,2) float32, its box
    in score-map pixels (tl, tr, br, bl).  Returns (poly (18,2) float32 in detector-input pixels (x2), NaN past the
    points, points) and, with ``centre``, the centre line q_0 .. q_S (S+1,2) float64 in score-map pixels (None for a
    kept rectangle)."""
    box = np.asarray(box, np.float32).astype(np.float64)
    ys, xs = np.nonzero(blob)
    out = np.full((POLY_POINTS, 2), np.nan, np.float32)

    def rect():
        out[:4] = 2 * box.astype(np.float32)
        return (out, 4, None) if centre else (out, 4)

    ox, oy = float(box[0, 0]), float(box[0, 1])
    ux, uy = float(box[1, 0]) - ox, float(box[1, 1]) - oy
    vx, vy = float(box[3, 0]) - ox, float(box[3, 1]) - oy
    W = math.sqrt(ux * ux + uy * uy)
    eu, ev = _unit(ux, uy), _unit(vx, vy)
    cnt = len(xs)
    if cnt == 0 or eu is None or ev is None:
        return rect()
    t = cnt / W
    r = W / t
    S = S_MAX if r >= S_MAX else int(math.floor(r))
    if S < 3:
        return rect()
    (eux, euy), (evx, evy) = eu, ev
    dx, dy = xs.astype(np.float64) - ox, ys.astype(np.float64) - oy
    u = dx * eux + dy * euy
    v = dx * evx + dy * evy
    band = np.clip(np.floor((S * u) / W), 0, S - 1).astype(np.int64)
    cu, cv = np.zeros(S), np.zeros(S)
    vsum = 0.0
    for j in range(S):
        sel = band == j
        n = int(sel.sum())
        if n == 0:
            return rect()
        cx, cy = int(xs[sel].astype(np.int64).sum()) / float(n), int(ys[sel].astype(np.int64).sum()) / float(n)
        ddx, ddy = cx - ox, cy - oy
        cu[j], cv[j] = ddx * eux + ddy * euy, ddx * evx + ddy * evy
        vsum = vsum + cv[j]
    vbar = vsum / S
    dev = 0.0
    for j in range(S):
        dev = max(dev, abs(cv[j] - vbar))
    if not dev > STRAIGHTNESS * t:
        return rect()
    qu, qv = np.zeros(S + 1), np.zeros(S + 1)
    for j in range(1, S):
        qu[j], qv[j] = (cu[j - 1] + cu[j]) * 0.5, (cv[j - 1] + cv[j]) * 0.5
    e0, e1 = _unit(cu[0] - cu[1], cv[0] - cv[1]), _unit(cu[S - 1] - cu[S - 2], cv[S - 1] - cv[S - 2])
    if e0 is None or e1 is None:
        return rect()
    ext = []
    for j, c, e in ((0, 0, e0), (S - 1, S - 1, e1)):
        sel = band == j
        proj = (u[sel] - cu[c]) * e[0] + (v[sel] - cv[c]) * e[1]
        ext.append(max(0.0, float(proj.max())))
    qu[0], qv[0] = cu[0] + ext[0] * e0[0], cv[0] + ext[0] * e0[1]
    qu[S], qv[S] = cu[S - 1] + ext[1] * e1[0], cv[S - 1] + ext[1] * e1[1]
    g = []
    for j in range(S):
        gj = _unit(qu[j + 1] - qu[j], qv[j + 1] - qv[j])
        if gj is None:
            return rect()
        g.append(gj)
    rho_band = np.zeros(S)
    for j in range(S):
        sel = band == j
        d = np.abs((u[sel] - qu[j]) * g[j][1] - (v[sel] - qv[j]) * g[j][0])
        rho_band[j] = max(0.0, float(d.max()))
    for j in range(S + 1):
        a, b = (0 if j == 0 else j - 1), (S if j == S else j + 1)
        tu, tv = _unit(qu[b] - qu[a], qv[b] - qv[a])
        nu, nv = -tv, tu
        rho = 0.0
        if j > 0:
            rho = max(rho, rho_band[j - 1])
        if j < S:
            rho = max(rho, rho_band[j])
        for side, slot in ((-rho, j), (rho, 2 * S + 1 - j)):
            pu, pv = qu[j] + side * nu, qv[j] + side * nv
            X = (ox + pu * eux) + pv * evx
            Y = (oy + pu * euy) + pv * evy
            out[slot] = 2 * np.float32(X), 2 * np.float32(Y)
    if not centre:
        return out, 2 * (S + 1)
    line = np.stack([ox + qu * eux + qv * evx, oy + qu * euy + qv * evy], -1)
    return out, 2 * (S + 1), line


# ------------------------------------------------------------------------------------------------ blobs with cv2
def filled_blob(seg):
    """cv2.findContours(RETR_TREE)[0] of a uint8 segmap, drawn filled: the blob getBoxes fits its rectangle to."""
    import cv2
    contour = cv2.findContours(seg.astype(np.uint8), cv2.RETR_TREE, cv2.CHAIN_APPROX_SIMPLE)[-2][0]
    out = np.zeros(seg.shape, np.uint8)
    cv2.drawContours(out, [contour], -1, 1, thickness=-1)
    return out.astype(bool), contour


def box_of(contour):
    """getBoxes' box of a contour (detection.py:273-284) in score-map pixels."""
    import cv2
    quad = cv2.boxPoints(cv2.minAreaRect(contour))
    side_a, side_b = np.linalg.norm(quad[0] - quad[1]), np.linalg.norm(quad[1] - quad[2])
    if abs(1 - max(side_a, side_b) / (min(side_a, side_b) + 1e-5)) <= 0.1:
        xs, ys = contour[:, 0, 0], contour[:, 0, 1]
        return np.array([[xs.min(), ys.min()], [xs.max(), ys.min()], [xs.max(), ys.max()], [xs.min(), ys.max()]],
                        np.float32)
    return np.roll(quad, 4 - int(quad.sum(axis=1).argmin()), 0).astype(np.float32)


def component_blobs(scores, labels, comps, count, text_threshold=0.4, link_threshold=0.4):
    """The filled blob of every kept component of one image, as getBoxes builds it (detection.py:244-272):
    labels (H,W) int32 and comps (max_boxes,7) int32 as b2o_get_boxes_test writes them."""
    import cv2
    from oracle.imageops import component_niter
    H, W = labels.shape
    both = (scores[..., 0] > text_threshold) & (scores[..., 1] > link_threshold)
    blobs = []
    for root, x, y, w, h, area, _ in comps[:count]:
        seg = np.zeros((H, W), np.uint8)
        seg[labels == root] = 1
        seg[both] = 0
        niter = component_niter(area, w, h)
        x_lo, y_lo = max(x - niter, 0), max(y - niter, 0)
        x_hi, y_hi = min(x + w + niter + 1, W), min(y + h + niter + 1, H)
        kernel = cv2.getStructuringElement(cv2.MORPH_RECT, (1 + niter, 1 + niter))
        seg[y_lo:y_hi, x_lo:x_hi] = cv2.dilate(seg[y_lo:y_hi, x_lo:x_hi], kernel)
        blobs.append(filled_blob(seg)[0])
    return blobs


# ------------------------------------------------------------------------------------------------ piecewise warpBox
def _dist(a, b):
    dx, dy = float(a[0]) - float(b[0]), float(a[1]) - float(b[1])
    return math.sqrt(dx * dx + dy * dy)


def warp_layout(poly, points):
    """(s, dw, dh, X (s+1,) float32, sh float32) of a polygon of >= 6 points, or None where its w or h is 0."""
    p = np.asarray(poly, np.float32)[:points]
    s = points // 2 - 1
    top, bot = p[:s + 1], p[::-1][:s + 1]
    cum = [0.0]
    for i in range(s):
        cum.append(cum[-1] + (_dist(top[i], top[i + 1]) + _dist(bot[i], bot[i + 1])) / 2)
    hs = 0.0
    for j in range(s + 1):
        hs = hs + _dist(top[j], bot[j])
    w, h = int(cum[s]), int(hs / (s + 1))
    if w <= 0 or h <= 0:
        return None
    scale = min(CROP_W / w, CROP_H / h)
    sw, sh = scale * w, scale * h
    X = np.array([sw * (c / cum[s]) for c in cum], np.float32)
    return s, int(sw), int(sh), X, np.float32(sh)


def warp_poly(img, poly, points, model=False):
    """The crop (31,200[,C]) uint8 that b2o_warp_polys cuts along a polygon of >= 6 points, with cv2; ``model``: with
    the models of cv2.getPerspectiveTransform / warpPerspective that tests/test_image_refs.py pins against cv2
    (tests/cvmodels.py, image_refs.warp_sample), which the kernel restates operation for operation."""
    import cv2
    out = np.zeros((CROP_H, CROP_W) + img.shape[2:], np.uint8)
    lay = warp_layout(poly, points)
    if lay is None:
        return out
    s, dw, dh, X, sh = lay
    p = np.asarray(poly, np.float32)[:points]
    dwc, dhc = min(dw, CROP_W), min(dh, CROP_H)
    cols = np.arange(dwc, dtype=np.float32)
    seg = np.zeros(dwc, np.int64)
    for j in range(1, s):
        seg[X[j] <= cols] = j
    for i in range(s):
        src = np.array([p[i], p[i + 1], p[points - 2 - i], p[points - 1 - i]], np.float32)
        dst = np.array([[X[i], 0], [X[i + 1], 0], [X[i + 1], sh], [X[i], sh]], np.float32)
        if model:
            from tests import cvmodels, image_refs
            full = image_refs.warp_sample(img, cvmodels.inv3(cvmodels.get_persp(src, dst)).reshape(-1), dw, dh)
        else:
            full = cv2.warpPerspective(img, cv2.getPerspectiveTransform(src, dst), (dw, dh), flags=cv2.INTER_LINEAR,
                                       borderMode=cv2.BORDER_CONSTANT, borderValue=0)
        keep = seg == i
        out[:dhc, :dwc][:, keep] = full[:dhc, :dwc][:, keep]
    return out


# ------------------------------------------------------------------------------------------------ shapes
def straight_band(angle_deg, length=60, thickness=9, size=120):
    """A filled straight band through the centre of a size x size map at ``angle_deg``."""
    import cv2
    m = np.zeros((size, size), np.uint8)
    a = math.radians(angle_deg)
    c = size / 2
    d = np.array([math.cos(a), math.sin(a)]) * length / 2
    p0, p1 = np.round((c - d) * 16).astype(int), np.round((c + d) * 16).astype(int)
    cv2.line(m, tuple(p0), tuple(p1), 1, thickness, cv2.LINE_8, 4)
    return m


def arc_band(sweep_deg, radius=60, thickness=9, rotate_deg=0.0, size=None):
    """An annular arc of ``sweep_deg`` (centre of the sweep at the top), and its analytic centre line as a function
    that gives each point's distance to the circle of ``radius`` (restricted to the sweep)."""
    size = size or int(2 * radius + 4 * thickness)
    yy, xx = np.mgrid[0:size, 0:size].astype(np.float64)
    cx, cy = size / 2, size / 2 + radius / 2
    ang = np.degrees(np.arctan2(xx - cx, cy - yy)) - rotate_deg          # 0 at the top, clockwise positive
    ang = (ang + 180) % 360 - 180
    rr = np.hypot(xx - cx, yy - cy)
    m = (np.abs(rr - radius) <= thickness / 2) & (np.abs(ang) <= sweep_deg / 2)

    def dist(pts):
        pts = np.asarray(pts, np.float64)
        a = np.degrees(np.arctan2(pts[:, 0] - cx, cy - pts[:, 1])) - rotate_deg
        a = np.clip((a + 180) % 360 - 180, -sweep_deg / 2, sweep_deg / 2) + rotate_deg
        on = np.stack([cx + radius * np.sin(np.radians(a)), cy - radius * np.cos(np.radians(a))], -1)
        return np.hypot(*(pts - on).T)
    return m.astype(np.uint8), dist


def sine_band(amplitude, wavelength=80, length=140, thickness=9):
    """A band along y = A sin(2 pi x / wavelength) and the distance of points to that curve (dense sampling)."""
    h = int(2 * amplitude + 3 * thickness)
    w = int(length + 3 * thickness)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    x0, yc = 1.5 * thickness, h / 2
    xs = np.linspace(x0, x0 + length, 4000)
    curve = np.stack([xs, yc + amplitude * np.sin(2 * np.pi * (xs - x0) / wavelength)], -1)
    m = np.zeros((h, w), bool)
    for k in range(0, len(curve), 4):
        m |= np.hypot(xx - curve[k, 0], yy - curve[k, 1]) <= thickness / 2

    def dist(pts):
        pts = np.asarray(pts, np.float64)
        return np.sqrt(((pts[:, None, :] - curve[None]) ** 2).sum(-1)).min(1)
    return m.astype(np.uint8), dist


def covered(poly, points, blob):
    """Share of the blob's pixels (integer coordinates, score-map pixels) inside the polygon (x2 coordinates)."""
    import cv2
    p = (np.asarray(poly, np.float32)[:points] / 2).reshape(-1, 1, 2)
    ys, xs = np.nonzero(blob)
    inside = [cv2.pointPolygonTest(p, (float(x), float(y)), False) >= 0 for x, y in zip(xs, ys)]
    return float(np.mean(inside))
