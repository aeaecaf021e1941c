"""Oracle: the OpenCV/NumPy image stages around the two networks.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Each function restates one reference
function and, like the reference, leans on OpenCV for the third-party arithmetic
(resize, threshold, connectedComponentsWithStats, dilate, findContours, minAreaRect,
getPerspectiveTransform, warpPerspective).  OpenCV here is 4.13 (unpinned upstream).
"""
import cv2
import numpy as np

IMAGENET_MEAN = np.array([0.485, 0.456, 0.406])
IMAGENET_STD = np.array([0.229, 0.224, 0.225])


# ----------------------------------------------------------------------------- inputs
def resize_image(image, max_scale, max_size):
    """tools.resize_image, reference tools.py:378-398.  Returns (image, scale)."""
    longest = max(image.shape)          # includes the channel axis, as upstream does
    scale = max_size / longest if longest * max_scale > max_size else max_scale
    out_w, out_h = int(image.shape[1] * scale), int(image.shape[0] * scale)
    return cv2.resize(image, dsize=(out_w, out_h)), scale


def pad(image, width, height, cval=255):
    """tools.pad, reference tools.py:356-375: bottom/right pad with ``cval``."""
    assert height >= image.shape[0] and width >= image.shape[1]
    shape = (height, width) + tuple(image.shape[2:])
    canvas = np.full(shape, cval, dtype=image.dtype)
    canvas[: image.shape[0], : image.shape[1]] = image
    return canvas


def compute_input(image):
    """detection.compute_input, reference detection.py:34-42 (RGB order)."""
    x = image.astype("float32")
    x -= IMAGENET_MEAN * 255
    x /= IMAGENET_STD * 255
    return x


def rgb_to_gray(image):
    """cv2.cvtColor(RGB2GRAY) at recognition.py:510."""
    return cv2.cvtColor(image, code=cv2.COLOR_RGB2GRAY)


# ----------------------------------------------------------------------------- getBoxes
def component_niter(area, w, h):
    """Dilation size, reference detection.py:258."""
    return int(np.sqrt(area * min(w, h) / (w * h)) * 2)


def get_boxes_single(scores, detection_threshold=0.7, text_threshold=0.4,
                     link_threshold=0.4, size_threshold=10, debug=None):
    """One image of ``getBoxes`` (reference detection.py:207-287).

    scores: (h, w, 2) float32.  Returns an array (n,4,2) float32 in detector-input pixels
    (score-map coordinates x2), or an empty (0,) array like ``np.array([])``.
    """
    text = np.ascontiguousarray(scores[..., 0])
    link = np.ascontiguousarray(scores[..., 1])
    H, W = text.shape
    text_bin = cv2.threshold(text, text_threshold, 1, cv2.THRESH_BINARY)[1]
    link_bin = cv2.threshold(link, link_threshold, 1, cv2.THRESH_BINARY)[1]
    union = np.clip(text_bin + link_bin, 0, 1).astype("uint8")
    count, labels, stats, _ = cv2.connectedComponentsWithStats(union, connectivity=4)
    both = np.logical_and(link_bin, text_bin)
    quads = []
    kept = []
    for cid in range(1, count):
        area = stats[cid, cv2.CC_STAT_AREA]
        if area < size_threshold:
            continue
        member = labels == cid
        if text[member].max() < detection_threshold:
            continue
        seg = np.zeros((H, W), dtype=text.dtype)
        seg[member] = 255
        seg[both] = 0
        x, y = stats[cid, cv2.CC_STAT_LEFT], stats[cid, cv2.CC_STAT_TOP]
        w, h = stats[cid, cv2.CC_STAT_WIDTH], stats[cid, cv2.CC_STAT_HEIGHT]
        niter = component_niter(area, w, h)
        x_lo, y_lo = max(x - niter, 0), max(y - niter, 0)
        x_hi, y_hi = min(x + w + niter + 1, W), min(y + h + niter + 1, H)
        kernel = cv2.getStructuringElement(cv2.MORPH_RECT, (1 + niter, 1 + niter))
        seg[y_lo:y_hi, x_lo:x_hi] = cv2.dilate(seg[y_lo:y_hi, x_lo:x_hi], kernel)
        outline = cv2.findContours(seg.astype("uint8"), mode=cv2.RETR_TREE,
                                   method=cv2.CHAIN_APPROX_SIMPLE)[-2][0]
        quad = cv2.boxPoints(cv2.minAreaRect(outline))
        side_a = np.linalg.norm(quad[0] - quad[1])
        side_b = np.linalg.norm(quad[1] - quad[2])
        ratio = max(side_a, side_b) / (min(side_a, side_b) + 1e-5)
        if abs(1 - ratio) <= 0.1:
            xs, ys = outline[:, 0, 0], outline[:, 0, 1]
            quad = np.array([[xs.min(), ys.min()], [xs.max(), ys.min()],
                             [xs.max(), ys.max()], [xs.min(), ys.max()]], dtype=np.float32)
        else:
            first = quad.sum(axis=1).argmin()
            quad = np.array(np.roll(quad, 4 - first, 0))
        quads.append(2 * quad)
        kept.append(cid)
    if debug is not None:
        debug.update(labels=labels, stats=stats, count=count, kept=kept)
    return np.array(quads)


def get_boxes(y_pred, **thresholds):
    """``getBoxes`` over a batch (reference detection.py:214-215, 286-287)."""
    return [get_boxes_single(scores, **thresholds) for scores in y_pred]


# ----------------------------------------------------------------------------- warpBox
def min_rotated_rectangle(points):
    """shapely's ``MultiPoint(points).minimum_rotated_rectangle.exterior`` minus its closing point (reference
    tools.py:544-547), restated from shapely's published algorithm (shapely/geometry/base.py, the pure-Python
    ``oriented_envelope``): convex hull; for every hull edge rotate the hull into the edge's frame and take the
    axis-parallel envelope; keep the envelope of least area and rotate it back.  Returns None when the hull is a point
    or a segment (shapely returns a geometry without ``.exterior`` -> the reference's AttributeError branch).
    shapely is absent offline: PARITY UNPINNED for this function (getBoxes only emits rectangles, on which it is the
    identity up to fp64 rounding -- ``order_corners`` keeps those bit for bit)."""
    import math
    pts = sorted({(float(x), float(y)) for x, y in np.asarray(points, dtype=np.float64)})
    if len(pts) < 3:
        return None
    cross = lambda o, a, b: (a[0] - o[0]) * (b[1] - o[1]) - (a[1] - o[1]) * (b[0] - o[0])
    lower, upper = [], []
    for q in pts:
        while len(lower) >= 2 and cross(lower[-2], lower[-1], q) <= 0:
            lower.pop()
        lower.append(q)
    for q in reversed(pts):
        while len(upper) >= 2 and cross(upper[-2], upper[-1], q) <= 0:
            upper.pop()
        upper.append(q)
    hull = lower[:-1] + upper[:-1]
    if len(hull) < 3:
        return None
    best = None
    for (x1, y1), (x2, y2) in zip(hull, hull[1:] + hull[:1]):
        length = math.sqrt((x2 - x1) ** 2 + (y2 - y1) ** 2)
        ux, uy = (x2 - x1) / length, (y2 - y1) / length
        vx, vy = -uy, ux
        xs = [ux * x + uy * y for x, y in hull]
        ys = [vx * x + vy * y for x, y in hull]
        area = (max(xs) - min(xs)) * (max(ys) - min(ys))
        if best is None or area < best[0] * (1.0 - 1e-9):      # exact ties are common for quads: the first edge in hull order wins
            env = [(min(xs), min(ys)), (max(xs), min(ys)), (max(xs), max(ys)), (min(xs), max(ys))]
            best = (area, [(ux * a + vx * b, uy * a + vy * b) for a, b in env])
    return np.array(best[1], dtype=np.float64)


def order_corners(points):
    """get_rotated_box, reference tools.py:533-581: minimum rotated rectangle (``min_rotated_rectangle``; the raw
    points on the reference's AttributeError branch, 548-550), then the imutils ordering tl, tr, br, bl.

    A 4-corner rectangle -- all that getBoxes emits -- is its own minimum rotated rectangle; it is kept bit for bit
    (corners within 1e-3 px) so that the fp64 round trip cannot move a float32 coordinate by an ulp.
    """
    pts = np.asarray(points)
    rect = min_rotated_rectangle(pts)
    if rect is not None:
        near = np.abs(rect[:, None, :] - pts[None, :, :].astype(np.float64)).max(-1).min(-1)
        if near.max() > 1e-3:
            pts = rect
    # kind="stable": upstream's default argsort breaks ties (a square at 45 degrees ties in x) by whatever the host's
    # NumPy sort does -- with AVX-512 it is not stable on 4 elements.  The stable order is the one the kernel follows.
    by_x = pts[np.argsort(pts[:, 0], kind="stable"), :]
    left, right = by_x[:2], by_x[2:]
    left = left[np.argsort(left[:, 1], kind="stable"), :]
    tl, bl = left
    delta = right.astype(np.float64) - tl.astype(np.float64)[np.newaxis]   # cdist works in float64
    dist = np.sqrt((delta ** 2).sum(axis=1))
    br, tr = right[np.argsort(dist, kind="stable")[::-1], :]
    return np.array([tl, tr, br, bl], dtype="float32")


def rotated_width_height(box):
    """get_rotated_width_height, reference tools.py:41-57 (cdist is float64 Euclidean)."""
    b = np.asarray(box, dtype=np.float64)
    d = lambda i, j: np.sqrt(((b[i] - b[j]) ** 2).sum())
    return int((d(0, 1) + d(2, 3)) / 2), int((d(0, 3) + d(1, 2)) / 2)


def warp_box(gray, box, target_height=31, target_width=200, return_transform=False):
    """tools.warpBox with margin=0, cval=0 on a gray image (reference tools.py:61-117)."""
    box = order_corners(box)
    w, h = rotated_width_height(box)
    scale = min(target_width / w, target_height / h)      # ZeroDivisionError if w or h is 0
    dst = np.array([[0, 0], [scale * w, 0], [scale * w, scale * h], [0, scale * h]]).astype("float32")
    M = cv2.getPerspectiveTransform(src=box, dst=dst)
    crop = cv2.warpPerspective(gray, M, dsize=(int(scale * w), int(scale * h)))
    # tools.py:108-113: a 3-channel image keeps its channels (color recognizer), a gray one stays 2-D
    full = np.zeros((target_height, target_width) + gray.shape[2:], dtype="uint8")
    full[: crop.shape[0], : crop.shape[1]] = crop
    if return_transform:
        return full, M
    return full
