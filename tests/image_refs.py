"""Plain NumPy references for the image stages of keras-ocr_b200/csrc/image.cu, and the seeded cases the GPU tests run.

warpBox is built from the pieces that are already pinned: ``oracle.imageops.order_corners`` /
``rotated_width_height`` for the plan, ``cvmodels.get_persp`` / ``inv3`` for the fp64 homography, and a vectorised
form of ``cvmodels.warp_model`` for the sampler (same operation order, separate fp64 roundings, ``np.rint`` half-even,
x re-based at multiples of bw0 like cv::WarpPerspectiveInvoker).  tests/test_image_refs.py pins all of it, and
``cvmodels.resize_model`` at every resize shape below, against cv2 on the CPU.

Importing this module needs neither a GPU nor cv2 (``warp_plan`` imports oracle.imageops, and with it cv2, when called).
"""
import numpy as np

from tests import cvmodels as M

CROP_H, CROP_W = 31, 200


# ----------------------------------------------------------------------------------------------------- warpBox
def warp_transform(quad, target_w=CROP_W, target_h=CROP_H):
    """(forward M (3,3), dw, dh) of tools.warpBox; raises ZeroDivisionError where warpBox does (w or h is 0)."""
    from oracle import imageops
    box = imageops.order_corners(quad)
    w, h = imageops.rotated_width_height(box)
    scale = min(target_w / w, target_h / h)
    dst = np.array([[0, 0], [scale * w, 0], [scale * w, scale * h], [0, scale * h]]).astype("float32")
    return M.get_persp(box, dst), int(scale * w), int(scale * h)


def warp_plan(quad):
    """(m (9,) float64 inverse homography, dw, dh), the WarpPlan the kernel derives; ZeroDivisionError as above."""
    fwd, dw, dh = warp_transform(quad)
    return M.inv3(fwd).reshape(-1), dw, dh


def warp_sample(img, m, dw, dh):
    """cv2.warpPerspective(INTER_LINEAR, BORDER_CONSTANT 0) of img (H,W) or (H,W,C) uint8 through the inverse map m,
    written into the top-left (dh, dw) of a zero (31, 200[, C]) crop.  Vectorised ``cvmodels.warp_model``."""
    H, W = img.shape[:2]
    out = np.zeros((CROP_H, CROP_W) + img.shape[2:], np.uint8)
    dw, dh = min(dw, CROP_W), min(dh, CROP_H)
    if dw <= 0 or dh <= 0:
        return out
    bh0 = min(16, dh)
    bw0 = min(1024 // bh0, dw)
    x = np.arange(dw)
    bx = ((x // bw0) * bw0).astype(np.float64)[None, :]
    x1 = (x % bw0).astype(np.float64)[None, :]
    y = np.arange(dh, dtype=np.float64)[:, None]
    X0 = m[0] * bx + m[1] * y + m[2]
    Y0 = m[3] * bx + m[4] * y + m[5]
    W0 = m[6] * bx + m[7] * y + m[8]
    Wv = W0 + m[6] * x1
    with np.errstate(divide="ignore"):
        Wv = np.where(Wv != 0, 32.0 / Wv, 0.0)
    fX = np.clip((X0 + m[0] * x1) * Wv, -2147483648.0, 2147483647.0)
    fY = np.clip((Y0 + m[3] * x1) * Wv, -2147483648.0, 2147483647.0)
    X, Y = np.rint(fX).astype(np.int64), np.rint(fY).astype(np.int64)
    sx, sy = np.clip(X >> 5, -32768, 32767), np.clip(Y >> 5, -32768, 32767)
    ax, ay = X & 31, Y & 31
    extra = (slice(None),) * 2 + (None,) * (img.ndim - 2)

    def px(yy, xx):
        ok = (yy >= 0) & (yy < H) & (xx >= 0) & (xx < W)
        v = img[np.clip(yy, 0, H - 1), np.clip(xx, 0, W - 1)].astype(np.int64)
        return np.where(ok[extra], v, 0)

    w00, w01 = ((32 - ax) * (32 - ay) * 32)[extra], (ax * (32 - ay) * 32)[extra]
    w10, w11 = ((32 - ax) * ay * 32)[extra], (ax * ay * 32)[extra]
    v = px(sy, sx) * w00 + px(sy, sx + 1) * w01 + px(sy + 1, sx) * w10 + px(sy + 1, sx + 1) * w11
    out[:dh, :dw] = (v + 16384) >> 15
    return out


def warp_box(img, quad):
    """tools.warpBox(margin=0, cval=0) -> (crop (31,200[,C]) uint8, plan (m, dw, dh) or None where warpBox raises
    ZeroDivisionError; the kernel writes an all-zero crop there)."""
    try:
        plan = warp_plan(quad)
    except ZeroDivisionError:
        return np.zeros((CROP_H, CROP_W) + img.shape[2:], np.uint8), None
    return warp_sample(img, *plan), plan


def crops_to_input(crops):
    """CRNN input (recognition.py:215-216): x[b, t, j(, c)] = crop[b, 30 - j, t(, c)] / 255 in fp16."""
    x = np.swapaxes(crops[:, ::-1], 1, 2)
    return (x.astype(np.float32) / np.float32(255)).astype(np.float16)


# ----------------------------------------------------------------------------------------------------- cases
def _rect(cx, cy, w, h, deg, start=0, reverse=False):
    a = np.deg2rad(deg)
    u = np.array([np.cos(a), np.sin(a)]) * w / 2
    v = np.array([-np.sin(a), np.cos(a)]) * h / 2
    c = np.array([cx, cy], np.float64)
    q = np.array([c - u - v, c + u - v, c + u + v, c - u + v])
    q = np.roll(q, -start, 0)
    return (q[::-1] if reverse else q).astype(np.float32)


def _axis(x0, y0, x1, y1, start=0):
    """Axis-parallel box with exact float32 corners (0 and 90 degrees: the x-sort ties in pairs)."""
    return np.roll(np.array([[x0, y0], [x1, y0], [x1, y1], [x0, y1]], np.float32), -start, 0)


def _diamond(cx, cy, rx, ry, start=0):
    """Rhombus with exact corners; rx == ry is a square at 45 degrees, where the top and bottom corners tie in x."""
    return np.roll(np.array([[cx, cy - ry], [cx + rx, cy], [cx, cy + ry], [cx - rx, cy]], np.float32), -start, 0)


def _pythagorean(x0, y0, a, start=0):
    """Rotated rectangle with integer corners (sides (3a, 4a) and (-4, 3)), exact in float32 far from the origin,
    where a rotated float corner would round off the rectangle and get_rotated_box would rectify it."""
    q = np.array([[0, 0], [3 * a, 4 * a], [3 * a - 4, 4 * a + 3], [-4, 3]], np.float64) + (x0, y0)
    return np.roll(q, -start, 0).astype(np.float32)


def _below_integer(target, limit=4000):
    """Integer sides s for which (target / s) * s rounds below ``target`` in fp64, so int() drops a pixel."""
    return [s for s in range(1, limit) if (target / s) * s < target]


def _page_quads(rng, H, W):
    q = []
    for _ in range(40):                                     # rotated rectangles, corners in any cyclic order
        q.append(_rect(rng.uniform(-20, W + 20), rng.uniform(-20, H + 20), rng.uniform(4, 180), rng.uniform(3, 60),
                       rng.uniform(-90, 90), int(rng.integers(4)), bool(rng.integers(2))))
    for s in range(4):                                      # exactly 0 / 90 degrees, every start corner
        q.append(_axis(10.5, 20, 150.5, 48, s))
        q.append(_axis(30, 5, 52, 140.25, s))
    for s in range(4):                                      # exactly +-45 degrees: squares (x ties) and rectangles
        q.append(_diamond(W / 2, H / 2, 30, 30, s))
        q.append(_diamond(40, 60, 12.5, 12.5, s))
        q.append(_rect(W / 2, H / 2, 120, 24, 45, s))
        q.append(_rect(W / 2, H / 2, 120, 24, -45, s))
    for deg in (0.0, 17.0, -33.0):                          # partly off each edge and each corner
        q += [_rect(-10, H / 2, 60, 30, deg), _rect(W + 8, H / 2, 50, 26, deg), _rect(W / 2, -6, 90, 24, deg),
              _rect(W / 2, H + 5, 90, 24, deg), _rect(0, 0, 40, 20, deg), _rect(W, H, 40, 20, deg)]
    q += [_axis(-0.5, -0.5, W - 0.5, H - 0.5), _axis(0, 0, W, H)]                   # the whole image
    q += [_axis(-80, 10, -20, 40), _axis(W + 3, 10, W + 90, 30), _rect(W / 2, -100, 80, 20, 30),
          _rect(W / 2, H + 300, 80, 20, -60)]                                         # wholly off the image
    q += [_pythagorean(60000, 50000, 12), _pythagorean(-70000, -40000, 7, 2),         # source beyond +-32768 px
          _axis(1e8, 1e8, 1e8 + 64, 1e8 + 16), _axis(-1e8, 0, -1e8 + 48, 24)]         # and beyond the int clamp
    q += [_axis(5, 30, 305, 32), _axis(0, 50, 1000, 53),                              # dh = 1
          _axis(100, 10, 101, 30), _axis(60, 10, 62, 35), _axis(70, 20, 73, 51)]      # dw = 1, 2, 3
    q += [_rect(W / 2, H / 2, 4000, 600, 10), _rect(W / 2, H / 2, 3000, 2500, -70)]   # scale << 1
    q += [_axis(3, 3, 203, 20), _axis(3, 3, 40, 34), _axis(3, 3, 203, 10), _axis(3, 3, 203, 7)]  # dw = 200, dh = 31,
    # dh = 10 / 7 (x re-based at 102 / 146), and sides where scale * side lands just below the integer
    for s in _below_integer(200.0)[:4]:
        q.append(_axis(2, 3, 2 + s, 3 + max(1, s // 10)))
    for s in _below_integer(31.0, 600)[:3]:
        q.append(_axis(4, 1, 4 + 10 * s, 1 + s))
    q += [_axis(50, 50, 50.6, 80), _axis(20, 20, 90, 20.4), np.full((4, 2), 33.0, np.float32)]  # degenerate: w or h 0
    return q


def warp_cases(seed=0):
    """Groups of (name, gray (n,H,W), rgb (n,H,W,3), quads (B,4,2) float32, image_index (B,) int32); every group's box
    count B is not a multiple of 32, so B * 6200 crop pixels do not fill whole 256-thread blocks."""
    rng = np.random.default_rng(seed)
    groups = []

    def add(name, n, H, W, quads):
        quads = np.stack(quads).astype(np.float32)
        assert len(quads) % 32 != 0
        groups.append(dict(name=name, gray=rng.integers(0, 256, (n, H, W), dtype=np.uint8),
                           rgb=rng.integers(0, 256, (n, H, W, 3), dtype=np.uint8), quads=quads,
                           image_index=rng.integers(0, n, len(quads)).astype(np.int32)))

    add("page", 3, 157, 211, _page_quads(rng, 157, 211))
    row = [_rect(rng.uniform(-10, 110), rng.uniform(-3, 4), rng.uniform(5, 90), rng.uniform(2, 12), rng.uniform(-30, 30))
           for _ in range(14)] + [_axis(0, 0, 97, 1), _axis(-0.5, -0.5, 96.5, 0.5), _axis(10, -2, 60, 3)]
    add("one_row", 2, 1, 97, row)
    col = [_rect(rng.uniform(-3, 4), rng.uniform(-10, 90), rng.uniform(2, 12), rng.uniform(5, 90), rng.uniform(-30, 30))
           for _ in range(14)] + [_axis(0, 0, 1, 83), _axis(-0.5, -0.5, 0.5, 82.5), _axis(-2, 10, 3, 70)]
    add("one_column", 2, 83, 1, col)
    small = [_rect(rng.uniform(-2, 7), rng.uniform(-2, 5), rng.uniform(1, 9), rng.uniform(1, 7), rng.uniform(-90, 90))
             for _ in range(11)]
    add("tiny_image", 1, 3, 5, small)
    return groups


# ----------------------------------------------------------------------------------------------------- resize
def resize_cases():
    """(id, hs, ws, hr, wr): the tools.resize_plan targets of the pipeline's defaults (max_scale 2, max_size 2048) for
    1-pixel-tall and -wide pages, a downscale, the identity, exactly 0.5 and an upright downscale; non-integer upscales
    at other settings; and two free targets."""
    from keras_ocr_b200 import tools
    cases = []
    for hs, ws, ms, mx in [(1, 700, 2, 2048), (1, 1500, 2, 2048), (700, 1, 2, 2048), (1500, 1, 2, 2048),
                           (1000, 3000, 2, 2048), (2048, 2048, 2, 2048), (4096, 4096, 2, 2048), (2500, 900, 2, 2048),
                           (300, 500, 2, 800), (131, 197, 2, 350), (77, 93, 3, 250)]:
        _, hr, wr = tools.resize_plan((hs, ws, 3), ms, mx)
        cases.append((f"{hs}x{ws}_to_{hr}x{wr}", hs, ws, hr, wr))
    cases += [("45x67_to_100x150", 45, 67, 100, 150), ("64x48_to_37x29", 64, 48, 37, 29)]
    return cases


def padded(hr, wr):
    """A padded size larger than (hr, wr) whose width is not a multiple of the kernel's 128-thread blocks."""
    wp = wr + 7 if (wr + 7) % 128 else wr + 8
    return hr + 3, wp


def resize_pad(src, hr, wr, hp, wp):
    """tools.resize_image's cv2.resize (cvmodels.resize_model) then tools.pad with 255."""
    out = np.full((hp, wp, 3), 255, np.uint8)
    out[:hr, :wr] = M.resize_model(src, wr, hr)
    return out


def gray_of(rgb):
    """cv2.cvtColor(RGB2GRAY) on uint8: 15-bit fixed point, round half up."""
    r, g, b = (rgb[..., c].astype(np.int64) for c in range(3))
    return ((9798 * r + 19235 * g + 3735 * b + 16384) >> 15).astype(np.uint8)


def all_rgb_triplets():
    """Every RGB triplet once, as one (4096, 4096, 3) uint8 image."""
    i = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([(i >> 16) & 255, (i >> 8) & 255, i & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
