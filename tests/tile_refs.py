"""NumPy statement of tiled detection (DESIGN.md section 1, "Tiles"): the grid of ``b2o_tile_plan``, the cut of
``b2o_cut_tiles`` and the stitch of ``b2o_stitch_tiles``."""
import numpy as np


def plan_axis(length, tile_size, margin):
    """(t, s, k) of one axis: tile extent, stride, the fewest tiles whose extents cover [0, length)."""
    t = min(tile_size, length)
    s = t - 2 * margin
    k = 1 if length <= tile_size else 1 + -(-(length - t) // s)
    return t, s, k


def plan(hp, wp, tile_size, margin):
    """The grid as a dict of b2o_tiles' fields, or None where b2o_tile_plan refuses the parameters."""
    if (hp < 32 or wp < 32 or margin < 0 or margin % 16 or tile_size % 32 or tile_size > 2048 or tile_size < 32
            or 4 * margin > tile_size):
        return None
    t_h, s_h, n_h = plan_axis(hp, tile_size, margin)
    t_w, s_w, n_w = plan_axis(wp, tile_size, margin)
    return {"hp": hp, "wp": wp, "tile_size": tile_size, "margin": margin, "t_h": t_h, "t_w": t_w, "s_h": s_h,
            "s_w": s_w, "n_h": n_h, "n_w": n_w}


def cores(length, t, s, k, margin):
    """[(lo, hi)] of every tile's core along an axis, in detector-input pixels."""
    return [(0 if i == 0 else i * s + margin, length if i == k - 1 else i * s + t - margin) for i in range(k)]


def score_cores(length, t, s, k, margin):
    """The same ranges in score-map pixels (halved, floor)."""
    return [(lo // 2, hi // 2) for lo, hi in cores(length, t, s, k, margin)]


def tile_index(p, g):
    """(image, tile row, tile column) of tile g: image-major, then tile row, then tile column."""
    per = p["n_h"] * p["n_w"]
    img, r = divmod(g, per)
    return img, r // p["n_w"], r % p["n_w"]


def cut(images, p, first=0, count=None):
    """Tiles [first, first + count) of images (n, hp, wp, 3) uint8 -> (count, t_h, t_w, 3) uint8, 255 past the page."""
    n = images.shape[0]
    total = n * p["n_h"] * p["n_w"]
    count = total - first if count is None else count
    out = np.full((count, p["t_h"], p["t_w"], 3), 255, np.uint8)
    for j in range(count):
        img, ty, tx = tile_index(p, first + j)
        oy, ox = ty * p["s_h"], tx * p["s_w"]
        part = images[img, oy:oy + p["t_h"], ox:ox + p["t_w"]]
        out[j, :part.shape[0], :part.shape[1]] = part
    return out


def stitch(tile_scores, p, n, first=0, out=None):
    """The cores of tiles [first, first + len(tile_scores)) into out (n, hp/2, wp/2, 2) float32 (a new NaN map when
    None); returns out."""
    if out is None:
        out = np.full((n, p["hp"] // 2, p["wp"] // 2, 2), np.nan, np.float32)
    ch = score_cores(p["hp"], p["t_h"], p["s_h"], p["n_h"], p["margin"])
    cw = score_cores(p["wp"], p["t_w"], p["s_w"], p["n_w"], p["margin"])
    for j in range(tile_scores.shape[0]):
        img, ty, tx = tile_index(p, first + j)
        (y0, y1), (x0, x1) = ch[ty], cw[tx]
        oy, ox = ty * p["s_h"] // 2, tx * p["s_w"] // 2
        out[img, y0:y1, x0:x1] = tile_scores[j, y0 - oy:y1 - oy, x0 - ox:x1 - ox]
    return out
