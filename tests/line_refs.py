"""fp64 NumPy restatement of the text-line grouping (DESIGN.md section 1, "Text lines"; csrc/lines.cu).

Every operation is an IEEE double operation in the order the kernel performs it (NumPy and Python floats never fuse a
multiply and an add), so ``group_lines`` reproduces every output bit of ``b2o_group_lines``.
"""
import math

import numpy as np

DEFAULTS = {"angle_tolerance": 15.0, "height_ratio": 0.5, "offset_ratio": 0.5, "gap_ratio": 1.5}


def cos_tol(angle_tolerance):
    """The value the host passes to the kernel."""
    return math.cos(math.radians(angle_tolerance))


def features(boxes):
    """(c,4,2) float32 boxes -> dict of (c,) float64 arrays u (ux, uy), w, h, centre (cx, cy)."""
    q = np.asarray(boxes, np.float32).reshape(-1, 4, 2).astype(np.float64)
    ex, ey = q[:, 1, 0] - q[:, 0, 0], q[:, 1, 1] - q[:, 0, 1]
    w = np.sqrt(ex * ex + ey * ey)
    fx, fy = q[:, 3, 0] - q[:, 0, 0], q[:, 3, 1] - q[:, 0, 1]
    h = np.sqrt(fx * fx + fy * fy)
    with np.errstate(invalid="ignore", divide="ignore"):
        ux = np.where(w == 0, 1.0, ex / w)
        uy = np.where(w == 0, 0.0, ey / w)
    cx = ((q[:, 0, 0] + q[:, 1, 0]) + (q[:, 2, 0] + q[:, 3, 0])) * 0.25
    cy = ((q[:, 0, 1] + q[:, 1, 1]) + (q[:, 2, 1] + q[:, 3, 1])) * 0.25
    return {"ux": ux, "uy": uy, "w": w, "h": h, "cx": cx, "cy": cy}


def link_rows(f, rows, params):
    """Boolean (len(rows), c): the link relation of the words ``rows`` (as word i) with every word j, conditions
    evaluated with i first.  The diagonal is False.  ``params`` may give ``cos_tol`` itself instead of the angle."""
    p = {**DEFAULTS, **params}
    ct = p["cos_tol"] if "cos_tol" in p else cos_tol(p["angle_tolerance"])
    rows = np.asarray(rows)
    a = {k: v[rows][:, None] for k, v in f.items()}
    b = {k: v[None, :] for k, v in f.items()}
    ok = (a["w"] > 0) & (a["h"] > 0) & (b["w"] > 0) & (b["h"] > 0)
    ok &= (a["ux"] * b["ux"] + a["uy"] * b["uy"]) >= ct
    hmin, hmax = np.minimum(a["h"], b["h"]), np.maximum(a["h"], b["h"])
    ok &= hmin >= p["height_ratio"] * hmax
    dx, dy = b["cx"] - a["cx"], b["cy"] - a["cy"]
    off = p["offset_ratio"] * hmin
    ok &= np.abs(dx * -a["uy"] + dy * a["ux"]) <= off
    ok &= np.abs(dx * -b["uy"] + dy * b["ux"]) <= off
    half = (a["w"] + b["w"]) * 0.5
    gap = p["gap_ratio"] * hmax
    ok &= (np.abs(dx * a["ux"] + dy * a["uy"]) - half) <= gap
    ok &= (np.abs(dx * b["ux"] + dy * b["uy"]) - half) <= gap
    ok[np.arange(len(rows)), rows] = False
    return ok


def link_matrix(boxes, **params):
    f = features(boxes)
    c = len(f["w"])
    return link_rows(f, np.arange(c), params) if c else np.zeros((0, 0), bool)


def components(f, params, block=256):
    """Root (lowest word index) of every word's connected component of the link graph."""
    c = len(f["w"])
    parent = np.arange(c)

    def find(a):
        while parent[a] != a:
            parent[a] = parent[parent[a]]
            a = parent[a]
        return a

    for r0 in range(0, c, block):
        rows = np.arange(r0, min(c, r0 + block))
        ii, jj = np.nonzero(link_rows(f, rows, params))
        for i, j in zip(rows[ii], jj):
            if j > i:
                a, b = find(i), find(j)
                if a != b:
                    parent[max(a, b)] = min(a, b)
    return np.array([find(i) for i in range(c)], np.int64)


def group_lines(boxes, **params):
    """One image's boxes (c,4,2) float32 -> list of (line_box (4,2) float32, word indices int32) in page order."""
    q = np.asarray(boxes, np.float32).reshape(-1, 4, 2)
    c = len(q)
    if c == 0:
        return []
    f = features(q)
    roots = components(f, params)
    by_root = np.argsort(roots, kind="stable")         # ascending root, then ascending word index
    ids, first = np.unique(roots[by_root], return_index=True)   # line id = rank of its root
    members = {r: by_root[s:e].tolist() for r, s, e in zip(ids.tolist(), first, list(first[1:]) + [c])}
    lines = []
    for r in ids:
        mem = members[r]
        sx = sy = 0.0
        for i in mem:                                  # sequential, ascending word index
            sx += float(f["ux"][i])
            sy += float(f["uy"][i])
        nrm = math.sqrt(sx * sx + sy * sy)
        ux, uy = (1.0, 0.0) if nrm == 0.0 else (sx / nrm, sy / nrm)
        nx, ny = -uy, ux
        pts = q[mem].reshape(-1, 2).astype(np.float64)
        a = pts[:, 0] * ux + pts[:, 1] * uy
        b = pts[:, 0] * nx + pts[:, 1] * ny
        amin, amax, bmin, bmax = float(a.min()), float(a.max()), float(b.min()), float(b.max())
        am, bm = (amin + amax) * 0.5, (bmin + bmax) * 0.5
        m = (am * ux + bm * nx, am * uy + bm * ny)
        box = np.array([[ca * ux + cb * nx, ca * uy + cb * ny]
                        for ca, cb in ((amin, bmin), (amax, bmin), (amax, bmax), (amin, bmax))]).astype(np.float32)
        order = sorted(mem, key=lambda i: (float(f["cx"][i]) * ux + float(f["cy"][i]) * uy, i))
        lines.append({"U": (ux, uy), "m": m, "low": mem[0], "box": box, "words": np.array(order, np.int32)})
    # page direction: the line with the most words, ties to the lowest word index (line ids ascend with it)
    dline = max(range(len(lines)), key=lambda k: (len(lines[k]["words"]), -k))
    dx, dy = lines[dline]["U"]
    lines.sort(key=lambda L: (L["m"][0] * -dy + L["m"][1] * dx, L["m"][0] * dx + L["m"][1] * dy, L["low"]))
    return [(L["box"], L["words"]) for L in lines]


def csr(groups, max_boxes, **params):
    """The outputs of b2o_group_lines for a batch of box groups: (line_counts (n,), word_order[i][:c],
    line_start[i][:L+1], line_boxes[i][:L]) as lists of arrays."""
    counts, order, start, lboxes = [], [], [], []
    for g in groups:
        lines = group_lines(np.asarray(g, np.float32).reshape(-1, 4, 2)[:max_boxes], **params)
        counts.append(len(lines))
        words = [w for _, w in lines]
        order.append(np.concatenate(words).astype(np.int32) if words else np.zeros(0, np.int32))
        start.append(np.concatenate([[0], np.cumsum([len(w) for w in words])]).astype(np.int32))
        lboxes.append(np.stack([b for b, _ in lines]) if lines else np.zeros((0, 4, 2), np.float32))
    return np.array(counts, np.int32), order, start, lboxes


# ----------------------------------------------------------------------------------------------- layouts
def word_box(x, y, w, h, angle_deg=0.0, turn=0, origin=(0.0, 0.0)):
    """A (4,2) float32 box of a w x h word whose top-left corner is (x, y) in a frame rotated by ``angle_deg`` about
    ``origin``; corners tl, tr, br, bl of the text, rolled by ``turn`` quarter turns (box[0] = corner ``turn``)."""
    t = math.radians(angle_deg)
    c, s = math.cos(t), math.sin(t)
    pts = np.array([[x, y], [x + w, y], [x + w, y + h], [x, y + h]], np.float64) - origin
    rot = np.stack([pts[:, 0] * c - pts[:, 1] * s, pts[:, 0] * s + pts[:, 1] * c], 1) + origin
    return np.roll(rot, -turn, axis=0).astype(np.float32)


def row(x0, y, widths, h, space, **kw):
    """Boxes of words laid out left to right from (x0, y) with ``space`` between them."""
    out, x = [], x0
    for w in widths:
        out.append(word_box(x, y, w, h, **kw))
        x += w + space
    return out
