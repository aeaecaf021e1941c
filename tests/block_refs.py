"""fp64 NumPy restatement of the text-block grouping (DESIGN.md section 1, "Text blocks"; csrc/blocks.cu).

Recursive XY-cut over one image's text lines.  Every operation is an IEEE double operation in the order the kernel
performs it (NumPy and Python floats never fuse a multiply and an add), so ``group_blocks`` reproduces every output
bit of ``b2o_group_blocks``.
"""
import math
import sys

import numpy as np

DEFAULTS = {"row_gap": 1.5, "col_gap": 1.0}


def frame(boxes, sizes):
    """Page direction D and normal N: box[1] - box[0] of the line with the most words, ties to the smallest index."""
    q = np.asarray(boxes, np.float32).reshape(-1, 4, 2).astype(np.float64)
    dl = max(range(len(q)), key=lambda l: (int(sizes[l]), -l))
    ex, ey = float(q[dl, 1, 0] - q[dl, 0, 0]), float(q[dl, 1, 1] - q[dl, 0, 1])
    en = math.sqrt(ex * ex + ey * ey)
    dx, dy = (1.0, 0.0) if en == 0.0 else (ex / en, ey / en)
    return (dx, dy), (-dy, dx)


def extents(boxes, D, N):
    """Per line (a_lo, a_hi, b_lo, b_hi): its corners projected on D and N, as Python floats."""
    q = np.asarray(boxes, np.float32).reshape(-1, 4, 2).astype(np.float64)
    a = q[:, :, 0] * D[0] + q[:, :, 1] * D[1]
    b = q[:, :, 0] * N[0] + q[:, :, 1] * N[1]
    return [tuple(float(v) for v in t) for t in zip(a.min(1), a.max(1), b.min(1), b.max(1))]


def scale(boxes):
    """Lower median of the line heights |q3 - q0|."""
    q = np.asarray(boxes, np.float32).reshape(-1, 4, 2).astype(np.float64)
    fx, fy = q[:, 3, 0] - q[:, 0, 0], q[:, 3, 1] - q[:, 0, 1]
    g = sorted(float(v) for v in np.sqrt(fx * fx + fy * fy))
    return g[(len(g) - 1) // 2]


def cut(node, lo, hi, thr):
    """The node's lines sorted by (lo, l) and cut before every line whose lo is at least thr past the running max of
    hi of the lines before it: the pieces, in ascending lo."""
    order = sorted(node, key=lambda l: (lo[l], l))
    pieces, run = [[order[0]]], hi[order[0]]
    for l in order[1:]:
        if lo[l] - run >= thr:
            pieces.append([])
        pieces[-1].append(l)
        run = max(run, hi[l])
    return pieces


def group_blocks(boxes, sizes, **params):
    """One image's lines, (L,4,2) float32 boxes and (L,) word counts -> list of (block_box (4,2) float32, line
    indices int32) in depth-first order."""
    p = {**DEFAULTS, **params}
    q = np.asarray(boxes, np.float32).reshape(-1, 4, 2)
    if len(q) == 0:
        return []
    D, N = frame(q, sizes)
    ext = extents(q, D, N)
    alo, ahi, blo, bhi = ([e[k] for e in ext] for k in range(4))
    s = scale(q)
    row_thr, col_thr = p["row_gap"] * s, p["col_gap"] * s
    sys.setrecursionlimit(max(sys.getrecursionlimit(), 2 * len(q) + 100))

    def split(node):
        pieces = cut(node, blo, bhi, row_thr)
        if len(pieces) == 1:
            pieces = cut(node, alo, ahi, col_thr)
        if len(pieces) == 1:
            return [sorted(node)]
        return [leaf for piece in pieces for leaf in split(piece)]

    out = []
    for block in split(list(range(len(q)))):
        a0, a1 = min(alo[l] for l in block), max(ahi[l] for l in block)
        b0, b1 = min(blo[l] for l in block), max(bhi[l] for l in block)
        box = np.array([[ca * D[0] + cb * N[0], ca * D[1] + cb * N[1]]
                        for ca, cb in ((a0, b0), (a1, b0), (a1, b1), (a0, b1))]).astype(np.float32)
        out.append((box, np.array(block, np.int32)))
    return out


def csr(pages, max_boxes, **params):
    """The outputs of b2o_group_blocks for a batch of pages, each (line boxes (L,4,2), word counts (L,)):
    (block_counts (n,), line_order[i][:L], block_start[i][:B+1], block_boxes[i][:B]) as lists of arrays."""
    counts, order, start, bboxes = [], [], [], []
    for boxes, sizes in pages:
        blocks = group_blocks(np.asarray(boxes, np.float32).reshape(-1, 4, 2)[:max_boxes], sizes[:max_boxes], **params)
        counts.append(len(blocks))
        lines = [l for _, l in blocks]
        order.append(np.concatenate(lines).astype(np.int32) if lines else np.zeros(0, np.int32))
        start.append(np.concatenate([[0], np.cumsum([len(l) for l in lines])]).astype(np.int32))
        bboxes.append(np.stack([b for b, _ in blocks]) if blocks else np.zeros((0, 4, 2), np.float32))
    return np.array(counts, np.int32), order, start, bboxes


# ----------------------------------------------------------------------------------------------- layouts
def line_box(x, y, w, h):
    """An axis-aligned (4,2) float32 line box, top-left (x, y), corners tl, tr, br, bl."""
    return np.array([[x, y], [x + w, y], [x + w, y + h], [x, y + h]], np.float32)


def column(x, y, w, h, pitch, count):
    """``count`` lines of width w and height h, one every ``pitch`` down from (x, y)."""
    return [line_box(x, y + k * pitch, w, h) for k in range(count)]


def random_page(rng, count, tilt=None):
    """``count`` line boxes and word counts: a grid of 1 to 4 columns of paragraphs (line gaps of 0.2 to 0.6 line
    heights inside a paragraph, 1 to 3 between paragraphs), sometimes a full-width title, the whole page tilted by
    ``tilt`` degrees (random when None) with per-corner jitter; shuffled."""
    if tilt is None:
        tilt = float(rng.choice([0.0, 0.0, rng.uniform(-10, 10), 90.0, 180.0]))
    t = math.radians(tilt)
    cs, sn = math.cos(t), math.sin(t)
    boxes = []
    while len(boxes) < count:
        h = float(rng.uniform(10, 30))
        cols = int(rng.integers(1, 5))
        width = float(rng.uniform(8, 30)) * h
        gutter = float(rng.uniform(0.3, 3.0)) * h
        x0, y0 = float(rng.uniform(0, 3000)), float(rng.uniform(0, 3000))
        y = y0
        if rng.uniform() < 0.3:
            boxes.append(line_box(x0, y, cols * width + (cols - 1) * gutter, 2 * h))
            y += 2 * h + float(rng.uniform(1, 3)) * h
        for col in range(cols):
            yc = y
            for _ in range(int(rng.integers(1, 4))):
                for _ in range(int(rng.integers(1, 8))):
                    boxes.append(line_box(x0 + col * (width + gutter), yc, width * float(rng.uniform(0.5, 1)), h))
                    yc += h * (1 + float(rng.uniform(0.2, 0.6)))
                yc += h * float(rng.uniform(1, 3))
    q = np.stack(boxes[:count]).astype(np.float64) if count else np.zeros((0, 4, 2))
    q = np.stack([q[..., 0] * cs - q[..., 1] * sn, q[..., 0] * sn + q[..., 1] * cs], -1)
    q = (q + rng.normal(0, 0.2, q.shape)).astype(np.float32)
    sizes = rng.integers(1, 9, count).astype(np.int32)
    perm = rng.permutation(count)
    return q[perm], sizes[perm]


def spiral(count, h=20.0):
    """``count`` lines in a spiral that forces one cut per level of the tree: a line along the top edge of the
    remaining area, then one down its right edge, one along its bottom edge and one up its left edge, each cut off by
    a gap of 2 line heights, the area shrinking inwards.  The vertical lines are tall boxes in the page frame of the
    horizontal ones (box[0] -> box[1] along +x).  Returns (boxes, word counts); the first line has the most words."""
    g = 2 * h
    x0, y0, x1, y1 = 0.0, 0.0, count * 3 * (h + g), count * 3 * (h + g)
    boxes = []
    for k in range(count):
        side = k % 4
        if side == 0:
            boxes.append(line_box(x0, y0, x1 - x0, h))
            y0 += h + g
        elif side == 1:
            boxes.append(line_box(x1 - h, y0, h, y1 - y0))
            x1 -= h + g
        elif side == 2:
            boxes.append(line_box(x0, y1 - h, x1 - x0, h))
            y1 -= h + g
        else:
            boxes.append(line_box(x0, y0, h, y1 - y0))
            x0 += h + g
    sizes = np.ones(count, np.int32)
    sizes[0] = 2
    return np.stack(boxes), sizes
