"""Plain NumPy restatement of wide-word windows (DESIGN.md section 1, "Wide words"; keras-ocr_b200/csrc/windows.cu):
the window count and plans of a box, the window crops, and the stitch of the windows' CTC steps.  fp64 throughout, in
the kernels' operation order and without contraction, so plans, crops, step positions, cuts and labels match bit for
bit; S sums float32 terms whose exp / log are not correctly rounded on either side, so it matches to a few ulps.

Importing this module needs neither a GPU nor cv2 (``extent`` imports oracle.imageops, and with it cv2, when called).
"""
import numpy as np

from tests import cvmodels as M
from tests import image_refs as I

CROP_W, CROP_H, STEPS, DISCARD = 200, 31, 48, 2
STRIDE, SHRINK, MAX_WINDOWS = 136, 8, 16          # B2O_WINDOW_STRIDE, B2O_WINDOW_SHRINK, B2O_MAX_WINDOWS


def extent(quad, max_windows):
    """(box (4,2) float32 in turn-0 order, wc, sh, K, ok): scale = min(T / w, 31 / h), T = 200 + (M - 1) S.  K = 1 for a
    word that fits (wc <= 200) or a box warpBox refuses (ok False); else 1 + ceil((wc - 200) / S), at most M."""
    from oracle import imageops
    box = imageops.order_corners(np.asarray(quad, np.float32)).astype(np.float32)
    w, h = imageops.rotated_width_height(box)
    if w <= 0 or h <= 0:
        return box, 0.0, 0.0, 1, False
    t = CROP_W + (max_windows - 1) * STRIDE
    scale = min(t / w, CROP_H / h)
    wc, sh = scale * w, scale * h
    if wc <= CROP_W:
        return box, wc, sh, 1, True
    return box, wc, sh, min(max_windows, 1 + int(np.ceil((wc - CROP_W) / STRIDE))), True


def starts(k, wc):
    """Window starts a_0 .. a_{K-1}: k S, the last flush with the word's end; (0,) for a word that fits."""
    if k == 1:
        return np.zeros(1)
    return np.array([float(i * STRIDE) for i in range(k - 1)] + [wc - CROP_W])


def plan(quad, max_windows, k):
    """dict of b2o_window_plan's fields for window slot k: m (9,) the inverse homography, a, wc, sh, k (= K), dw, dh,
    valid."""
    box, wc, sh, K, ok = extent(quad, max_windows)
    out = {"m": np.zeros(9), "a": 0.0, "wc": wc, "sh": sh, "k": K, "dw": 0, "dh": 0, "valid": 0}
    if not ok or k >= K:
        return out
    a = starts(K, wc)[k]
    x0, x1, y1 = np.float32(0.0 - a), np.float32(wc - a), np.float32(sh)
    dst = np.array([[x0, 0], [x1, 0], [x1, y1], [x0, y1]], np.float32)
    out.update(a=a, dw=int(wc) if K == 1 else CROP_W, dh=int(sh))
    try:
        out["m"] = M.inv3(M.get_persp(box, dst)).reshape(-1)
        out["valid"] = 1
    except (ZeroDivisionError, FloatingPointError):      # a singular system: an all-zero crop
        pass
    return out


def crop(img, quad, max_windows, k):
    """Window k's (31, 200[, C]) uint8 crop: warpPerspective through the plan into a zero crop."""
    p = plan(quad, max_windows, k)
    if not p["valid"]:
        return np.zeros((CROP_H, CROP_W) + img.shape[2:], np.uint8)
    return I.warp_sample(img, p["m"], p["dw"], p["dh"])


def positions(a, theta=None):
    """P (48,) float64: step t at crop column x = 4u + 1.5 of grid row r = t + 2 (u = r without an STN), clamped to
    [0, 200], made non-decreasing by a running max, plus a."""
    r = np.arange(STEPS, dtype=np.float64) + DISCARD
    if theta is None:
        u = r
    else:
        th4, th5 = np.float64(np.float32(theta[4])), np.float64(np.float32(theta[5]))
        gy = -1.0 + (2.0 * r) / 49.0
        u = (0.5 * ((th4 * gy + th5) + 1.0)) * 50.0
    x = np.fmin(np.fmax(4.0 * u + 1.5, 0.0), float(CROP_W))
    return a + np.maximum.accumulate(np.fmax(x, 0.0))


def steps(logits):
    """Per-step first argmax (all-NaN row: 0) and log(max p + 1e-7) in float32, max p = 1 / sum_c exp(l_c - l_max)
    summed in ascending c."""
    lg = np.asarray(logits, np.float32)
    best = np.zeros(lg.shape[0], np.int64)
    term = np.zeros(lg.shape[0], np.float32)
    for t, row in enumerate(lg):
        m, arg = np.float32(-np.inf), -1
        for c, v in enumerate(row):
            if v > m:
                m, arg = v, c
        s = np.float32(0)
        for v in row:
            s = np.float32(s + np.exp(np.float32(v - m)))
        best[t] = max(arg, 0)
        term[t] = np.log(np.float32(np.float32(1) / s) + np.float32(1e-7))
    return best, term


def cut(pk, bk, pn, bn, a0, a1, blank):
    """The cut between window k (positions pk, argmax bk) and k + 1 (pn, bn) starting at a0 and a1."""
    end = a0 + CROP_W
    mid = 0.5 * (a1 + end)
    lo, hi = a1 + SHRINK, end - SHRINK
    cands = [t for t in range(STEPS) if lo <= pn[t] <= hi]
    for t in sorted(cands, key=lambda t: (abs(pn[t] - mid), t)):
        p = pn[t]
        near = min(range(STEPS), key=lambda u: (abs(pk[u] - p), u))
        if bn[t] == blank and bk[near] == blank:
            return p
    return mid


def stitch(logits, thetas, a, max_windows):
    """One word from its K windows: logits (K,48,C), thetas (K,6) or None, a (K,) -> (labels (48 M,) int32 -1 padded,
    S float32, kept [(window, step)] in order, cuts)."""
    logits = np.asarray(logits, np.float32)
    K, blank = logits.shape[0], logits.shape[2] - 1
    pos = [positions(a[k], None if thetas is None else thetas[k]) for k in range(K)]
    st = [steps(logits[k]) for k in range(K)]
    cuts = []
    for k in range(K - 1):                        # never below the previous cut: no range is read twice
        c = cut(pos[k], st[k][0], pos[k + 1], st[k + 1][0], a[k], a[k + 1], blank)
        cuts.append(max(c, cuts[-1]) if cuts else c)
    labels, kept, prev, s = [], [], -1, np.float32(0)
    for k in range(K):
        lo = cuts[k - 1] if k else -np.inf
        hi = cuts[k] if k + 1 < K else np.inf
        for t in range(STEPS):
            if lo <= pos[k][t] < hi:
                c = int(st[k][0][t])
                s = np.float32(s + st[k][1][t])
                kept.append((k, t))
                if c != blank and c != prev:
                    labels.append(c)
                prev = c
    row = np.full(STEPS * max_windows, -1, np.int32)
    row[:len(labels)] = labels
    return row, s, kept, cuts


def random_boxes(seed, n, wide=0.7):
    """n rotated rectangles (float32 (n,4,2)), ``wide`` of them 7 to 40 times as wide as tall (wider than the crop at
    full height), the others 0.5 to 6.4 times."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        h = rng.uniform(8, 40)
        w = h * (rng.uniform(7, 40) if rng.random() < wide else rng.uniform(0.5, 6.4))
        out.append(I._rect(rng.uniform(0, 900), rng.uniform(0, 180), w, h, rng.uniform(-90, 90), int(rng.integers(4)),
                           bool(rng.integers(2))))
    return np.stack(out).astype(np.float32)


def wide_list(quads, m):
    """The wide boxes' indices (int32) and the CSR of their window starts (int32), as the recognizer builds them."""
    k = np.array([extent(q, m)[3] for q in quads])
    words = np.flatnonzero(k >= 2).astype(np.int32)
    start = np.zeros(len(words) + 1, np.int32)
    start[1:] = np.cumsum(k[words])
    return words, start


def stitch_case(seed, n_words, theta=True, classes=37):
    """Seeded inputs of b2o_stitch_windows: (quads, M, words, start, logits (W,48,classes) float32 with the blank
    favoured, theta (W,6) float32 near the identity or None)."""
    rng = np.random.default_rng(seed)
    quads = random_boxes(seed, n_words, wide=1.0)
    m = int(rng.choice([2, 4, 16]))
    words, start = wide_list(quads, m)
    total = int(start[-1])
    lg = rng.normal(size=(total, 48, classes)).astype(np.float32)
    lg[..., classes - 1] += rng.uniform(0, 2.5, size=(total, 48)).astype(np.float32)
    th = np.tile(np.array([1, 0, 0, 0, 1, 0], np.float32), (total, 1))
    th[:, 4] = rng.uniform(0.9, 1.05, total)
    th[:, 5] = rng.uniform(-0.05, 0.05, total)
    return quads, m, words, start, lg, th if theta else None


def greedy(logits):
    """Plain greedy CTC of one 48-step crop: (labels list, S)."""
    best, term = steps(logits)
    blank = np.asarray(logits).shape[1] - 1
    out, prev, s = [], -1, np.float32(0)
    for c, v in zip(best, term):
        if c != blank and c != prev:
            out.append(int(c))
        prev = c
        s = np.float32(s + v)
    return out, s


# ----------------------------------------------------------------------------------------------- rendered pages
LETTERS = list("abcdefghijklmnopqrstuvwxyz")


def long_word_page(seed, h=768, w=768, scale=0.9, thick=2, merged=0.3):
    """A white page of cv2.putText Hershey items, one per line: a word of 14 to 30 letters, or (with probability
    ``merged``) two words of 7 to 12 letters a quarter of a glyph height apart, which the detector takes as one box.
    Returns (page, items): items as (text, centre (x, y)) with the text the detector box should read (a merged pair's
    words concatenated), the centre that of the whole item."""
    import cv2

    rng = np.random.default_rng(seed)
    page = np.full((h, w, 3), 255, np.uint8)
    font = cv2.FONT_HERSHEY_SIMPLEX
    th = cv2.getTextSize("Ag", font, scale, thick)[0][1]
    items, y = [], 30 + th
    while y < h - 30:
        if rng.random() < merged:
            parts = ["".join(rng.choice(LETTERS, int(rng.integers(7, 13)))) for _ in range(2)]
        else:
            parts = ["".join(rng.choice(LETTERS, int(rng.integers(14, 31))))]
        x = 30
        for k, word in enumerate(parts):
            cv2.putText(page, word, (int(x), int(y)), font, scale, (0, 0, 0), thick, cv2.LINE_AA)
            x += cv2.getTextSize(word, font, scale, thick)[0][0] + (int(th / 4) if k == 0 else 0)
        if x < w - 10:
            items.append(("".join(parts), (30 + (x - 30) / 2, y - th / 2)))
        else:                                     # ran off the page: blank the line again
            page[max(0, int(y - 2 * th)):int(y + th), :] = 255
        y += int(2.6 * th)
    return page, items


def exact_reads(result, items):
    """Words of one page's ``Pipeline.recognize`` result whose box holds exactly one item centre and whose text is that
    item's."""
    import cv2

    n = 0
    for word in result:
        box = np.asarray(word[1], np.float32).reshape(-1, 1, 2)
        inside = [t for t, c in items if cv2.pointPolygonTest(box, (float(c[0]), float(c[1])), False) >= 0]
        n += len(inside) == 1 and word[0] == inside[0]
    return n
