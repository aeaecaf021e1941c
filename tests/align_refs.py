"""fp64 references for character positions (``b2o_ctc_align``, ``b2o_char_cells``; DESIGN.md section 1).

* ``viterbi``: the best single CTC alignment of a label sequence over lp (T, K) (blank = K-1), with the kernel's tie rule:
  among equal predecessors staying wins, then advancing by one, then skipping a blank; the alignment ends in the last
  label's state unless the trailing blank scores strictly more.  Returns the score and each character's span (first,
  last step), and the smallest winning margin of the decisions on the returned path (``margin``, for the GPU tests).
* ``brute_force``: the same by enumerating all K^T alignments (tiny T, K only).  Among the optimal alignments the tie
  rule picks the one whose state at the last step is smallest, then whose states at steps T-2, T-3, ..., 0 are largest.
* ``cells``: the character quads of a reading's spans through the STN's theta and warpBox's inverse homography, in the
  kernel's operation order (fp64, one rounding to float32).
"""
import itertools

import numpy as np

from tests import cvmodels as M
from tests import rotation_refs as RR

NEG = -np.inf
STEPS, DISCARD, CROP_W, CROP_H = 48, 2, 200, 31


def _states(labels, blank):
    ext = [blank]
    for c in labels:
        ext += [int(c), blank]
    ext = np.array(ext)
    skip = np.zeros(len(ext), bool)
    skip[2:] = (ext[2:] != blank) & (ext[2:] != ext[:-2])
    return ext, skip


def spans_of(states, n):
    """(n, 2) int32 first / last step of every character's state (2k+1) on a state sequence."""
    out = np.full((n, 2), -1, np.int32)
    for t, s in enumerate(states):
        if s & 1:
            k = s >> 1
            if out[k, 0] < 0:
                out[k, 0] = t
            out[k, 1] = t
    return out


def viterbi(lp, labels):
    """(score, spans (n,2) int32, margin) of the best alignment of ``labels`` under lp (T, K); score -inf and spans -1
    where no alignment exists (or a label is outside [0, K-2]).  ``margin``: the smallest gap between the chosen and the
    best other candidate over the decisions on the returned path (inf when there is none)."""
    lp = np.asarray(lp, np.float64)
    T, K = lp.shape
    labels = [int(c) for c in labels]
    n = len(labels)
    if any(c < 0 or c > K - 2 for c in labels):
        return NEG, np.full((n, 2), -1, np.int32), np.inf
    ext, skip = _states(labels, K - 1)
    S = len(ext)
    d = np.full(S, NEG)
    d[0] = lp[0, K - 1]
    if S > 1:
        d[1] = lp[0, ext[1]]
    back = np.zeros((T, S), np.int64)
    gaps = np.full((T, S), np.inf)
    cols = np.arange(S)
    for t in range(1, T):
        cand = np.full((3, S), NEG)
        cand[0] = d
        cand[1, 1:] = d[:-1]
        cand[2, 2:] = np.where(skip[2:], d[:-2], NEG)
        ch = np.argmax(cand, 0)                                  # the first maximum: stay, advance, skip
        best = cand[ch, cols]
        rest = cand.copy()
        rest[ch, cols] = NEG
        second = rest.max(0)
        ok = (best > NEG) & (second > NEG)
        gaps[t, ok] = best[ok] - second[ok]
        back[t] = ch
        d = best + lp[t, ext]
    last, tail = (d[S - 2] if n else NEG), d[S - 1]
    s = S - 1 if tail > last else S - 2
    score = max(last, tail)
    if not np.isfinite(score):
        return NEG, np.full((n, 2), -1, np.int32), np.inf
    margin = abs(tail - last) if n and np.isfinite(last) and np.isfinite(tail) else np.inf
    states = [0] * T
    for t in range(T - 1, -1, -1):
        states[t] = s
        if t > 0:
            margin = min(margin, gaps[t, s])
            s -= back[t, s]
    return float(score), spans_of(states, n), float(margin)


def brute_force(lp, labels):
    """(score, spans) of ``viterbi`` by enumerating every alignment; the tie rule as in the module docstring."""
    lp = np.asarray(lp, np.float64)
    T, K = lp.shape
    blank, labels = K - 1, tuple(int(c) for c in labels)
    best, pick = NEG, None
    for path in itertools.product(range(K), repeat=T):
        # the state sequence of an alignment: the label index walks forward on every new label
        states, k, prev, ok = [], -1, None, True
        for c in path:
            if c == blank:
                states.append(2 * (k + 1))
            else:
                if c != prev:
                    k += 1
                    if k >= len(labels) or labels[k] != c:
                        ok = False
                        break
                states.append(2 * k + 1)
            prev = c
        if not ok or k != len(labels) - 1:
            continue
        v = float(sum(lp[t, c] for t, c in enumerate(path)))
        key = (states[-1],) + tuple(-s for s in states[-2::-1])
        if v > best or (v == best and key < pick[0]):
            best, pick = v, (key, states)
    if pick is None:
        return NEG, np.full((len(labels), 2), -1, np.int32)
    return best, spans_of(pick[1], len(labels))


def greedy_runs(lp):
    """The argmax path's collapse and the runs of its labels: (labels, spans (n,2))."""
    path = np.argmax(np.asarray(lp), -1)
    blank = lp.shape[1] - 1
    labels, spans, prev = [], [], None
    for t, c in enumerate(path):
        if c != blank:
            if c != prev:
                labels.append(int(c))
                spans.append([t, t])
            else:
                spans[-1][1] = t
        prev = c
    return labels, np.array(spans, np.int32).reshape(-1, 2)


def cut_x(spans, j, theta):
    """Crop x of the cut before character j (kernel operation order)."""
    r = 0.5 * float(spans[j - 1][1] + spans[j][0]) + DISCARD
    u = r
    if theta is not None:
        gy = -1.0 + (2.0 * r) / 49.0
        u = (0.5 * ((float(np.float32(theta[4])) * gy + float(np.float32(theta[5]))) + 1.0)) * 50.0
    return 4.0 * u + 1.5


def plan(quad, turn):
    """(rolled box (4,2) float32, inverse homography m (9,) float64, sw, sh) of the crop in ``turn``, or None where
    warpBox raises ZeroDivisionError; ``quad`` None: the 200 x 31 crop frame (m None)."""
    if quad is None:
        frame = np.array([[0, 0], [CROP_W, 0], [CROP_W, CROP_H], [0, CROP_H]], np.float32)
        return frame, None, float(CROP_W), float(CROP_H)
    from oracle import imageops
    box = RR.turned_box(quad, turn)
    try:
        fwd, _, _ = RR.turned_transform(quad, turn)
    except ZeroDivisionError:
        return None
    w, h = imageops.rotated_width_height(box)
    scale = min(CROP_W / w, CROP_H / h)
    return box, M.inv3(fwd).reshape(-1), float(np.float32(scale * w)), float(np.float32(scale * h))


def cells(spans, theta=None, quad=None, turn=0):
    """(n, 4, 2) float32 cells of a reading's spans (n, 2): NaN where the plan is invalid."""
    spans = np.asarray(spans)
    n = len(spans)
    p = plan(quad, turn)
    if p is None:
        return np.full((n, 4, 2), np.nan, np.float32)
    box, m, sw, sh = p
    cuts, run = [0.0], 0.0
    for j in range(1, n):
        run = max(run, min(max(cut_x(spans, j, theta), 0.0), sw))
        cuts.append(run)
    cuts.append(sw)
    out = np.empty((n, 4, 2), np.float32)
    for k in range(n):
        a, b = cuts[k], cuts[k + 1]
        for c, (x, y) in enumerate(((a, 0.0), (b, 0.0), (b, sh), (a, sh))):
            if (k == 0 and c in (0, 3)) or (k == n - 1 and c in (1, 2)):
                out[k, c] = box[c]
            elif m is None:
                out[k, c] = (x, y)
            else:
                X = (m[0] * x + m[1] * y) + m[2]
                Y = (m[3] * x + m[4] * y) + m[5]
                W = (m[6] * x + m[7] * y) + m[8]
                out[k, c] = (X / W, Y / W)
    return out
