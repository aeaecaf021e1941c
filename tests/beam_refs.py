"""fp64 references for CTC beam-search decoding (``b2o_ctc_beam_decode``, ``b2o_crnn_forward_beam``).

* ``log_probs``: lp[t,c] = log(softmax(l_t)_c + 1e-7), the per-step inputs of the decoder (blank = K-1).
* ``forward_logprob``: the exact log-probability of a label sequence, sum over every alignment that collapses to it, by
  the CTC forward algorithm (checked against ``torch.nn.functional.ctc_loss`` and brute force on the CPU).
* ``brute_force``: every label sequence's exact log-probability by enumerating all K^T alignments (tiny T, K only).
* ``beam_search``: CTC prefix beam search with the kernel's definition -- candidates via blank, via the last label and
  by EVERY label (no shortlist: the kernel's pruning argument is what the tests check), merged with logaddexp, the W best
  kept, equal scores ordered by label sequence (a prefix before its extensions).  It also records the smallest gap at the
  selection boundary of every step (``prune_margin``: W-th against (W+1)-th candidate) and between consecutive returned
  paths (``rank_margin``); exact ties (gap 0, resolved by the tie rule) are counted apart in ``ties``.
"""
import itertools

import numpy as np

NEG = -np.inf


def log_probs(logits):
    """(..., T, K) logits -> fp64 log(softmax + 1e-7)."""
    lg = np.asarray(logits, np.float64)
    m = lg.max(-1, keepdims=True)
    e = np.exp(lg - m)
    return np.log(e / e.sum(-1, keepdims=True) + 1e-7)


def collapse(path, blank):
    """Alignment -> label sequence: merge repeats, drop blanks."""
    out, prev = [], None
    for c in path:
        if c != prev and c != blank:
            out.append(int(c))
        prev = c
    return tuple(out)


def forward_logprob(lp, labels):
    """log sum over the alignments of ``labels`` (a sequence of non-blank labels) of sum_t lp[t, path_t]."""
    lp = np.asarray(lp, np.float64)
    T, K = lp.shape
    blank = K - 1
    ext = [blank]
    for c in labels:
        ext += [int(c), blank]
    ext = np.array(ext)
    S = len(ext)
    skip = np.zeros(S, bool)                                      # s-2 -> s: a label that differs from the one before
    skip[2:] = (ext[2:] != blank) & (ext[2:] != ext[:-2])
    alpha = np.full(S, NEG)
    alpha[0] = lp[0, blank]
    if S > 1:
        alpha[1] = lp[0, ext[1]]
    for t in range(1, T):
        a = alpha.copy()
        a[1:] = np.logaddexp(a[1:], alpha[:-1])
        a[2:] = np.where(skip[2:], np.logaddexp(a[2:], alpha[:-2]), a[2:])
        alpha = a + lp[t, ext]
    return float(np.logaddexp(alpha[-1], alpha[-2]) if S > 1 else alpha[-1])


def brute_force(lp):
    """{label sequence: exact log-probability} by enumerating all K^T alignments."""
    lp = np.asarray(lp, np.float64)
    T, K = lp.shape
    out = {}
    for path in itertools.product(range(K), repeat=T):
        seq = collapse(path, K - 1)
        v = float(sum(lp[t, c] for t, c in enumerate(path)))
        out[seq] = np.logaddexp(out[seq], v) if seq in out else v
    return out


def ranked(scores):
    """[(sequence, logp)] of a {sequence: logp} dict in the decoder's order: logp descending, then sequence ascending."""
    return sorted(scores.items(), key=lambda kv: (-kv[1], kv[0]))


def beam_search(lp, beam_width, top_paths=None):
    """CTC prefix beam search on one (T, K) array of per-step log-probabilities.  Returns (paths, logp, info): the
    ``top_paths`` (default: all) best label sequences as tuples, their fp64 scores, and {"prune_margin", "rank_margin",
    "ties"}."""
    lp = np.asarray(lp, np.float64)
    T, K = lp.shape
    blank, W = K - 1, beam_width
    beams, pb, pnb = [()], np.array([0.0]), np.array([NEG])
    prune, ties = np.inf, 0
    for t in range(T):
        row = lp[t]
        n = len(beams)
        score = np.logaddexp(pb, pnb)
        last = np.array([b[-1] if b else -1 for b in beams])
        has = last >= 0
        ext = score[:, None] + row[None, :blank]                 # every beam by every label
        ext[np.nonzero(has)[0], last[has]] = pb[has] + row[last[has]]     # a repeated label only after a blank
        stay_b = score + row[blank]
        stay_nb = np.where(has, pnb + row[np.maximum(last, 0)], NEG)
        index = {b: i for i, b in enumerate(beams)}
        for i, b in enumerate(beams):                             # an extension that is already a beam merges into it
            a = index.get(b[:-1]) if b else None
            if a is not None:
                stay_nb[i] = np.logaddexp(stay_nb[i], ext[a, b[-1]])
                ext[a, b[-1]] = NEG
        stay = np.logaddexp(stay_b, stay_nb)
        valid = np.isfinite(ext)
        every = np.concatenate([stay, ext[valid]])
        if every.size > W:
            top = -np.partition(-every, [W - 1, W])[[W - 1, W]]
            gap = top[0] - top[1]
            if gap == 0:
                ties += 1
            else:
                prune = min(prune, gap)
            theta = top[0]
        else:
            theta = -np.inf
        pool = [(-stay[i], beams[i], i, -1) for i in range(n) if stay[i] >= theta]
        for a in range(n):
            cols = np.nonzero(valid[a] & (ext[a] >= theta))[0]
            if cols.size > W:                                     # W of this row's own candidates come first anyway
                cols = cols[np.lexsort((cols, -ext[a, cols]))[:W]]
            pool += [(-ext[a, c], beams[a] + (int(c),), a, int(c)) for c in cols]
        pool.sort(key=lambda x: (x[0], x[1]))
        keep = pool[:W]
        beams = [k[1] for k in keep]
        pb = np.array([stay_b[k[2]] if k[3] < 0 else NEG for k in keep])
        pnb = np.array([stay_nb[k[2]] if k[3] < 0 else ext[k[2], k[3]] for k in keep])
    score = np.logaddexp(pb, pnb)
    order = sorted(range(len(beams)), key=lambda i: (-score[i], beams[i]))
    p = len(order) if top_paths is None else min(top_paths, len(order))
    final = score[order]
    gaps = final[:-1] - final[1:] if len(final) > 1 else np.zeros(0)
    gaps = gaps[:p]                                               # order of the returned paths and the one after them
    ties += int((gaps == 0).sum())
    rank = float(gaps[gaps > 0].min()) if (gaps > 0).any() else np.inf
    return [beams[i] for i in order[:p]], final[:p], {"prune_margin": float(prune), "rank_margin": rank, "ties": ties}
