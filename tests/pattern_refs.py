"""fp64 reference for the pattern-constrained CTC beam search (``b2o_ctc_beam_pattern_decode``; DESIGN.md section 1,
"Patterns"), and seeded pattern generators the tests share.

* ``beam_search_pattern``: the search of tests/beam_refs.py with a DFA state per beam -- a candidate in state q is kept
  after step t only if dist[q] <= T-1-t, an extension only by a label whose successor is defined -- with no shortlist
  (the kernel's pruning argument is what the tests check).  It records ``prune_margin``, ``rank_margin`` and ``ties`` as
  beam_refs.beam_search does.
* ``random_pattern``: a seeded random regular expression over the constructs ``recognition.Pattern`` accepts.
"""
import re

import numpy as np

NEG = -np.inf


def beam_search_pattern(lp, beam_width, trans, dist, start, top_paths=None):
    """The constrained search on one (T, K) array of log-probabilities and the host tables of a ``Pattern``.  Returns
    (paths, logp, info) for the ``top_paths`` (default: all) best surviving readings; fewer when fewer survive."""
    lp = np.asarray(lp, np.float64)
    T, K = lp.shape
    blank, W = K - 1, beam_width
    trans = np.asarray(trans, np.int64)
    dist = np.asarray(dist, np.int64)
    beams, pb, pnb, q = [()], np.array([0.0]), np.array([NEG]), np.array([start])
    prune, ties = np.inf, 0
    for t in range(T):
        limit = T - 1 - t
        row = lp[t]
        n = len(beams)
        if n == 0:
            break
        score = np.logaddexp(pb, pnb)
        last = np.array([b[-1] if b else -1 for b in beams])
        has = last >= 0
        ext = score[:, None] + row[None, :blank]
        ext[np.nonzero(has)[0], last[has]] = pb[has] + row[last[has]]
        nxt = trans[q]                                           # (n, K-1) successor states
        allowed = (nxt >= 0) & (dist[np.maximum(nxt, 0)] <= limit)
        stay_b = score + row[blank]
        stay_nb = np.where(has, pnb + row[np.maximum(last, 0)], NEG)
        index = {b: i for i, b in enumerate(beams)}
        for i, b in enumerate(beams):
            a = index.get(b[:-1]) if b else None
            if a is not None:
                stay_nb[i] = np.logaddexp(stay_nb[i], ext[a, b[-1]])
                ext[a, b[-1]] = NEG
        stay = np.logaddexp(stay_b, stay_nb)
        keep_ok = dist[q] <= limit
        stay = np.where(keep_ok, stay, NEG)
        ext = np.where(allowed, ext, NEG)
        valid = np.isfinite(ext)
        every = np.concatenate([stay[np.isfinite(stay)], ext[valid]])
        theta = -np.inf
        if every.size > W:
            top = -np.partition(-every, [W - 1, W])[[W - 1, W]]
            gap = top[0] - top[1]
            if gap == 0:
                ties += 1
            else:
                prune = min(prune, gap)
            theta = top[0]
        pool = [(-stay[i], beams[i], i, -1) for i in range(n) if np.isfinite(stay[i]) and stay[i] >= theta]
        for a in range(n):
            pool += [(-ext[a, c], beams[a] + (int(c),), a, int(c))
                     for c in np.nonzero(valid[a] & (ext[a] >= theta))[0]]
        pool.sort(key=lambda x: (x[0], x[1]))
        keep = pool[:W]
        beams = [k[1] for k in keep]
        pb = np.array([stay_b[k[2]] if k[3] < 0 else NEG for k in keep])
        pnb = np.array([stay_nb[k[2]] if k[3] < 0 else ext[k[2], k[3]] for k in keep])
        q = np.array([q[k[2]] if k[3] < 0 else nxt[k[2], k[3]] for k in keep], np.int64)
    if not beams:
        return [], np.zeros(0), {"prune_margin": float(prune), "rank_margin": np.inf, "ties": ties}
    score = np.logaddexp(pb, pnb)
    order = sorted(range(len(beams)), key=lambda i: (-score[i], beams[i]))
    p = len(order) if top_paths is None else min(top_paths, len(order))
    final = score[order]
    gaps = final[:-1] - final[1:] if len(final) > 1 else np.zeros(0)
    gaps = gaps[:p]
    ties += int((gaps == 0).sum())
    rank = float(gaps[gaps > 0].min()) if (gaps > 0).any() else np.inf
    return [beams[i] for i in order[:p]], final[:p], {"prune_margin": float(prune), "rank_margin": rank, "ties": ties}


def _class(rng, alphabet):
    """A random character class over ``alphabet`` (ranges, single characters, \\d, negation) that is not empty."""
    while True:
        parts = []
        for _ in range(int(rng.integers(1, 4))):
            kind = rng.integers(3)
            if kind == 0:
                lo, hi = sorted(alphabet[int(i)] for i in rng.integers(len(alphabet), size=2))
                parts.append(f"{lo}-{hi}")
            elif kind == 1:
                parts.append(alphabet[int(rng.integers(len(alphabet)))])
            elif any(c.isdigit() for c in alphabet):
                parts.append("\\d")
        neg = "^" if rng.random() < 0.25 else ""
        body = "".join(parts)
        if not body or body.startswith("^"):
            continue
        text = f"[{neg}{body}]"
        if any(re.fullmatch(text, c) for c in alphabet):
            return text


def random_pattern(rng, alphabet, depth=4):
    """A random regular expression over ``alphabet`` with nesting up to ``depth``: literals, ``.``, ``\\d`` (when the
    alphabet has digits), classes, groups ``( )`` / ``(?: )``, ``|`` and every quantifier, bounds small enough that the
    pattern usually compiles."""
    def atom(d):
        r = rng.random()
        if d <= 0 or r < 0.45:
            return alphabet[int(rng.integers(len(alphabet)))]
        if r < 0.52:
            return "."
        if r < 0.58 and any(c.isdigit() for c in alphabet):
            return "\\d"
        if r < 0.72:
            return _class(rng, alphabet)
        open_ = "(?:" if rng.random() < 0.5 else "("
        return open_ + alt(d - 1) + ")"

    def quant():
        r = rng.random()
        if r < 0.55:
            return ""
        m = int(rng.integers(0, 4))
        return ["?", "*", "+", f"{{{m}}}", f"{{{m},}}", f"{{{m},{m + int(rng.integers(0, 3))}}}"][int(rng.integers(6))]

    def cat(d):
        return "".join(atom(d) + quant() for _ in range(int(rng.integers(1, 4))))

    def alt(d):
        return "|".join(cat(d) for _ in range(int(rng.integers(1, 3))))

    return alt(depth)
