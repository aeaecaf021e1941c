"""fp64 references for hotword boosting (``recognition.Hotwords``, ``b2o_ctc_beam_hotword_decode``,
``b2o_crnn_forward_beam_hotword``).

* ``dict_trie``: the trie of a word list as nested Python dicts, numbered breadth-first by (depth, parent, label) --
  what ``recognition.compile_trie``'s arrays must describe.
* ``prefixes``: every live prefix of a list (the prefixes of its words, the empty one included).
* ``beam_search_hot``: ``lm_refs.beam_search_lm`` with every candidate ranked by F = A + G + H, H(a) = float32(gamma |a|)
  for a live prefix a, else 0, and the returned paths by F_end = A + G + float32(alpha l(</s> | hist)) + H_end,
  H_end(a) = float32(gamma |a|) for a listed word, else 0.  Without a model (``keys=None``) G = 0 and alpha = 0.  Every
  label extends every beam (no shortlist); margins and exact ties as in ``lm_refs``.
* ``fused_score``: F_end of one label sequence with its exact acoustic log-probability (the forward algorithm).
"""
import numpy as np

from tests import beam_refs as BR
from tests import lm_refs as LR

NEG = -np.inf


def encode(words, alphabet):
    index = {ch: i for i, ch in enumerate(alphabet)}
    return [tuple(index[ch] for ch in w) for w in words]


def dict_trie(seqs):
    """(nodes, final): nodes[i] = (parent, label, prefix) in breadth-first (depth, parent, label) order, the root
    (-1, -1, ()); final[i] whether prefix i is listed."""
    root = {}
    for s in seqs:
        d = root
        for c in s:
            d = d.setdefault(c, {})
        d[None] = True                                       # end of a word
    nodes, final, level = [(-1, -1, ())], [bool(root.get(None))], [(0, root)]
    while level:
        nxt = []
        for i, d in level:                                   # parents in node order
            for c in sorted(k for k in d if k is not None):
                nodes.append((i, c, nodes[i][2] + (c,)))
                final.append(bool(d[c].get(None)))
                nxt.append((len(nodes) - 1, d[c]))
        level = nxt
    return nodes, final


def prefixes(seqs):
    out = {()}
    for s in seqs:
        out.update(tuple(s[:i]) for i in range(1, len(s) + 1))
    return out


def _zero_model(K):
    return np.zeros(1, np.uint64), np.zeros((1, K), np.float32), 2, 0.0, 0.0


def bonus(gamma, n):
    return float(np.float32(np.float32(gamma) * np.float32(n)))


def beam_search_hot(lp, beam_width, seqs, gamma, keys=None, rows=None, order=2, alpha=0.0, beta=0.0, top_paths=None):
    """The search on one (T, K) array of log-probabilities: ``seqs`` the listed words as label tuples, ``gamma`` the
    weight; (keys, rows, order, alpha, beta) the device tables of a model, or keys=None for none.  Returns (paths, A,
    F_end, info) for the ``top_paths`` (default: all) best readings."""
    lp = np.asarray(lp, np.float64)
    T, K = lp.shape
    if keys is None:
        keys, rows, order, alpha, beta = _zero_model(K)
    blank, W = K - 1, beam_width
    live, words = prefixes(seqs), set(map(tuple, seqs))
    where = {int(k): i for i, k in enumerate(keys)}
    a32, b32 = np.float32(alpha), np.float32(beta)
    rows = np.asarray(rows, np.float32)
    row_of = {}

    def lrow(prefix):
        if prefix not in row_of:
            row_of[prefix] = rows[LR.lookup_row(where, order, prefix)]
        return row_of[prefix]

    def H(prefix):
        return bonus(gamma, len(prefix)) if prefix in live else 0.0

    beams, pb, pnb, G = [()], np.array([0.0]), np.array([NEG]), [np.float32(0.0)]
    prune, ties = np.inf, 0
    for t in range(T):
        row = lp[t]
        n = len(beams)
        score = np.logaddexp(pb, pnb)
        last = np.array([b[-1] if b else -1 for b in beams])
        has = last >= 0
        ext = score[:, None] + row[None, :blank]
        ext[np.nonzero(has)[0], last[has]] = pb[has] + row[last[has]]
        stay_b = score + row[blank]
        stay_nb = np.where(has, pnb + row[np.maximum(last, 0)], NEG)
        index = {b: i for i, b in enumerate(beams)}
        for i, b in enumerate(beams):
            a = index.get(b[:-1]) if b else None
            if a is not None:
                stay_nb[i] = np.logaddexp(stay_nb[i], ext[a, b[-1]])
                ext[a, b[-1]] = NEG
        stay = np.logaddexp(stay_b, stay_nb)
        gext = np.array([np.float32(G[a]) + (a32 * lrow(beams[a])[:blank] + b32) for a in range(n)], np.float32)
        gext = gext.astype(np.float64)
        hstay = np.array([H(b) for b in beams])
        hext = np.array([[H(b + (c,)) for c in range(blank)] for b in beams]).reshape(n, blank)
        f_stay = stay + np.array(G, np.float64) + hstay
        f_ext = ext + gext + hext
        valid = np.isfinite(ext)
        every = np.concatenate([f_stay, f_ext[valid]])
        theta = -np.inf
        if every.size > W:
            top = -np.partition(-every, [W - 1, W])[[W - 1, W]]
            gap = top[0] - top[1]
            if gap == 0:
                ties += 1
            else:
                prune = min(prune, gap)
            theta = top[0]
        pool = [(-f_stay[i], beams[i], i, -1) for i in range(n) if f_stay[i] >= theta]
        for a in range(n):
            pool += [(-f_ext[a, c], beams[a] + (int(c),), a, int(c))
                     for c in np.nonzero(valid[a] & (f_ext[a] >= theta))[0]]
        pool.sort(key=lambda x: (x[0], x[1]))
        keep = pool[:W]
        beams = [k[1] for k in keep]
        pb = np.array([stay_b[k[2]] if k[3] < 0 else NEG for k in keep])
        pnb = np.array([stay_nb[k[2]] if k[3] < 0 else ext[k[2], k[3]] for k in keep])
        G = [G[k[2]] if k[3] < 0 else np.float32(gext[k[2], k[3]]) for k in keep]
    A = np.logaddexp(pb, pnb)
    hend = np.array([bonus(gamma, len(b)) if b in words else 0.0 for b in beams])
    fend = (A + np.array(G, np.float64) + np.array([np.float32(a32 * lrow(b)[blank]) for b in beams], np.float64)
            + hend)
    order_ = sorted(range(len(beams)), key=lambda i: (-fend[i], beams[i]))
    p = len(order_) if top_paths is None else min(top_paths, len(order_))
    final = fend[order_]
    gaps = final[:-1] - final[1:] if len(final) > 1 else np.zeros(0)
    gaps = gaps[:p]
    ties += int((gaps == 0).sum())
    rank = float(gaps[gaps > 0].min()) if (gaps > 0).any() else np.inf
    return ([beams[i] for i in order_[:p]], A[order_][:p], final[:p],
            {"prune_margin": float(prune), "rank_margin": rank, "ties": ties})


def fused_score(lp, path, seqs, gamma, keys=None, rows=None, order=2, alpha=0.0, beta=0.0):
    """F_end of one label sequence: its exact acoustic log-probability + G + alpha l(</s> | path) + H_end."""
    lp = np.asarray(lp, np.float64)
    if keys is None:
        keys, rows, order, alpha, beta = _zero_model(lp.shape[1])
    h = bonus(gamma, len(path)) if tuple(path) in set(map(tuple, seqs)) else 0.0
    return LR.fused_score(lp, tuple(path), keys, rows, order, alpha, beta) + h


def exhaustive_best(lp, seqs, gamma, **model):
    """(path, F_end) of the label sequence with the largest F_end over every sequence of nonzero probability (tiny T,
    K only: ``beam_refs.brute_force``)."""
    best = None
    for seq in BR.brute_force(lp):
        f = fused_score(lp, seq, seqs, gamma, **model)
        if best is None or f > best[1] or (f == best[1] and seq < best[0]):
            best = (seq, f)
    return best
