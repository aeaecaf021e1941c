"""fp64 references for the character language model (``recognition.CharLM``) and the LM-fused CTC prefix beam search
(``b2o_ctc_beam_lm_decode``, ``b2o_crnn_forward_beam_lm``).

* ``KneserNey``: interpolated Kneser-Ney evaluated directly from the counts, P(w | h) = max(a(h w) - D, 0) / a(h) +
  gamma(h) P(w | h') with the recursion written out (no backoff form, no tables): what ``CharLM.fit`` must equal.
* ``read_arpa``: a plain ARPA reader, {tuple of tokens: (log10 p, log10 bo)}.
* ``backoff_logp``: ARPA semantics on a model's tables, the per-(h, w) recursion the folded rows must equal.
* ``lookup_row``: the longest listed suffix of a prefix's history in the device keys, as the kernel looks it up.
* ``beam_search_lm``: ``beam_refs.beam_search`` with every candidate ranked by F = A + G: A the fp64 acoustic score, G
  accumulated in float32 from the float32 rows exactly as the kernel adds it, F in fp64; every label extends every beam
  (no shortlist: the kernel's per-beam pruning is what the tests check).  The returned paths rank by F_end = F +
  float32(alpha * l(</s> | hist)).  Margins as in ``beam_refs``: ``prune_margin`` over F, ``rank_margin`` over F_end,
  exact ties counted in ``ties``.
"""
import math

import numpy as np

NEG = -np.inf
BOS = 127


class KneserNey:
    """Interpolated Kneser-Ney of order n over symbols 0..V-1 (V - 1 = </s>), <s> = BOS, straight from the counts."""

    def __init__(self, words, alphabet, order):
        index = {ch: i for i, ch in enumerate(alphabet)}
        self.n, self.V = order, len(alphabet) + 1
        eos = len(alphabet)
        raw = {}
        for w in words:
            seq = (BOS,) + tuple(index[c] for c in w) + (eos,)
            for m in range(1, order + 1):
                for i in range(len(seq) - m + 1):
                    raw[seq[i:i + m]] = raw.get(seq[i:i + m], 0) + 1
        self.adj = {}
        for g, c in raw.items():
            if len(g) == order or g[0] == BOS:
                self.adj[g] = c
            else:
                self.adj[g] = len({v for v in range(BOS + 1) if (v,) + g in raw})
        self.adj.pop((BOS,), None)
        self.D = {}
        for m in range(1, order + 1):
            vals = [c for g, c in self.adj.items() if len(g) == m]
            n1, n2 = vals.count(1), vals.count(2)
            self.D[m] = n1 / (n1 + 2 * n2) if n1 and n2 else 0.5

    def prob(self, w, h):
        """P(w | h), h a tuple of at most n-1 symbols."""
        h = tuple(h)[len(h) - (self.n - 1):] if len(h) > self.n - 1 else tuple(h)
        m = len(h) + 1
        grams = {g: c for g, c in self.adj.items() if len(g) == m and g[:-1] == h}
        total = sum(grams.values())
        lower = (1.0 / self.V) if m == 1 else self.prob(w, h[1:])
        if total == 0:
            return lower
        d = self.D[m]
        return max(grams.get(h + (w,), 0) - d, 0.0) / total + d * len(grams) / total * lower


def read_arpa(text):
    """{tuple of tokens: (log10 p, log10 bo or 0.0)} of an ARPA text."""
    out, m = {}, 0
    for line in text.splitlines():
        s = line.strip()
        if s.startswith("\\") and s.endswith("-grams:"):
            m = int(s[1:-7])
        elif s == "\\end\\":
            break
        elif m and s:
            f = s.split()
            out[tuple(f[1:m + 1])] = (float(f[0]), float(f[m + 1]) if len(f) == m + 2 else 0.0)
    return out


def backoff_logp(lm, w, h):
    """Natural-log P(w | h) by ARPA's recursion on ``lm.logp10`` / ``lm.backoff10``, fp64."""
    h = tuple(h)[-(lm.order - 1):]
    if h + (w,) in lm.logp10:
        return lm.logp10[h + (w,)] * math.log(10)
    return lm.backoff10.get(h, 0.0) * math.log(10) + backoff_logp(lm, w, h[1:]) if h else NEG


def history_key(h):
    k = len(h) << 56
    for i, s in enumerate(h):
        k |= int(s) << (8 * (len(h) - 1 - i))
    return k


def lookup_row(keys, order, prefix):
    """Index of the longest listed suffix of the last order-1 symbols of "<s> prefix" in the sorted ``keys``."""
    seq = (BOS,) + tuple(prefix)
    where = {int(k): i for i, k in enumerate(keys)} if not isinstance(keys, dict) else keys
    for n in range(min(order - 1, len(seq)), 0, -1):
        i = where.get(history_key(seq[len(seq) - n:]))
        if i is not None:
            return i
    return 0


def beam_search_lm(lp, beam_width, keys, rows, order, alpha, beta, top_paths=None):
    """The fused search on one (T, K) array of log-probabilities and the device tables (keys, float32 rows).
    Returns (paths, A, F_end, info) for the ``top_paths`` (default: all) best readings."""
    lp = np.asarray(lp, np.float64)
    T, K = lp.shape
    blank, W = K - 1, beam_width
    where = {int(k): i for i, k in enumerate(keys)}
    a32, b32 = np.float32(alpha), np.float32(beta)
    rows = np.asarray(rows, np.float32)
    row_of = {}

    def lrow(prefix):
        if prefix not in row_of:
            row_of[prefix] = rows[lookup_row(where, order, prefix)]
        return row_of[prefix]

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
        gext = gext.astype(np.float64)                # float32 sums, each rounded as the kernel rounds them
        f_stay = stay + np.array(G, np.float64)
        f_ext = ext + gext
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
    F = A + np.array(G, np.float64)
    fend = F + np.array([np.float32(a32 * lrow(b)[blank]) for b in beams], np.float64)
    order_ = sorted(range(len(beams)), key=lambda i: (-fend[i], beams[i]))
    p = len(order_) if top_paths is None else min(top_paths, len(order_))
    final = fend[order_]
    gaps = final[:-1] - final[1:] if len(final) > 1 else np.zeros(0)
    gaps = gaps[:p]
    ties += int((gaps == 0).sum())
    rank = float(gaps[gaps > 0].min()) if (gaps > 0).any() else np.inf
    return ([beams[i] for i in order_[:p]], A[order_][:p], final[:p],
            {"prune_margin": float(prune), "rank_margin": rank, "ties": ties})


def fused_score(lp, path, keys, rows, order, alpha, beta):
    """F_end of one label sequence with its exact acoustic log-probability (the forward algorithm)."""
    from tests import beam_refs as BR
    where = {int(k): i for i, k in enumerate(keys)}
    rows = np.asarray(rows, np.float32)
    a32, b32 = np.float32(alpha), np.float32(beta)
    g = np.float32(0.0)
    for i, c in enumerate(path):
        g = np.float32(g + np.float32(np.float32(a32 * rows[lookup_row(where, order, path[:i])][c]) + b32))
    blank = rows.shape[1] - 1
    return BR.forward_logprob(lp, path) + float(g) + float(np.float32(a32 * rows[lookup_row(where, order, path)][blank]))
