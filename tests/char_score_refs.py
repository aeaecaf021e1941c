"""fp64 references for character scores (``b2o_ctc_char_scores``, DESIGN.md section 1, "Character scores").

* ``definition``: the definition taken literally -- ``beam_refs.forward_logprob`` of every one-character edit of the
  reading (the K-1 substitutions, then the deletion labelled K-1), one forward pass per edit.
* ``recipe``: the kernel's computation in fp64 -- one forward (alpha) and one backward (beta) pass over the reading's
  2n+1 states, a gamma sweep per (position, substituted label) and a split at the suffix's first label per deletion.
* ``scores``: F (n, K) -> the confidences, the top-A alternatives and posteriors under the tie rule, and the ranking
  margins the GPU test needs.
"""
import numpy as np

from tests import beam_refs as BR

NEG = -np.inf


def edits(y, k, n_classes):
    """The K one-character edits of ``y`` at position k: substitutions by 0 .. K-2, then the deletion."""
    y = list(y)
    return [y[:k] + [c] + y[k + 1:] for c in range(n_classes - 1)] + [y[:k] + y[k + 1:]]


def definition(lp, y):
    """(F (n, K) fp64, logp): F[k, e] = forward_logprob(y[k -> e]) for a (T, K) lp at any T, logp = F(y)."""
    lp = np.asarray(lp, np.float64)
    n_classes = lp.shape[1]
    f = np.full((len(y), n_classes), NEG)
    for k in range(len(y)):
        f[k] = [BR.forward_logprob(lp, z) for z in edits(y, k, n_classes)]
    return f, BR.forward_logprob(lp, list(y))


def _lae(a, b):
    with np.errstate(invalid="ignore"):
        return np.logaddexp(a, b)


def recipe(lp, y):
    """(F (n, K) fp64, logp) by forward-backward: the alpha / beta / gamma recipe the kernel runs, in fp64."""
    lp = np.asarray(lp, np.float64)
    T, K = lp.shape
    blank, n, y = K - 1, len(y), [int(c) for c in y]
    ext = [blank]
    for c in y:
        ext += [c, blank]
    ext = np.array(ext)
    S = len(ext)
    skip = np.zeros(S, bool)
    skip[2:] = (ext[2:] != blank) & (ext[2:] != ext[:-2])
    alpha, beta = np.full((T, S), NEG), np.full((T, S), NEG)
    alpha[0, 0] = lp[0, blank]
    if n:
        alpha[0, 1] = lp[0, ext[1]]
    for t in range(1, T):
        a = alpha[t - 1].copy()
        a[1:] = _lae(a[1:], alpha[t - 1, :-1])
        a[2:] = np.where(skip[2:], _lae(a[2:], alpha[t - 1, :-2]), a[2:])
        alpha[t] = a + lp[t, ext]
    beta[T - 1, S - 1] = lp[T - 1, blank]
    if n:
        beta[T - 1, S - 2] = lp[T - 1, ext[S - 2]]
    for t in range(T - 2, -1, -1):
        b = beta[t + 1].copy()
        b[:-1] = _lae(b[:-1], beta[t + 1, 1:])
        b[:-2] = np.where(skip[2:], _lae(b[:-2], beta[t + 1, 2:]), b[:-2])
        beta[t] = b + lp[t, ext]
    logp = float(_lae(alpha[T - 1, S - 1], alpha[T - 1, S - 2]) if n else alpha[T - 1, 0])
    f = np.full((n, K), NEG)
    c = np.arange(K - 1)
    for k in range(n):
        prev = y[k - 1] if k else -1
        nxt = y[k + 1] if k + 1 < n else -1
        # A[t] = A(t-1): the prefix y_<k ends at step t-1 (A(-1) = 0 for an empty prefix)
        a_in = np.full((T, K - 1), NEG)
        a_in[0] = 0.0 if k == 0 else NEG
        if k:
            a_in[1:] = np.where(c[None] != prev, _lae(alpha[:-1, 2 * k], alpha[:-1, 2 * k - 1])[:, None],
                                alpha[:-1, 2 * k][:, None])
        else:
            a_in[1:] = alpha[:-1, 0][:, None]
        # B[t] = B(t+1): the suffix y_>k starts at step t+1 (B(T) = 0 for an empty suffix)
        b_out = np.full((T, K - 1), NEG)
        b_out[T - 1] = 0.0 if k == n - 1 else NEG
        if k + 1 < n:
            b_out[:-1] = np.where(c[None] != nxt, _lae(beta[1:, 2 * k + 2], beta[1:, 2 * k + 3])[:, None],
                                  beta[1:, 2 * k + 2][:, None])
        else:
            b_out[:-1] = beta[1:, 2 * k + 2][:, None]
        g, acc = np.full(K - 1, NEG), np.full(K - 1, NEG)
        for t in range(T):
            g = lp[t, :K - 1] + _lae(g, a_in[t])
            acc = _lae(acc, g + b_out[t])
        f[k, :K - 1] = acc
        if k == n - 1:                                            # deleting the last character: the prefix's end
            f[k, blank] = _lae(alpha[T - 1, 2 * k], alpha[T - 1, 2 * k - 1]) if k else alpha[T - 1, 0]
        else:                                                     # split at the step the suffix's first label starts
            d_in = np.full(T, NEG)
            d_in[0] = 0.0 if k == 0 else NEG
            if k and prev != nxt:
                d_in[1:] = _lae(alpha[:-1, 2 * k], alpha[:-1, 2 * k - 1])
            else:
                d_in[1:] = alpha[:-1, 2 * k]
            f[k, blank] = np.logaddexp.reduce(d_in + beta[:, 2 * k + 3])
    return f, logp


def scores(f, y, alternatives):
    """F (n, K) -> (conf (n,), labels (n, A) int, post (n, A), margin (n,)): pi = exp(F - logsumexp F) per position,
    conf = pi[y_k], the A largest pi best first (equal values: smaller label), -1 / 0 past the K edits and everywhere
    at a position whose edits all score -inf.  ``margin``: the smallest gap between consecutive values of the ranking
    down to place A+1 (inf with nothing to rank; a gap between two impossible edits, F = -inf in any precision, counts
    as inf) -- where it exceeds the kernel's error, the kernel's labels are the reference's."""
    f = np.asarray(f, np.float64)
    n, K = f.shape
    conf = np.zeros(n)
    labels = np.full((n, alternatives), -1, np.int64)
    post = np.zeros((n, alternatives))
    margin = np.full(n, np.inf)
    for k in range(n):
        m = f[k].max()
        if not np.isfinite(m):
            continue
        pi = np.exp(f[k] - m)
        pi /= pi.sum()
        conf[k] = pi[y[k]]
        order = np.lexsort((np.arange(K), -pi))
        a = min(alternatives, K)
        labels[k, :a] = order[:a]
        post[k, :a] = pi[order[:a]]
        top = order[:min(alternatives + 1, K)]
        gaps = pi[top[:-1]] - pi[top[1:]]
        gaps[np.isneginf(f[k, top[:-1]]) & np.isneginf(f[k, top[1:]])] = np.inf     # impossible edits tie exactly
        if alternatives and gaps.size:
            margin[k] = gaps.min()
    return conf, labels, post, margin
