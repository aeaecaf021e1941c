"""fp64 references for lexicon-constrained CTC decoding (``b2o_ctc_lexicon_decode``, ``b2o_crnn_forward_lexicon``).

* ``scores``: every entry's exact CTC forward log-probability over lp = ``beam_refs.log_probs`` (blank = K-1), -inf for
  an entry that cannot be aligned in T steps.  Short lexicons go through ``beam_refs.forward_logprob`` entry by entry;
  ``scores_many`` runs the same recursion for a whole lexicon at once (linear domain, fp64, rescaled every step, states
  that can no longer reach the end dropped) and is checked against ``forward_logprob`` on the CPU.
* ``top_entries``: the decoder's result order -- score descending, equal scores by lexicon index ascending, -inf
  entries never returned -- and the smallest gap between consecutive scores among the returned entries and the first
  one left out (``margin``); exact ties (gap 0, resolved by the index rule) are counted apart in ``ties``.
"""
import numpy as np

from tests import beam_refs as BR


def alignable(entry, steps=48):
    """An entry fits in ``steps`` steps when its length plus its adjacent repeats (each needs a blank) does."""
    entry = list(entry)
    return len(entry) + sum(a == b for a, b in zip(entry, entry[1:])) <= steps


def scores(lp, entries):
    """(n,) fp64 scores of label sequences ``entries`` by ``beam_refs.forward_logprob``."""
    t = np.asarray(lp).shape[0]
    return np.array([BR.forward_logprob(lp, e) if alignable(e, t) else -np.inf for e in entries])


def need_steps(lab):
    """(n, 2L+1) steps each state of (n, L) equal-length entries needs to reach a final state: one per label still to
    come, one per blank a repeated label among them needs, one more from a blank state."""
    n, length = lab.shape
    rep = np.zeros((n, length), np.int64)
    rep[:, 1:] = lab[:, 1:] == lab[:, :-1]
    after = np.cumsum(rep[:, ::-1], 1)[:, ::-1] - rep               # repeats at positions > i
    label_need = (length - 1 - np.arange(length))[None, :] + after
    need = np.zeros((n, 2 * length + 1), np.int64)
    need[:, 1::2] = label_need
    need[:, 0:-1:2] = label_need + 1
    need[:, -1] = 0
    return need


def scores_many(lp, entries):
    """``scores`` for a whole lexicon at once: entries of equal length share one vectorised recursion."""
    lp = np.asarray(lp, np.float64)
    T, K = lp.shape
    blank = K - 1
    q = np.exp(lp)
    out = np.full(len(entries), -np.inf)
    by_len = {}
    for i, e in enumerate(entries):
        if alignable(e, T):
            by_len.setdefault(len(e), []).append(i)
    for length, idx in by_len.items():
        lab = np.array([entries[i] for i in idx], np.int64).reshape(len(idx), length)
        n, S = len(idx), 2 * length + 1
        ext = np.full((n, S), blank, np.int64)
        ext[:, 1::2] = lab
        skip = np.zeros((n, S), bool)
        skip[:, 3::2] = lab[:, 1:] != lab[:, :-1]
        need = need_steps(lab)
        alpha = np.zeros((n, S))
        alpha[:, 0] = q[0, blank]
        alpha[:, 1] = q[0, ext[:, 1]]
        alpha[need > T - 1] = 0.0
        logscale = np.zeros(n)
        for t in range(1, T):
            a = alpha.copy()
            a[:, 1:] += alpha[:, :-1]
            a[:, 2:] += np.where(skip[:, 2:], alpha[:, :-2], 0.0)
            alpha = a * q[t][ext]
            alpha[need > T - 1 - t] = 0.0                         # cannot reach the end any more: exact to drop
            m = alpha.max(1)
            alpha /= m[:, None]
            logscale += np.log(m)
        out[idx] = np.log(alpha[:, -1] + alpha[:, -2]) + logscale
    return out


def top_entries(ref, p):
    """(indices, scores, {"margin", "ties"}) of the ``p`` best entries of fp64 ``ref`` in the decoder's order."""
    ref = np.asarray(ref, np.float64)
    order = np.lexsort((np.arange(len(ref)), -ref))
    order = order[np.isfinite(ref[order])]
    head = ref[order[:p + 1]]
    gaps = head[:-1] - head[1:]
    ties = int((gaps == 0).sum())
    margin = float(gaps[gaps > 0].min()) if (gaps > 0).any() else np.inf
    return order[:p], ref[order[:p]], {"margin": margin, "ties": ties}
