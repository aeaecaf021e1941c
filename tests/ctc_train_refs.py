"""fp64 references for training the recognizer's output layer (``b2o_ctc_loss_grad``, ``b2o_rmsprop_step``).

* ``keep_mask``: the dropout mask of include/b2ocr.h, rebuilt bit for bit from the kernel's hash (splitmix64 of the seed,
  the step, the cached row, the step t and the feature c).
* ``dropped`` / ``drop``: the features after dropout, in the kernel's fp32 arithmetic (x * fp32(1 / (1 - rate)), or 0),
  from a cache and its rows or from features already gathered.
* ``loss_grad``: the Keras ``ctc_batch_cost`` loss of one crop, L = -log sum over alignments of prod_t q[t, path_t] with
  q = softmax(l) + 1e-7 and blank = K-1, and its gradient dL/dl, by the forward-backward algorithm in the log domain,
  in fp64.  Also the pieces the GPU test's bound needs: p, q, the posteriors gamma and D_t = sum_c gamma_c p_c / q_c.
* ``batch_grads``: (1/B) sum x^T g and (1/B) sum g over a batch.
* ``rmsprop``: one Keras RMSprop step with momentum 0, in fp64.
"""
import numpy as np

T, FEAT = 48, 256
MASK64 = (1 << 64) - 1


def mix64(z):
    """splitmix64's finaliser on uint64 numpy values (wrapping arithmetic)."""
    z = np.asarray(z, dtype=np.uint64)
    with np.errstate(over="ignore"):
        z = z + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def keep_mask(rows, rate, seed, step):
    """(B, 48, 256) bool: which features of cached rows ``rows`` survive Dropout(rate) at (seed, step)."""
    rows = np.asarray(rows, dtype=np.uint64)
    key0 = mix64(mix64(np.uint64(seed)) ^ np.uint64(step))
    t = np.arange(T, dtype=np.uint64)[:, None]
    c = np.arange(FEAT, dtype=np.uint64)[None, :]
    key = rows[:, None, None] * np.uint64(T * FEAT) + t * np.uint64(FEAT) + c
    h = mix64(key0 ^ key) >> np.uint64(40)
    thr = np.uint64(int(np.float64(np.float32(rate)) * 16777216.0))
    return h >= thr


def dropped(features, rows, rate, seed, step):
    """float32 (B, 48, 256): the features of ``rows`` (of an (n, 48, 256) fp16 array) as the kernel uses them."""
    return drop(np.asarray(features)[np.asarray(rows)], rows, rate, seed, step)


def drop(x, rows, rate, seed, step):
    """float32 (B, 48, 256): features x (B, 48, 256) of the dataset rows ``rows`` after the kernel's dropout."""
    x = np.asarray(x).astype(np.float32)
    rate = np.float32(rate)
    if rate == 0:
        return x
    scale = np.float32(1.0) / (np.float32(1.0) - rate)
    return np.where(keep_mask(rows, rate, seed, step), x * scale, np.float32(0.0)).astype(np.float32)


def logits(x, w, bias):
    """fp64 logits of (B, 48, 256) features."""
    return np.asarray(x, np.float64) @ np.asarray(w, np.float64) + np.asarray(bias, np.float64)


def _ext(labels, blank):
    ext = [blank]
    for c in labels:
        ext += [int(c), blank]
    ext = np.array(ext)
    skip = np.zeros(len(ext), bool)
    skip[2:] = (ext[2:] != blank) & (ext[2:] != ext[:-2])
    return ext, skip


def loss_grad(lg, labels):
    """One crop: (L, g, info) for (48, K) logits and a label sequence (non-blank labels, at least one).  g = dL/dl
    (48, K); info holds p, q, gamma (48, K: the posterior occupancy of each class), D (48,).  L = inf, g = 0 for a
    sequence that cannot be aligned."""
    lg = np.asarray(lg, np.float64)
    Tn, K = lg.shape
    blank = K - 1
    e = np.exp(lg - lg.max(-1, keepdims=True))
    p = e / e.sum(-1, keepdims=True)
    q = p + 1e-7
    lq = np.log(q)
    ext, skip = _ext(labels, blank)
    S = len(ext)
    la = np.full((Tn, S), -np.inf)
    la[0, 0] = lq[0, blank]
    la[0, 1] = lq[0, ext[1]]
    for t in range(1, Tn):
        a = la[t - 1].copy()
        a[1:] = np.logaddexp(a[1:], la[t - 1, :-1])
        a[2:] = np.where(skip[2:], np.logaddexp(a[2:], la[t - 1, :-2]), a[2:])
        la[t] = a + lq[t, ext]
    lb = np.full((Tn, S), -np.inf)                                 # beta_t: steps t+1 .. T-1, q_t not included
    lb[-1, S - 1] = lb[-1, S - 2] = 0.0
    for t in range(Tn - 2, -1, -1):
        n = lb[t + 1] + lq[t + 1, ext]
        b = n.copy()
        b[:-1] = np.logaddexp(b[:-1], n[1:])
        b[:-2] = np.where(skip[2:], np.logaddexp(b[:-2], n[2:]), b[:-2])
        lb[t] = b
    logp = np.logaddexp(la[-1, S - 1], la[-1, S - 2])
    if not np.isfinite(logp):
        return np.inf, np.zeros_like(lg), None
    occ = np.exp(la + lb - logp)                                   # (T, S) posterior of every state
    gamma = np.zeros((Tn, K))
    for s in range(S):
        gamma[:, ext[s]] += occ[:, s]
    D = (gamma * p / q).sum(-1)
    g = p * (D[:, None] - gamma / q)
    return -logp, g, {"p": p, "q": q, "gamma": gamma, "D": D}


def batch_grads(x, g):
    """(1/B) sum over crops and steps of x^T g, and of g: fp64 (256, K), (K,)."""
    x = np.asarray(x, np.float64)
    g = np.asarray(g, np.float64)
    b = x.shape[0]
    return np.einsum("btc,btk->ck", x, g, optimize=True) / b, g.sum((0, 1)) / b


def rmsprop(param, grad, acc, lr=1e-3, rho=0.9, eps=1e-7):
    """One Keras RMSprop step (momentum 0) in fp64: (new param, new acc)."""
    param, grad, acc = (np.asarray(a, np.float64) for a in (param, grad, acc))
    acc = rho * acc + (1 - rho) * grad * grad
    return param - lr * grad / (np.sqrt(acc) + eps), acc
