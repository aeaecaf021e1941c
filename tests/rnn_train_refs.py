"""fp64 references for fine-tuning the recognizer's recurrent head (``b2o_rnn_loss_grad``).

* ``head_losses``: the trainable head -- lstm_10 / lstm_10_back on the fc_9 features, l1 = hf + hb, lstm_11 /
  lstm_11_back on l1, l2 = [h11f, h11b], steps 2..49, Dropout (``ctc_train_refs.dropped``'s mask), fc_12 and the Keras
  ``ctc_batch_cost`` of ``ctc_train_refs.loss_grad`` -- in torch fp64, so autograd gives the gradient of every tensor.
  ``rounding`` switches on the device's documented roundings (W and U to fp16, h and l1 to fp16), each taken as the
  identity by the gradient; the LSTM recurrence is ``stage_refs.lstm_emulated``'s, go_backwards outputs kept in
  processing order (recognition.py:298-319).
* ``backward``: the same gradients by hand, from given activations (the device's own, read from its workspace), with a
  running first-order bound of the device's fp32 arithmetic next to every value (see tests/test_gpu_fit_recurrent.py).
"""
import numpy as np
import torch

from tests import ctc_train_refs as TR
from tests import stage_refs as R

LAYERS = ("lstm_10", "lstm_10_back", "lstm_11", "lstm_11_back")
STEPS, UNITS, DISCARD = 50, 128, 2
U32 = 2.0 ** -24


def gamma(n):
    return n * U32 / (1 - n * U32)


def tensor_names(k):
    """The 14 trained tensors in the order of the flat parameter vector, with their shapes."""
    out = []
    for layer in LAYERS:
        out += [(f"{layer}.kernel", (128, 512)), (f"{layer}.recurrent_kernel", (128, 512)), (f"{layer}.bias", (512,))]
    return out + [("fc_12.kernel", (256, k)), ("fc_12.bias", (k,))]


def flat(tensors, k):
    return np.concatenate([np.asarray(tensors[n], np.float32).reshape(-1) for n, _ in tensor_names(k)])


def unflat(vec, k):
    out, at = {}, 0
    for n, shape in tensor_names(k):
        size = int(np.prod(shape))
        out[n] = np.asarray(vec[at:at + size]).reshape(shape)
        at += size
    return out


def _st16(v, on):
    """fp16 rounding whose gradient is the identity (straight-through)."""
    return v + (R.f16(v) - v).detach() if on else v


def lstm(xw, u, go_backwards, rounding):
    """``stage_refs.lstm_emulated`` in differentiable torch: xw (B,T,512) = x W + b, u (128,512); outputs in processing
    order, h rounded to fp16 between steps when ``rounding``."""
    if go_backwards:
        xw = torch.flip(xw, [1])
    b, t, _ = xw.shape
    h = torch.zeros(b, UNITS, dtype=torch.float64)
    c = torch.zeros(b, UNITS, dtype=torch.float64)
    outs = []
    for s in range(t):
        zi, zf, zc, zo = torch.split(xw[:, s] + h @ u, UNITS, dim=1)
        c = torch.sigmoid(zf) * c + torch.sigmoid(zi) * torch.tanh(zc)
        h = _st16(torch.sigmoid(zo) * torch.tanh(c), rounding)
        outs.append(h)
    return torch.stack(outs, 1)


class _CTC(torch.autograd.Function):
    """Keras ctc_batch_cost of one crop on (48, K) logits, its gradient from ``ctc_train_refs.loss_grad``."""

    @staticmethod
    def forward(ctx, lg, labels):
        L, g, _ = TR.loss_grad(lg.detach().numpy(), labels)
        ctx.save_for_backward(torch.from_numpy(g))
        return torch.tensor(L, dtype=torch.float64)

    @staticmethod
    def backward(ctx, grad_out):
        (g,) = ctx.saved_tensors
        return grad_out * g, None


def forward(params, x, rounding=True, return_all=False):
    """params: name -> torch fp64 tensor; x (B,50,128) fc_9 features.  Returns l2 (B,50,256) (and l1, hf, hb)."""
    def w_of(layer):
        return (_st16(params[layer + ".kernel"], rounding), _st16(params[layer + ".recurrent_kernel"], rounding),
                params[layer + ".bias"])
    x = torch.as_tensor(np.asarray(x, np.float64))
    hs = []
    for layer, back in (("lstm_10", False), ("lstm_10_back", True)):
        w, u, b = w_of(layer)
        hs.append(lstm(x @ w + b, u, back, rounding))
    l1 = _st16(hs[0] + hs[1], rounding)
    outs = []
    for layer, back in (("lstm_11", False), ("lstm_11_back", True)):
        w, u, b = w_of(layer)
        outs.append(lstm(l1 @ w + b, u, back, rounding))
    l2 = torch.cat(outs, -1)
    return (l2, l1, hs[0], hs[1]) if return_all else l2


def head_losses(tensors, x, targets, rows, dropout=0.0, seed=0, step=0, rounding=True):
    """(losses (B,) fp64 numpy, grads name -> fp64 numpy of the batch mean loss).  x: (B,50,128) fc_9 rows of the batch,
    rows: their dataset rows (the dropout key), targets: label lists."""
    k = np.shape(tensors["fc_12.bias"])[0]
    params = {n: torch.tensor(np.asarray(tensors[n], np.float64), requires_grad=True) for n, _ in tensor_names(k)}
    l2 = forward(params, x, rounding)[:, DISCARD:]
    if dropout > 0:
        mask = torch.from_numpy(TR.keep_mask(rows, dropout, seed, step))
        scale = float(np.float32(1.0) / (np.float32(1.0) - np.float32(dropout)))
        l2 = torch.where(mask, l2 * scale, torch.zeros_like(l2))
    lg = l2 @ params["fc_12.kernel"] + params["fc_12.bias"]
    losses = torch.stack([_CTC.apply(lg[i], list(targets[i])) for i in range(len(targets))])
    finite = torch.where(torch.isfinite(losses), losses, torch.zeros_like(losses))
    (finite.sum() / len(targets)).backward()
    return losses.detach().numpy(), {n: p.grad.numpy() for n, p in params.items()}


def bptt(acts, u, dh_out, e_out=None):
    """Backpropagation through one LSTM direction from its activations, in processing order, as bptt_kernel runs it.
    acts (B,50,5,128) = i, f, g, o, c; u (128,512); dh_out (B,50,128) = dL/dh from above (e_out its bound).
    Returns dz (B,50,512) and its running fp32 error bound."""
    b = acts.shape[0]
    acts = np.asarray(acts, np.float64)
    u = np.asarray(u, np.float64)
    ua = np.abs(u)
    e_out = np.zeros_like(dh_out) if e_out is None else e_out
    dz = np.zeros((b, STEPS, 512))
    ez = np.zeros((b, STEPS, 512))
    dcn = np.zeros((b, UNITS))
    edcn = np.zeros((b, UNITS))
    for s in range(STEPS - 1, -1, -1):
        i, f, g, o, c = (acts[:, s, j] for j in range(5))
        cp = acts[:, s - 1, 4] if s > 0 else np.zeros_like(c)
        if s < STEPS - 1:
            rec = dz[:, s + 1] @ u.T
            e_rec = ez[:, s + 1] @ ua.T + gamma(130) * (np.abs(dz[:, s + 1]) @ ua.T)
        else:
            rec = e_rec = np.zeros_like(c)
        dh = dh_out[:, s] + rec
        e_dh = e_out[:, s] + e_rec + U32 * np.abs(dh)
        tc = np.tanh(c)
        e_tc = 4 * U32 * np.abs(tc)                                    # tanhf: at most 2 ulp
        t1 = 1 - tc * tc
        t2 = dh * o
        dc = dcn + t2 * t1
        e_dc = (edcn + (e_dh * np.abs(o) + U32 * np.abs(t2)) * np.abs(t1)
                + np.abs(t2) * (2 * np.abs(tc) * e_tc + U32 * np.abs(t1)) + U32 * np.abs(dc))
        zo = dh * tc * o * (1 - o)
        zi = dc * g * i * (1 - i)
        zf = dc * cp * f * (1 - f)
        zg = dc * i * (1 - g * g)
        dz[:, s] = np.concatenate([zi, zf, zg, zo], 1)
        ez[:, s] = np.concatenate([
            e_dc * np.abs(g * i * (1 - i)) + 4 * U32 * np.abs(zi),
            e_dc * np.abs(cp * f * (1 - f)) + 4 * U32 * np.abs(zf),
            e_dc * np.abs(i * (1 - g * g)) + 3 * U32 * np.abs(zg) + 2 * U32 * np.abs(dc * i * g * g),
            (e_dh * np.abs(tc) + np.abs(dh) * e_tc) * np.abs(o * (1 - o)) + 4 * U32 * np.abs(zo)], 1)
        dcn = dc * f
        edcn = e_dc * np.abs(f) + U32 * np.abs(dcn)
    return dz, ez


def _wsum(a, dz, ez):
    """sum over (b, s) of a^T dz, and the bound of the device's chunked fp32 sum divided by B."""
    n = a.shape[0] * a.shape[1]
    aa = np.abs(a)
    val = np.einsum("bsm,bsn->mn", a, dz)
    err = gamma(n + 1) * np.einsum("bsm,bsn->mn", aa, np.abs(dz)) + np.einsum("bsm,bsn->mn", aa, ez)
    return val, err


def backward(x, acts, h1, l1, l2, g, tensors, rows, dropout=0.0, seed=0, step=0, rounding=True):
    """The gradients of the batch mean loss by hand, from given activations: x (B,50,128) fc_9 rows, acts
    (4,B,50,5,128), h1 (2,B,50,128) = hf, hb (processing order), l1 (B,50,128), l2 (B,50,256), g (B,48,K) =
    dL_b/dlogits.  With ``rounding`` W and U are taken fp16-rounded, as the device uses them.  Returns (grads, bounds), name -> fp64 arrays (batch means)."""
    x, l1, l2, g = (np.asarray(a, np.float64) for a in (x, l1, l2, g))
    h1 = np.asarray(h1, np.float64)
    b = x.shape[0]
    k = g.shape[-1]
    wf = np.asarray(tensors["fc_12.kernel"], np.float64)
    rnd = R.f16 if rounding else (lambda a: np.asarray(a, np.float64))
    W = {n: rnd(tensors[n + ".kernel"]) for n in LAYERS}
    U = {n: rnd(tensors[n + ".recurrent_kernel"]) for n in LAYERS}
    # dL/dl2: mask * scale * g w^T on the kept steps
    ms = np.ones((b, 48, 256))
    if dropout > 0:
        scale = float(np.float32(1.0) / (np.float32(1.0) - np.float32(dropout)))
        ms = TR.keep_mask(rows, dropout, seed, step) * scale
    dl2 = np.zeros((b, STEPS, 256))
    e_dl2 = np.zeros_like(dl2)
    dl2[:, DISCARD:] = ms * (g @ wf.T)
    e_dl2[:, DISCARD:] = ms * gamma(k) * (np.abs(g) @ np.abs(wf).T) + U32 * np.abs(dl2[:, DISCARD:])
    dz, ez = {}, {}
    for j, n in enumerate(LAYERS[2:]):
        dz[n], ez[n] = bptt(acts[2 + j], U[n], dl2[..., 128 * j:128 * (j + 1)], e_dl2[..., 128 * j:128 * (j + 1)])
    # dL/dl1[t] = dz_11[t] W_11^T + dz_11b[49 - t] W_11b^T
    zb, ezb = dz["lstm_11_back"][:, ::-1], ez["lstm_11_back"][:, ::-1]
    wa, wb = np.abs(W["lstm_11"]), np.abs(W["lstm_11_back"])
    dl1 = dz["lstm_11"] @ W["lstm_11"].T + zb @ W["lstm_11_back"].T
    e_dl1 = (gamma(1024) * (np.abs(dz["lstm_11"]) @ wa.T + np.abs(zb) @ wb.T)
             + ez["lstm_11"] @ wa.T + ezb @ wb.T)
    for j, n in enumerate(LAYERS[:2]):
        dz[n], ez[n] = bptt(acts[j], U[n], dl1, e_dl1)
    grads, bounds = {}, {}
    for j, n in enumerate(LAYERS):
        xin = x if j < 2 else l1
        if j % 2:
            xin = xin[:, ::-1]                                         # going backwards, step s read input 49 - s
        h = h1[j] if j < 2 else l2[..., 128 * (j - 2):128 * (j - 1)]
        hprev = np.concatenate([np.zeros_like(h[:, :1]), h[:, :-1]], 1)
        for part, a in (("kernel", xin), ("recurrent_kernel", hprev), ("bias", np.ones((b, STEPS, 1)))):
            v, e = _wsum(a, dz[n], ez[n])
            v = v[0] if part == "bias" else v
            e = e[0] if part == "bias" else e
            grads[f"{n}.{part}"] = v / b
            bounds[f"{n}.{part}"] = e / b + U32 * np.abs(v / b)
    xk = l2[:, DISCARD:] * ms
    n = b * 48
    grads["fc_12.kernel"] = np.einsum("btc,btk->ck", xk, g) / b
    bounds["fc_12.kernel"] = gamma(n + 1) * np.einsum("btc,btk->ck", np.abs(xk), np.abs(g)) / b + \
        U32 * np.abs(grads["fc_12.kernel"])
    grads["fc_12.bias"] = g.sum((0, 1)) / b
    bounds["fc_12.bias"] = gamma(n + 1) * np.abs(g).sum((0, 1)) / b + U32 * np.abs(grads["fc_12.bias"])
    return grads, bounds


def forward_acts(tensors, x):
    """fp64 forward without rounding that also returns what ``backward`` needs: (acts (4,B,50,5,128), h1 (2,B,50,128),
    l1 (B,50,128), l2 (B,50,256)), in processing order."""
    x = np.asarray(x, np.float64)

    def run(layer, inp, back):
        w = np.asarray(tensors[layer + ".kernel"], np.float64)
        u = np.asarray(tensors[layer + ".recurrent_kernel"], np.float64)
        xw = inp @ w + np.asarray(tensors[layer + ".bias"], np.float64)
        if back:
            xw = xw[:, ::-1]
        b = xw.shape[0]
        h = np.zeros((b, UNITS))
        c = np.zeros((b, UNITS))
        acts, hs = np.zeros((b, STEPS, 5, UNITS)), np.zeros((b, STEPS, UNITS))
        sig = lambda v: 1 / (1 + np.exp(-v))                                         # noqa: E731
        for s in range(STEPS):
            zi, zf, zc, zo = np.split(xw[:, s] + h @ u, 4, 1)
            i, f, g, o = sig(zi), sig(zf), np.tanh(zc), sig(zo)
            c = f * c + i * g
            h = o * np.tanh(c)
            acts[:, s] = np.stack([i, f, g, o, c], 1)
            hs[:, s] = h
        return acts, hs
    a0, hf = run("lstm_10", x, False)
    a1, hb = run("lstm_10_back", x, True)
    l1 = hf + hb
    a2, h2f = run("lstm_11", l1, False)
    a3, h2b = run("lstm_11_back", l1, True)
    return np.stack([a0, a1, a2, a3]), np.stack([hf, hb]), l1, np.concatenate([h2f, h2b], -1)
