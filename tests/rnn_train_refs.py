"""fp64 references for fine-tuning the recognizer's recurrent head (``b2o_rnn_loss_grad``).

* ``head_losses``: the trainable head -- lstm_10 / lstm_10_back on the fc_9 features, l1 = hf + hb, lstm_11 /
  lstm_11_back on l1, l2 = [h11f, h11b], steps 2..49, Dropout (``ctc_train_refs.dropped``'s mask), fc_12 and the Keras
  ``ctc_batch_cost`` of ``ctc_train_refs.loss_grad`` -- in torch fp64, so autograd gives the gradient of every tensor.
  ``rounding`` switches on the device's documented roundings (W and U to fp16, h and l1 to fp16), each taken as the
  identity by the gradient; the LSTM recurrence is ``stage_refs.lstm_emulated``'s, go_backwards outputs kept in
  processing order (recognition.py:298-319).
* ``backward``: the same gradients by hand, from given activations (the device's own, read from its workspace), with a
  running first-order bound of the device's fp32 arithmetic next to every value (see tests/test_gpu_fit_recurrent.py).
* ``forward_state``: the fp64 forward with every value the device saves for the backward (xw, the gate activations
  and c, h), rounding emulated or not; ``forward_acts`` its unrounded activations.
* ``state_ratios``: checks the device's saved forward state step by step, each step on the device's own previous
  state, so that the ``backward`` above is known to run on the activations of the right step, gate and direction.
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
    val = np.einsum("bsm,bsn->mn", a, dz, optimize=True)
    err = (gamma(n + 1) * np.einsum("bsm,bsn->mn", aa, np.abs(dz), optimize=True)
           + np.einsum("bsm,bsn->mn", aa, ez, optimize=True))
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
    grads["fc_12.kernel"] = np.einsum("btc,btk->ck", xk, g, optimize=True) / b
    bounds["fc_12.kernel"] = gamma(n + 1) * np.einsum("btc,btk->ck", np.abs(xk), np.abs(g), optimize=True) / b + \
        U32 * np.abs(grads["fc_12.kernel"])
    grads["fc_12.bias"] = g.sum((0, 1)) / b
    bounds["fc_12.bias"] = gamma(n + 1) * np.abs(g).sum((0, 1)) / b + U32 * np.abs(grads["fc_12.bias"])
    return grads, bounds


def forward_acts(tensors, x):
    """fp64 forward without rounding that also returns what ``backward`` needs: (acts (4,B,50,5,128), h1 (2,B,50,128),
    l1 (B,50,128), l2 (B,50,256)), in processing order."""
    st = forward_state(tensors, x, rounding=False)
    return st["acts"], st["h1"], st["l1"], st["l2"]


def _sig(v):
    return 1 / (1 + np.exp(-v))


def forward_state(tensors, x, rounding=True):
    """The fp64 forward with every value ``b2o_rnn_loss_grad`` keeps in its workspace, as a dict: xw (4,B,50,512) =
    x W + b per direction in input order (row b*50 + t), acts (4,B,50,5,128) = i, f, g, o, c, h1 (2,B,50,128) = hf, hb,
    l1 (B,50,128), l2 (B,50,256), all but xw in processing order.  ``rounding``: W and U rounded to fp16, h and l1
    rounded to fp16, as the device rounds them."""
    x = np.asarray(x, np.float64)
    rnd = R.f16 if rounding else (lambda a: np.asarray(a, np.float64))

    def run(layer, inp, back):
        w = rnd(tensors[layer + ".kernel"])
        u = rnd(tensors[layer + ".recurrent_kernel"])
        xw = inp @ w + np.asarray(tensors[layer + ".bias"], np.float64)
        xs = xw[:, ::-1] if back else xw
        b = xw.shape[0]
        h = np.zeros((b, UNITS))
        c = np.zeros((b, UNITS))
        acts, hs = np.zeros((b, STEPS, 5, UNITS)), np.zeros((b, STEPS, UNITS))
        for s in range(STEPS):
            zi, zf, zc, zo = np.split(xs[:, s] + h @ u, 4, 1)
            i, f, g, o = _sig(zi), _sig(zf), np.tanh(zc), _sig(zo)
            c = f * c + i * g
            h = rnd(o * np.tanh(c))
            acts[:, s] = np.stack([i, f, g, o, c], 1)
            hs[:, s] = h
        return xw, acts, hs
    w0, a0, hf = run("lstm_10", x, False)
    w1, a1, hb = run("lstm_10_back", x, True)
    l1 = rnd(hf + hb)
    w2, a2, h2f = run("lstm_11", l1, False)
    w3, a3, h2b = run("lstm_11_back", l1, True)
    return {"xw": np.stack([w0, w1, w2, w3]), "acts": np.stack([a0, a1, a2, a3]), "h1": np.stack([hf, hb]), "l1": l1,
            "l2": np.concatenate([h2f, h2b], -1)}


# 1 / (1 + expf(-z)): expf's 2 ulp (4u relative) pass through the addition with weight e / (1 + e) < 1, then the
# addition and the division round once each.  tanhf: 2 ulp.
SIG_REL = 6 * U32
TANH_REL = 4 * U32


def _slope_bound(deriv, z, ez):
    """max of a derivative that falls with |z| (sigmoid', tanh') over [z - ez, z + ez]."""
    return deriv(np.maximum(np.abs(z) - ez, 0.0))


def state_ratios(x, tensors, xw, acts, h1, l1, l2):
    """Worst |device - fp64| / bound of the training forward's saved state, each value judged on the device's own
    inputs of its step, so that no bound grows along the 50 steps.  x (B,50,128): the fc_9 rows the crops read (zeros
    for a row outside the cache); xw, acts, h1, l1, l2: the workspace slots of ``b2o_rnn_loss_grad`` (layouts as in
    ``forward_state``).  Returns {"xw", "i", "f", "g", "o", "c", "h"} -> worst ratio over the four directions.
    * xw[d] = x W16 + b (x the fc_9 rows for layer 1, the device's own l1 for layer 2): the MMA's fp32 sum of exact
      fp16 products within stage_refs.gamma(128) |x| |W16|, then the bias in one rounding, u |xw|.
    * z at processing step s = xw[d][t(s)] + h_{s-1} U16 (t(s) = s, or 49 - s going backwards; h_{s-1} the device's
      fp16 h, 0 at s = 0): the MMA sum that starts from xw, within ez = stage_refs.gamma(129) (|xw| + |h| |U16|).
    * i, f, o = sigmoid(z), g = tanh(z): the largest slope over z +- ez times ez, plus SIG_REL / TANH_REL relative.
    * c = f c' + i g with the device's c' (acts at s - 1): the gate errors times their weights plus 2u (|f c'| + |i g|).
    * h: the stored fp16 h = fp16(o tanh(c)) of the device's own o and c: half an fp16 ulp plus 5u |o tanh c|.
    Each bound is taken 1.01 times (second-order terms) plus 1e-30 absolute."""
    x, xw, acts, h1, l1, l2 = (np.asarray(a, np.float64) for a in (x, xw, acts, h1, l1, l2))
    out = dict.fromkeys(("xw", "i", "f", "g", "o", "c", "h"), 0.0)

    def worst(name, dev, ref, bound):
        out[name] = max(out[name], float((np.abs(dev - ref) / (1.01 * bound + 1e-30)).max()))
    dsig = lambda v: _sig(v) * (1 - _sig(v))                                            # noqa: E731
    dtanh = lambda v: 1 - np.tanh(v) ** 2                                               # noqa: E731
    for d, layer in enumerate(LAYERS):
        w16, u16 = R.f16(tensors[layer + ".kernel"]), R.f16(tensors[layer + ".recurrent_kernel"])
        inp = x if d < 2 else l1
        ref = inp @ w16 + np.asarray(tensors[layer + ".bias"], np.float64)
        worst("xw", xw[d], ref, R.gamma(128) * (np.abs(inp) @ np.abs(w16)) + U32 * np.abs(ref))
        h = h1[d] if d < 2 else l2[..., 128 * (d - 2):128 * (d - 1)]
        hprev = np.concatenate([np.zeros_like(h[:, :1]), h[:, :-1]], 1)
        xs = xw[d][:, ::-1] if d % 2 else xw[d]
        z = xs + hprev @ u16
        ez = R.gamma(129) * (np.abs(xs) + np.abs(hprev) @ np.abs(u16))
        zi, zf, zg, zo = (z[..., 128 * j:128 * (j + 1)] for j in range(4))
        ei, ef, eg, eo = (ez[..., 128 * j:128 * (j + 1)] for j in range(4))
        a = acts[d]
        gates = {}
        for j, (name, zz, ee) in enumerate((("i", zi, ei), ("f", zf, ef), ("g", zg, eg), ("o", zo, eo))):
            if name == "g":
                val = np.tanh(zz)
                err = _slope_bound(dtanh, zz, ee) * ee + TANH_REL * np.abs(val)
            else:
                val = _sig(zz)
                err = _slope_bound(dsig, zz, ee) * ee + SIG_REL * val
            gates[name] = (val, err)
            worst(name, a[:, :, j], val, err)
        (i, e_i), (f, e_f), (g, e_g) = gates["i"], gates["f"], gates["g"]
        cp = np.concatenate([np.zeros_like(a[:, :1, 4]), a[:, :-1, 4]], 1)
        c = f * cp + i * g
        worst("c", a[:, :, 4], c, np.abs(cp) * e_f + np.abs(g) * e_i + np.abs(i) * e_g
              + 2 * U32 * (np.abs(f * cp) + np.abs(i * g)))
        p = a[:, :, 3] * np.tanh(a[:, :, 4])
        worst("h", h, p, 0.5 * R.ulp16(h) + 5 * U32 * np.abs(p))
    return out
