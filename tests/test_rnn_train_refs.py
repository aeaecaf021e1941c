"""The fp64 reference of the trainable recurrent head (tests/rnn_train_refs.py) checked on its own, no GPU:
* its differentiable LSTM equals ``stage_refs.lstm_emulated`` with the roundings on, and ``oracle.crnn.lstm`` with them off;
* autograd's gradients of all 14 tensors equal central differences of the loss;
* the hand-written backward (the one the GPU test runs on the device's activations) equals autograd, with and without
  dropout, and it follows the reference's go_backwards quirk: a model whose backward outputs are re-reversed into input
  order has different gradients, which the backward does not match;
* the per-step checker of the saved forward state accepts the rounding-emulating fp64 forward and rejects swapped gates,
  a cell state one step late, a backward direction's activations in input order and xw without its bias.
"""
import numpy as np
import torch

from tests import ctc_train_refs as TR
from tests import rnn_train_refs as RR
from tests import stage_refs as R


def _tensors(k, seed):
    rng = np.random.default_rng(seed)
    t = {}
    for layer in RR.LAYERS:
        t[layer + ".kernel"] = (rng.normal(size=(128, 512)) * 0.12).astype(np.float32)
        t[layer + ".recurrent_kernel"] = (rng.normal(size=(128, 512)) * 0.08).astype(np.float32)
        t[layer + ".bias"] = (rng.normal(size=512) * 0.3).astype(np.float32)
    t["fc_12.kernel"] = (rng.normal(size=(256, k)) * 0.3).astype(np.float32)
    t["fc_12.bias"] = (rng.normal(size=k) * 0.3).astype(np.float32)
    return t


def _x(b, seed):
    return np.maximum(np.random.default_rng(seed).normal(size=(b, 50, 128)), 0).astype(np.float16).astype(np.float64)


def test_lstm_matches_emulation_and_oracle():
    from oracle import crnn
    t = _tensors(5, 1)
    x = _x(2, 2)
    xw = x @ R.f16(t["lstm_10_back.kernel"]) + t["lstm_10_back.bias"]
    ours = RR.lstm(torch.from_numpy(xw), R.f16(torch.from_numpy(t["lstm_10_back.recurrent_kernel"].astype(np.float64))),
                   True, True).numpy()
    assert np.array_equal(ours, R.lstm_emulated(xw, t["lstm_10_back.recurrent_kernel"], go_backwards=True))
    wt = {k: torch.from_numpy(v) for k, v in t.items()}
    params = {k: torch.from_numpy(v.astype(np.float64)) for k, v in t.items()}
    l2, l1, _, _ = RR.forward(params, x, rounding=False, return_all=True)
    xf = torch.from_numpy(x).float()
    o1 = crnn.lstm(wt, xf, "lstm_10") + crnn.lstm(wt, xf, "lstm_10_back", go_backwards=True)
    o2 = torch.cat([crnn.lstm(wt, o1, "lstm_11"), crnn.lstm(wt, o1, "lstm_11_back", go_backwards=True)], -1)
    assert np.abs(l1.numpy() - o1.double().numpy()).max() < 1e-5
    assert np.abs(l2.numpy() - o2.double().numpy()).max() < 1e-5


def test_autograd_matches_central_differences():
    k = 5
    t = {n: v.astype(np.float64) for n, v in _tensors(k, 3).items()}
    x = _x(2, 4)
    targets = [[0, 1, 1, 2], [3]]
    rows = [7, 2]
    _, grads = RR.head_losses(t, x, targets, rows, dropout=0.25, seed=5, step=1, rounding=False)
    rng = np.random.default_rng(6)
    for name, shape in RR.tensor_names(k):
        for _ in range(2):
            idx = tuple(int(rng.integers(0, s)) for s in shape)
            h = 1e-5
            vals = []
            for sgn in (1, -1):
                tt = dict(t)
                tt[name] = t[name].copy()
                tt[name][idx] += sgn * h
                vals.append(RR.head_losses(tt, x, targets, rows, 0.25, 5, 1, rounding=False)[0].mean())
            fd = (vals[0] - vals[1]) / (2 * h)
            assert abs(fd - grads[name][idx]) <= 1e-6 * (1 + abs(fd)), (name, idx, fd, grads[name][idx])


def _manual(t, x, targets, rows, dropout, seed, step, rereverse=False):
    """backward() on the fp64 forward's own activations (no rounding)."""
    acts, h1, l1, l2 = RR.forward_acts(t, x)
    k = t["fc_12.bias"].shape[0]
    xk = l2[:, 2:]
    if dropout > 0:
        xk = xk * TR.keep_mask(rows, dropout, seed, step) * float(np.float32(1) / (np.float32(1) - np.float32(dropout)))
    lg = xk @ t["fc_12.kernel"] + t["fc_12.bias"]
    g = np.stack([TR.loss_grad(lg[i], targets[i])[1] for i in range(len(targets))])
    assert g.shape[-1] == k
    return RR.backward(x, acts, h1, l1, l2, g, t, rows, dropout, seed, step, rounding=False)[0]


def _rereversed_grads(t, x, targets):
    """autograd of a model whose go_backwards outputs are flipped back into input order (not the reference's)."""
    k = t["fc_12.bias"].shape[0]
    p = {n: torch.tensor(t[n], requires_grad=True) for n, _ in RR.tensor_names(k)}
    xt = torch.from_numpy(x)

    def run(layer, inp, back):
        out = RR.lstm(inp @ p[layer + ".kernel"] + p[layer + ".bias"], p[layer + ".recurrent_kernel"], back, False)
        return torch.flip(out, [1]) if back else out
    l1 = run("lstm_10", xt, False) + run("lstm_10_back", xt, True)
    l2 = torch.cat([run("lstm_11", l1, False), run("lstm_11_back", l1, True)], -1)[:, 2:]
    lg = l2 @ p["fc_12.kernel"] + p["fc_12.bias"]
    loss = torch.stack([RR._CTC.apply(lg[i], targets[i]) for i in range(len(targets))]).mean()
    loss.backward()
    return {n: v.grad.numpy() for n, v in p.items()}


def test_manual_backward_matches_autograd_and_the_quirk():
    k = 6
    t = {n: v.astype(np.float64) for n, v in _tensors(k, 8).items()}
    x = _x(3, 9)
    targets = [[0, 0, 1], [4], [1, 2, 3, 4, 0]]
    rows = [0, 5, 2]
    for dropout in (0.0, 0.25):
        _, auto = RR.head_losses(t, x, targets, rows, dropout, 3, 2, rounding=False)
        man = _manual(t, x, targets, rows, dropout, 3, 2)
        for name in auto:
            scale = np.abs(auto[name]).max()
            assert np.abs(man[name] - auto[name]).max() <= 1e-10 * scale, (name, dropout)
    wrong = _rereversed_grads(t, x, targets)
    _, auto = RR.head_losses(t, x, targets, rows, 0.0, 0, 0, rounding=False)
    for name in ("lstm_10_back.kernel", "lstm_11_back.recurrent_kernel", "lstm_10.kernel"):
        rel = np.abs(wrong[name] - auto[name]).max() / np.abs(auto[name]).max()
        assert rel > 1e-2, (name, rel)


def _state_worst(x, t, st):
    return max(RR.state_ratios(x, t, st["xw"], st["acts"], st["h1"], st["l1"], st["l2"]).values())


def test_state_checker_accepts_the_emulation_and_rejects_mutations():
    """The per-step check of the device's saved forward state (run on the GPU by tests/test_gpu_fit_recurrent.py) passes
    the fp64 forward with the device's roundings, and fails each way a saving kernel could be wrong."""
    k = 5
    t = _tensors(k, 11)
    x = _x(3, 12)
    x[1] = 0                                                      # a crop whose row lies outside the cache
    st = RR.forward_state(t, x, rounding=True)
    assert np.array_equal(st["xw"][0, 1], np.broadcast_to(t["lstm_10.bias"].astype(np.float64), (50, 512)))
    ok = RR.state_ratios(x, t, st["xw"], st["acts"], st["h1"], st["l1"], st["l2"])
    assert max(ok.values()) <= 1.0, ok
    swapped = st["acts"].copy()                                   # i and f in each other's slot
    swapped[:, :, :, [0, 1]] = swapped[:, :, :, [1, 0]]
    shifted = st["acts"].copy()                                   # c of the step before (the state before the update)
    shifted[:, :, 1:, 4] = st["acts"][:, :, :-1, 4]
    shifted[:, :, 0, 4] = 0
    input_order = st["acts"].copy()                               # a backward direction's activations in input order
    input_order[3] = st["acts"][3][:, ::-1]
    no_bias = st["xw"].copy()
    no_bias[2] -= t["lstm_11.bias"].astype(np.float64)
    for name, mutated in (("i/f swapped", dict(st, acts=swapped)), ("c one step late", dict(st, acts=shifted)),
                          ("acts in input order", dict(st, acts=input_order)), ("xw without bias", dict(st, xw=no_bias))):
        assert _state_worst(x, t, mutated) > 1.0, name


def test_flat_layout():
    k = 7
    t = _tensors(k, 1)
    v = RR.flat(t, k)
    assert v.size == 526_336 + 257 * k
    back = RR.unflat(v, k)
    assert all(np.array_equal(back[n], t[n]) for n, _ in RR.tensor_names(k))
    assert np.array_equal(v[131_584:131_584 + 65_536].reshape(128, 512), t["lstm_10_back.kernel"])
