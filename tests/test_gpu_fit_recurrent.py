"""Fine-tuning the recognizer's recurrent head on the GPU (``b2o_crnn_sequence_features``, ``b2o_rnn_loss_grad``,
``Recognizer.fit_recurrent``) against the fp64 references of tests/rnn_train_refs.py.

Bounds.  u = 2^-24, gamma(n) = n u / (1 - n u).
* Sequence features: bit for bit the "fc_9" tap of a full forward (the same kernels stop earlier), on the trained
  recognizer and on the stn=False and color=True variants.
* Training forward, dropout 0: l1 and l2 within LSTM_TIGHT = 2^-9 of the fp16-emulating fp64 LSTM fed x W + b with the
  fp16-rounded W (tests/test_gpu_crnn_stages.py derives it for the inference LSTM, whose arithmetic this is), and within
  LSTM_LOOSE = 2^-7 of ``oracle.crnn.lstm``.  Loss against fit_top's loss on the inference features of the same crops: the
  CTC loss is 2-Lipschitz per step in the max norm of the logits (g_t = p (D - r) with sum_k p_k D <= 1 and
  sum_k p_k r_k = sum_k gamma_k p_k / q_k <= 1), and each logit moves by at most 2^-9 sum_c |w_ck| when l2 does, so
  |L_train - L_fit_top| <= 2 sum_t max_k (2^-9 sum_c |w_ck| + 2 gamma(257) (sum_c |l2_c w_ck| + |b_k|)) + 2 tau_L, with
  tau_L = 1.01 (eps + u) + u |L| the CTC kernel's own bound (tests/test_gpu_fit_top.py), eps <= 48 (3u + delta_t).
* Gradients, teacher-forced: the reference backward (``rnn_train_refs.backward``) runs on the device's own activations
  (acts, hf / hb, l1, l2 and g = dL/dlogits, read from their documented workspace slots), so only the backward
  arithmetic is judged.  It carries a first-order running bound through every fp32 operation of the device: each
  rounding u |result|; the recurrent product U dz and the other dot products gamma(n) sum |terms| (n = 130 for the
  quarter chains plus two shuffle additions, K for dL/dl2, 1024 for dL/dl1, B * 50 + 1 for the chunked weight sums and
  their ordered second pass); tanhf 2 ulp = 4u |tanh c|; the errors of the inputs propagated with the absolute partial
  derivatives.  The test allows 1.01 times that bound (second-order terms) plus 1e-30 absolute.
  They run at b = 11 (LSTM CTAs of 8 and 3 crops), 8 (one full CTA), 16 (one split-K chunk), 17 (a one-crop second
  chunk), 64 and 256 (4 and 16 chunks: the batch sizes training runs at), each case asserting its chunk count as read off
  the workspace size the library reports.
* Saved forward state (what the teacher-forced check trusts): ``rnn_train_refs.state_ratios`` judges xw, the gates, c and
  h of every direction and processing step on the device's own inputs of that step (its docstring derives the bounds),
  at b = 1, 17 and 64 with a permuted index and a row outside the cache; acts, hf / hb, l1 and l2 are bit-identical over
  loss-only and gradient calls, with and without dropout.
* fc_12's gradient, the loss and g of b2o_rnn_loss_grad equal b2o_ctc_loss_grad's on the device's own l2 bit for bit.
* The whole chain against autograd (``rnn_train_refs.head_losses`` with the roundings emulated, the fp64 forward rather
  than the device's activations): no rigorous bound exists, because an fp16 rounding of h can fall the other way in
  fp32; relative Frobenius error per tensor <= AUTOGRAD_TOL = 2^-6.
* Dropout keys past 2^31 (rows 174,763 and 200,003 of a 200,004-row cache): dL/dl2 is 0 exactly where the mask drops.
* One crop whose text cannot be aligned (25 copies of one letter need 49 steps) has loss +inf and adds nothing: the
  gradient times b equals the one of the other crops times b - 1 within the same kind of bound (checked to 1e-5 relative).
* ``fit_recurrent`` is restated call by call through the C ABI and must match it bit for bit.
The worst ratio of each check is printed.

End to end, on the decisive Hershey recognizer with lstm_11 and lstm_11_back re-drawn as Keras initialises them (fc_12
kept), with fit_top's 4096 training and 1024 held-out crops, 8 epochs at learning rate 1e-3, batch 64, seed 3.  Measured
once on an H100 80GB HBM3 (700 W): exact reads 0.0000 before, 0.9932 after fit_recurrent (1.6 s), 0.8740 after fit_top
from the same start with the same data, epochs and seed; the trained model reads 0.9941.  The test asks for at least the
trained model's rate minus MARGIN = 0.01 and strictly more than fit_top.  One epoch of fit_recurrent on the trained model
took it from 0.9941 to 0.9951.

Measured on an H100 80GB HBM3 (700 W).  Worst teacher-forced gradient ratios, the largest on fc_12: 0.050 of the bound
(b = 11, K = 1024), 0.017 (b = 17, K = 2), 0.0096 (b = 64, K = 1024), 0.00042 (b = 256, K = 38).  Saved state, worst
over b = 1, 17, 64: xw 0.015, i 0.31, f 0.32, g 0.11, o 0.31, c 0.050 and h 0.99 of their bounds (h's bound is mostly
the half fp16 ulp its rounding may take).  Against autograd: 1.1e-5 relative (fc_12.kernel), the losses 2.2e-6.  The
batch-size, saved-state, fc_12, autograd, dropout-key, model-variant and fit-loop checks add about 13 s to the file's run
time on that H100.
"""
import numpy as np
import pytest
import torch

from keras_ocr_b200 import _lib, weights as W
from keras_ocr_b200.recognition import Recognizer
from tests import ctc_train_refs as TR
from tests import rnn_train_refs as RR
from tests import stage_refs as R

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
LSTM_TIGHT = 2.0 ** -9
LSTM_LOOSE = 2.0 ** -7
AUTOGRAD_TOL = 2.0 ** -6


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _gamma(n):
    return n * U / (1 - n * U)


@pytest.fixture(scope="module")
def ctx(cuda_device):
    return _lib.Context(0)


def _a256(x):
    return (x + 255) // 256 * 256


def ws_slots(b, k, ctx, chunks=None):
    """Byte offsets of the workspace slots documented in include/b2ocr.h (b2o_rnn_loss_grad); ``chunks``: the number of
    split-K partials, (b + 15) // 16 as documented."""
    rows = b * 50
    chunks = (b + 15) // 16 if chunks is None else chunks
    sizes = [("w16t", 4 * 128 * 512 * 2), ("u16", 4 * 128 * 512 * 2), ("xz", 4 * rows * 512 * 4),
             ("acts", 4 * rows * 640 * 4), ("h1", 2 * rows * 128 * 2), ("l1", rows * 128 * 2), ("l2", rows * 256 * 2),
             ("dl2", rows * 256 * 4), ("dl1", rows * 128 * 4), ("partial", chunks * 526336 * 4),
             ("ctc", ctx.ctc_train_workspace_bytes(b, k))]
    out, at = {}, 0
    for name, n in sizes:
        out[name] = at
        at += _a256(n)
    out["end"] = at
    return out


def device_chunks(ctx, b, k):
    """The number of split-K chunks the LSTM weight gradients are summed over at batch b, read off the workspace size
    the library reports."""
    nbytes = ctx.rnn_train_workspace_bytes(b, k)
    found = [n for n in range(1, b + 1) if ws_slots(b, k, ctx, n)["end"] == nbytes]
    assert len(found) == 1, (b, k, nbytes)
    return found[0]


def state_of(ws, b, k, ctx):
    """The forward state in the workspace after a call: xw (valid after a loss-only call), acts, h1, l1, l2."""
    sl = ws_slots(b, k, ctx)
    return {"xw": _view(ws, sl["xz"], (4, b, 50, 512), torch.float32),
            "acts": _view(ws, sl["acts"], (4, b, 50, 5, 128), torch.float32),
            "h1": _view(ws, sl["h1"], (2, b, 50, 128), torch.float16),
            "l1": _view(ws, sl["l1"], (b, 50, 128), torch.float16),
            "l2": _view(ws, sl["l2"], (b, 50, 256), torch.float16)}


def _view(ws, off, shape, dtype):
    n = int(np.prod(shape)) * torch.tensor([], dtype=dtype).element_size()
    return ws[off:off + n].view(dtype).view(shape).cpu().numpy()


def run(ctx, x_t, n_rows, index, k, params_t, off, lab, dropout=0.0, seed=0, step=0, grads=True):
    """(loss, grad or None, ws) with ws the workspace tensor after the call."""
    b = len(index)
    idx = torch.from_numpy(np.asarray(index, np.int32)).cuda()
    loss = torch.empty(b, dtype=torch.float32, device="cuda")
    grad = torch.empty_like(params_t) if grads else None
    nbytes = ctx.rnn_train_workspace_bytes(b, k)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    ctx.rnn_loss_grad(x_t.data_ptr(), n_rows, idx.data_ptr(), b, k, params_t.data_ptr(), off.data_ptr(), lab.data_ptr(),
                      dropout, seed, step, loss.data_ptr(), grad.data_ptr() if grads else None, ws.data_ptr(), nbytes,
                      _stream())
    return loss.cpu().numpy(), (grad.cpu().numpy() if grads else None), ws


def _csr(targets):
    off = np.zeros(len(targets) + 1, np.int32)
    off[1:] = np.cumsum([len(t) for t in targets])
    lab = np.array([c for t in targets for c in t], np.int16)
    return torch.from_numpy(off).cuda(), torch.from_numpy(lab).cuda()


def _targets(rng, k, b):
    """Label sequences of lengths 1 to 48, with doubled letters, all alignable in 48 steps."""
    out = []
    for i in range(b):
        kind = i % 4
        if kind == 0:
            seq = [int(c) for c in rng.integers(0, k - 1, int(rng.integers(1, 4)))]
        elif kind == 1:
            seq = [int(j % (k - 1)) for j in range(48)] if k > 2 else [0, 0, 0]
        elif kind == 2:
            n = int(rng.integers(2, 12))
            seq = [int(c) for c in rng.integers(0, k - 1, n)]
            for j in range(1, n, 3):
                seq[j] = seq[j - 1]
        else:
            seq = [int(rng.integers(0, k - 1))] * int(rng.integers(1, 25))
        out.append(seq)
    return out


def _tensors(k, seed):
    rng = np.random.default_rng(seed)
    t = {}
    for layer in RR.LAYERS:
        t[layer + ".kernel"] = (rng.normal(size=(128, 512)) * 0.12).astype(np.float32)
        t[layer + ".recurrent_kernel"] = (rng.normal(size=(128, 512)) * 0.08).astype(np.float32)
        t[layer + ".bias"] = (rng.normal(size=512) * 0.3).astype(np.float32)
    t["fc_12.kernel"] = (rng.normal(size=(256, k)) * rng.choice([0.05, 0.3])).astype(np.float32)
    t["fc_12.bias"] = (rng.normal(size=k) * 0.5).astype(np.float32)
    if k > 2:
        t["fc_12.bias"][k - 1] += 2.0
    return t


def _x(n, seed):
    return np.maximum(np.random.default_rng(seed).normal(size=(n, 50, 128)), 0).astype(np.float16)


def _synth(seeds):
    from oracle.train_crnn_full import synth_crop
    made = [synth_crop(s) for s in seeds]
    return np.stack([m[0] for m in made]), [m[1] for m in made]


def _input(rec, crops):
    t = torch.from_numpy(np.ascontiguousarray(crops)).cuda()
    x = torch.empty((len(crops), 200, 31) + ((3,) if rec.color else ()), dtype=torch.float16, device="cuda")
    rec.ctx.crops_to_input(t.data_ptr(), len(crops), x.data_ptr(), _stream(), color=rec.color)
    return x


# ------------------------------------------------------------------------------------------ 1. sequence features
def _sequence_features_vs_tap(rec, crops, what):
    """b2o_crnn_sequence_features of ``crops`` on ``rec`` against the "fc_9" tap of a full forward, bit for bit."""
    rec.keep_workspace = True
    b = len(crops)
    x = _input(rec, crops)
    rec.predict_device(x)
    tap = rec.tap("fc_9", (b, 50, 128), torch.float16).cpu().numpy()
    out = torch.empty((b, 50, 128), dtype=torch.float16, device="cuda")
    nbytes = rec.ctx.crnn_workspace_bytes(b)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    feats = torch.empty((b, 48, 256), dtype=torch.float16, device="cuda")
    n0 = rec.ctx.launch_count()
    rec.ctx.crnn_features(x.data_ptr(), b, feats.data_ptr(), ws.data_ptr(), nbytes, _stream())
    n1 = rec.ctx.launch_count()
    rec.ctx.crnn_sequence_features(x.data_ptr(), b, out.data_ptr(), ws.data_ptr(), nbytes, _stream())
    n2 = rec.ctx.launch_count()
    assert np.array_equal(out.cpu().numpy().view(np.int16), tap.view(np.int16))
    print(f"sequence features ({what}): {n2 - n1} launches (b2o_crnn_features: {n1 - n0}), bit-identical to the "
          f"fc_9 tap")
    assert 0 < n2 - n1 < n1 - n0
    small = torch.empty(16, dtype=torch.uint8, device="cuda")
    with pytest.raises(_lib.B2OError):                    # the last forward stopped after fc_9: no l1 / l2 to tap
        rec.ctx.crnn_tap("l2", ws.data_ptr(), b, small.data_ptr(), 16, _stream())


def test_sequence_features_are_the_fc9_tap():
    crops, _ = _synth(range(72_000_000, 72_000_019))
    _sequence_features_vs_tap(Recognizer(weights=W.synthetic_crnn_weights(decisive=True)), crops, "trained")


@pytest.mark.parametrize("variant", ["stn_false", "color"])
def test_sequence_features_are_the_fc9_tap_on_variants(variant):
    """build_model(stn=False), whose fc_9 reads bn_7's output directly, and build_model(color=True), on RGB crops."""
    crops, _ = _synth(range(72_000_000, 72_000_019))
    if variant == "stn_false":
        rec = Recognizer(weights=W.synthetic_crnn_weights(5, stn=False), build_params={"stn": False})
    else:
        rec = Recognizer(weights=W.synthetic_crnn_weights(6, color=True), build_params={"color": True})
        crops = np.stack([crops, crops[:, ::-1], 255 - crops], -1)
    _sequence_features_vs_tap(rec, crops, variant)


# ------------------------------------------------------------------------------------------ 2. training forward
def test_training_forward(ctx):
    from oracle import crnn
    hw = W.synthetic_crnn_weights(decisive=True)
    rec = Recognizer(weights=hw)
    crops, words = _synth(range(73_000_000, 73_000_021))
    b = len(crops)
    seq = rec._features(crops, sequence=True)
    feats = rec._features(crops)
    k = 37
    targets = [[rec.alphabet.index(c) for c in wd] for wd in words]
    off, lab = _csr(targets)
    params = torch.from_numpy(RR.flat(hw, k)).cuda()
    loss, _, ws = run(ctx, seq, b, np.arange(b), k, params, off, lab, grads=False)
    sl = ws_slots(b, k, ctx)
    l1 = _view(ws, sl["l1"], (b, 50, 128), torch.float16).astype(np.float64)
    l2 = _view(ws, sl["l2"], (b, 50, 256), torch.float16).astype(np.float64)
    x = seq.cpu().numpy().astype(np.float64)

    def xw(inp, name):
        return inp @ R.f16(hw[name + ".kernel"]) + hw[name + ".bias"].astype(np.float64)
    ref1 = R.f16(R.lstm_emulated(xw(x, "lstm_10"), hw["lstm_10.recurrent_kernel"]) +
                 R.lstm_emulated(xw(x, "lstm_10_back"), hw["lstm_10_back.recurrent_kernel"], go_backwards=True))
    ref2 = np.concatenate([R.lstm_emulated(xw(l1, "lstm_11"), hw["lstm_11.recurrent_kernel"]),
                           R.lstm_emulated(xw(l1, "lstm_11_back"), hw["lstm_11_back.recurrent_kernel"],
                                           go_backwards=True)], -1)
    e1, e2 = float(np.abs(l1 - ref1).max()), float(np.abs(l2 - ref2).max())
    wt = {n: torch.from_numpy(np.asarray(v)) for n, v in hw.items()}
    xf, l1f = torch.from_numpy(x).float(), torch.from_numpy(l1).float()
    o1 = (crnn.lstm(wt, xf, "lstm_10") + crnn.lstm(wt, xf, "lstm_10_back", go_backwards=True)).double().numpy()
    o2 = torch.cat([crnn.lstm(wt, l1f, "lstm_11"), crnn.lstm(wt, l1f, "lstm_11_back", go_backwards=True)],
                   -1).double().numpy()
    f1, f2 = float(np.abs(l1 - o1).max()), float(np.abs(l2 - o2).max())
    assert max(e1, e2) <= LSTM_TIGHT and max(f1, f2) <= LSTM_LOOSE, (e1, e2, f1, f2)
    # the loss against fit_top's on the inference features
    ref_loss = torch.empty(b, dtype=torch.float32, device="cuda")
    wtop = torch.from_numpy(hw["fc_12.kernel"]).cuda()
    btop = torch.from_numpy(hw["fc_12.bias"]).cuda()
    idx = torch.arange(b, dtype=torch.int32, device="cuda")
    ctx.ctc_loss_grad(feats.data_ptr(), b, idx.data_ptr(), b, k, wtop.data_ptr(), btop.data_ptr(), off.data_ptr(),
                      lab.data_ptr(), 0.0, 0, 0, ref_loss.data_ptr(), None, None, None, None, 0, _stream())
    ref_loss = ref_loss.cpu().numpy().astype(np.float64)
    wa = np.abs(hw["fc_12.kernel"]).astype(np.float64)
    lg = l2[:, 2:] @ hw["fc_12.kernel"].astype(np.float64) + hw["fc_12.bias"]
    delta = 10 * U + 2 * U * (lg.max(-1) - lg.min(-1)) + _gamma(k + 8)
    worst = 0.0
    for i in range(b):
        mag = np.abs(l2[i, 2:]) @ wa + np.abs(hw["fc_12.bias"])
        shift = (LSTM_TIGHT * wa.sum(0)[None, :] + 2 * _gamma(257) * mag).max(-1)
        tau_l = 1.01 * ((3 * U + delta[i]).sum() + U) + U * abs(ref_loss[i]) + 1e-12
        bound = 2 * shift.sum() + 2 * tau_l
        worst = max(worst, abs(loss[i] - ref_loss[i]) / bound)
    print(f"training forward: l1 / l2 within {e1:.3g} / {e2:.3g} of the emulation, {f1:.3g} / {f2:.3g} of "
          f"oracle.crnn.lstm; loss vs fit_top's: worst {worst:.3g} of its bound")
    assert worst <= 1.0


# ------------------------------------------------------------------------------------------ 3. gradients
# (b, K, chunks): LSTM CTAs of 8 crops with a partial last one (11), one full CTA (8), one chunk of 16 crops, one crop
# more (a one-crop chunk tail), and the batch sizes training runs at (64 by default, 256 in scripts/bench_fit_recurrent.py)
GRAD_CASES = [(11, 2, 1), (11, 38, 1), (11, 1024, 1), (8, 38, 1), (16, 38, 1), (17, 2, 2), (64, 1024, 4),
              (256, 38, 16)]


@pytest.mark.parametrize("b,k,chunks", GRAD_CASES, ids=[str(k) if b == 11 else f"{k}-b{b}" for b, k, _ in GRAD_CASES])
def test_gradients_teacher_forced(ctx, b, k, chunks):
    n_rows = b + 12
    assert device_chunks(ctx, b, k) == chunks
    seed = k if b == 11 else 1000 * b + k
    rng = np.random.default_rng(seed)
    t = _tensors(k, seed)
    xs = _x(n_rows, seed + 1)
    targets = _targets(rng, k, b)
    index = rng.permutation(n_rows)[:b]
    x_t = torch.from_numpy(xs).cuda()
    params = torch.from_numpy(RR.flat(t, k)).cuda()
    off, lab = _csr(targets)
    report = []
    for dropout, seed, step in ((0.0, 0, 0), (0.25, 7, 3)):
        loss, grad, ws = run(ctx, x_t, n_rows, index, k, params, off, lab, dropout, seed, step)
        assert np.isfinite(loss).all()
        sl = ws_slots(b, k, ctx)
        acts = _view(ws, sl["acts"], (4, b, 50, 5, 128), torch.float32)
        h1 = _view(ws, sl["h1"], (2, b, 50, 128), torch.float16)
        l1 = _view(ws, sl["l1"], (b, 50, 128), torch.float16)
        l2 = _view(ws, sl["l2"], (b, 50, 256), torch.float16)
        g = _view(ws, sl["ctc"], (b, 48, k), torch.float32)
        ref, bound = RR.backward(xs[index], acts, h1, l1, l2, g, t, index, dropout, seed, step)
        dev = RR.unflat(grad, k)
        worst = {}
        for name, _ in RR.tensor_names(k):
            r = np.abs(dev[name] - ref[name]) / (1.01 * bound[name] + 1e-30)
            worst[name] = float(r.max())
        name = max(worst, key=worst.get)
        report.append(f"dropout {dropout}: worst {worst[name]:.3g} of the bound ({name})")
        assert worst[name] <= 1.0, (k, dropout, worst)
        if dropout == 0:
            only, none, _ = run(ctx, x_t, n_rows, index, k, params, off, lab, grads=False)
            assert none is None and np.array_equal(only.view(np.int32), loss.view(np.int32))
    print(f"rnn_loss_grad b={b} ({chunks} chunks) K={k}: " + "; ".join(report))


def _problem(b, k, seed, out_of_range=True):
    """(tensors, x cache, n_rows, permuted index with one row outside the cache when b > 1 and out_of_range, targets)."""
    n_rows = b + 7
    rng = np.random.default_rng(seed)
    t = _tensors(k, seed)
    xs = _x(n_rows, seed + 1)
    index = rng.permutation(n_rows)[:b]
    if b > 1 and out_of_range:
        index[b // 2] = n_rows + 3
    return t, xs, n_rows, index, _targets(rng, k, b)


@pytest.mark.parametrize("b", [1, 17, 64])
def test_forward_state_vs_fp64(ctx, b):
    """The state the teacher-forced gradient test feeds to the reference backward, checked step by step by
    ``rnn_train_refs.state_ratios`` (xw of all four directions in input order, the gates and c per processing step, h),
    with a permuted index and one row outside the cache (its x reads as zeros: xw = the bias).  The forward does not
    depend on dropout or on whether gradients are asked for: acts, h1, l1 and l2 are bit-identical over loss-only and
    gradient calls with dropout 0 and 0.25, so the state checked here is the one the gradient test reads."""
    k = 38
    t, xs, n_rows, index, targets = _problem(b, k, 500 + b)
    x_t = torch.from_numpy(xs).cuda()
    params = torch.from_numpy(RR.flat(t, k)).cuda()
    off, lab = _csr(targets)
    states = []
    for dropout, seed, step in ((0.0, 0, 0), (0.25, 7, 3)):
        for grads in (False, True):
            ws = run(ctx, x_t, n_rows, index, k, params, off, lab, dropout, seed, step, grads=grads)[2]
            states.append(state_of(ws, b, k, ctx))
    first = states[0]
    for st in states[1:]:
        for name in ("acts", "h1", "l1", "l2"):
            assert np.array_equal(st[name].view(np.uint8), first[name].view(np.uint8)), name
    assert np.array_equal(states[2]["xw"].view(np.uint8), first["xw"].view(np.uint8))     # gradient calls reuse xw for dz
    x = np.where((index < n_rows)[:, None, None], xs[np.minimum(index, n_rows - 1)], 0)
    ratios = RR.state_ratios(x, t, first["xw"], first["acts"], first["h1"], first["l1"], first["l2"])
    print(f"forward state b={b}: worst " + ", ".join(f"{n} {v:.3g}" for n, v in ratios.items()) + " of their bounds")
    assert max(ratios.values()) <= 1.0, ratios


@pytest.mark.parametrize("b", [17, 64])
def test_fc12_gradient_is_the_fit_top_kernel(ctx, b):
    """fc_12's part of b2o_rnn_loss_grad is b2o_ctc_loss_grad on the device's own l2: with l2's kept steps placed at
    the crops' rows of an (n_rows, 48, 256) cache, the fit_top entry point gives the same loss, g = dL/dlogits and fc_12
    gradients in every bit, with and without dropout."""
    k = 38
    t, xs, n_rows, index, targets = _problem(b, k, 600 + b, out_of_range=False)
    x_t = torch.from_numpy(xs).cuda()
    params = torch.from_numpy(RR.flat(t, k)).cuda()
    off, lab = _csr(targets)
    idx = torch.from_numpy(index.astype(np.int32)).cuda()
    n_lstm = sum(int(np.prod(shape)) for _, shape in RR.tensor_names(k)[:12])
    fc_w, fc_b = params[n_lstm:n_lstm + 256 * k], params[n_lstm + 256 * k:]
    for dropout, seed, step in ((0.0, 0, 0), (0.25, 7, 3)):
        loss, grad, ws = run(ctx, x_t, n_rows, index, k, params, off, lab, dropout, seed, step)
        sl = ws_slots(b, k, ctx)
        l2 = ws[sl["l2"]:sl["l2"] + b * 50 * 256 * 2].view(torch.float16).view(b, 50, 256)
        feats = torch.zeros((n_rows, 48, 256), dtype=torch.float16, device="cuda")
        feats[idx.long()] = l2[:, 2:]
        loss2 = torch.empty(b, dtype=torch.float32, device="cuda")
        gw, gb = torch.empty(256 * k, dtype=torch.float32, device="cuda"), torch.empty(k, dtype=torch.float32,
                                                                                       device="cuda")
        nbytes = ctx.ctc_train_workspace_bytes(b, k)
        ws2 = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        ctx.ctc_loss_grad(feats.data_ptr(), n_rows, idx.data_ptr(), b, k, fc_w.data_ptr(), fc_b.data_ptr(),
                          off.data_ptr(), lab.data_ptr(), dropout, seed, step, loss2.data_ptr(), gw.data_ptr(),
                          gb.data_ptr(), None, ws2.data_ptr(), nbytes, _stream())
        n_g = b * 48 * k * 4
        assert np.isfinite(loss).all()
        assert np.array_equal(loss2.cpu().numpy().view(np.int32), loss.view(np.int32))
        assert torch.equal(ws2[:n_g], ws[sl["ctc"]:sl["ctc"] + n_g])
        assert np.array_equal(gw.cpu().numpy().view(np.int32), grad[n_lstm:n_lstm + 256 * k].view(np.int32))
        assert np.array_equal(gb.cpu().numpy().view(np.int32), grad[n_lstm + 256 * k:].view(np.int32))


def test_gradients_vs_autograd(ctx):
    """The whole chain against autograd through ``rnn_train_refs.head_losses`` with the device's roundings emulated
    (the fp64 forward, not the device's activations), at a batch of two chunks with dropout.  There is no rigorous bound:
    an fp16 rounding of h that falls the other way in fp32 than in fp64 moves everything after it.  Relative Frobenius
    error per tensor <= AUTOGRAD_TOL."""
    k, b = 38, 17
    t, xs, n_rows, index, targets = _problem(b, k, 700, out_of_range=False)
    x_t = torch.from_numpy(xs).cuda()
    params = torch.from_numpy(RR.flat(t, k)).cuda()
    loss, grad, _ = run(ctx, x_t, n_rows, index, k, params, *_csr(targets), 0.25, 7, 3)
    ref_loss, ref = RR.head_losses(t, xs[index].astype(np.float64), targets, index, 0.25, 7, 3, rounding=True)
    dev = RR.unflat(grad, k)
    err = {n: float(np.linalg.norm(dev[n] - ref[n]) / np.linalg.norm(ref[n])) for n, _ in RR.tensor_names(k)}
    name = max(err, key=err.get)
    loss_err = float(np.abs(loss - ref_loss).max() / np.abs(ref_loss).max())
    print(f"gradients vs autograd: worst relative Frobenius error {err[name]:.3g} ({name}), loss {loss_err:.3g}")
    assert err[name] <= AUTOGRAD_TOL, err


def test_unalignable_crop_adds_nothing(ctx):
    k, n_rows = 38, 9
    rng = np.random.default_rng(3)
    t = _tensors(k, 3)
    x_t = torch.from_numpy(_x(n_rows, 4)).cuda()
    params = torch.from_numpy(RR.flat(t, k)).cuda()
    good = _targets(rng, k, 5)
    loss, grad, _ = run(ctx, x_t, n_rows, [0, 1, 2, 3, 4, 5], k, params, *_csr(good[:3] + [[3] * 25] + good[3:]))
    assert loss[3] == np.inf and np.isfinite(np.delete(loss, 3)).all()
    loss2, grad2, _ = run(ctx, x_t, n_rows, [0, 1, 2, 4, 5], k, params, *_csr(good))
    assert np.array_equal(np.delete(loss, 3).view(np.int32), loss2.view(np.int32))
    scale = np.abs(grad2).max()
    assert np.abs(grad * 6 - grad2 * 5).max() <= 1e-5 * scale
    bad_row, _, _ = run(ctx, x_t, n_rows, [0, 99], k, params, *_csr(good[:2]), grads=False)
    assert np.isfinite(bad_row[0]) and np.isnan(bad_row[1])


def test_dropout_keys_past_2_31(ctx):
    """Crops at rows 174,763 and 200,003 of a 200,004-row fc_9 cache (2.6 GB, only the used rows written), whose dropout
    keys row * 48 * 256 pass 2^31: on the kept steps dL/dl2 is 0 exactly where the mask rebuilt from 64-bit keys drops a
    feature, wherever g w^T is certainly not 0 (|g w^T| above twice the gamma(K) bound of its fp32 sum)."""
    rows, n_rows = np.array([0, 174_763, 200_003]), 200_004
    assert int(rows[1]) * 48 * 256 >= 2 ** 31 > (int(rows[1]) - 1) * 48 * 256
    k, dropout, seed, step = 38, 0.25, 7, 3
    t = _tensors(k, 31)
    params = torch.from_numpy(RR.flat(t, k)).cuda()
    targets = _targets(np.random.default_rng(31), k, len(rows))
    x_t = torch.empty((n_rows, 50, 128), dtype=torch.float16, device="cuda")
    try:
        x_t[torch.from_numpy(rows).cuda()] = torch.from_numpy(_x(len(rows), 32)).cuda()
        loss, _, ws = run(ctx, x_t, n_rows, rows, k, params, *_csr(targets), dropout, seed, step)
    finally:
        del x_t
        torch.cuda.empty_cache()
    sl = ws_slots(len(rows), k, ctx)
    dl2 = _view(ws, sl["dl2"], (len(rows), 50, 256), torch.float32)
    g = _view(ws, sl["ctc"], (len(rows), 48, k), torch.float32).astype(np.float64)
    w = t["fc_12.kernel"].astype(np.float64)
    sure = np.abs(g @ w.T) > 2 * _gamma(k) * (np.abs(g) @ np.abs(w).T)
    mask = TR.keep_mask(rows, dropout, seed, step)
    print(f"dropout keys past 2^31: dL/dl2's zeros checked on {sure.mean():.4f} of the kept steps' features")
    assert np.isfinite(loss).all() and sure.mean() > 0.9
    assert not dl2[:, :2].any() and np.array_equal((dl2[:, 2:] != 0)[sure], mask[sure])


# ------------------------------------------------------------------------------------------ 4. determinism
def test_determinism_and_batch_independence(ctx):
    k, n_rows, b = 38, 40, 29
    rng = np.random.default_rng(9)
    t = _tensors(k, 9)
    targets = _targets(rng, k, b)
    index = rng.permutation(n_rows)[:b]
    x_t = torch.from_numpy(_x(n_rows, 10)).cuda()
    params = torch.from_numpy(RR.flat(t, k)).cuda()
    off, lab = _csr(targets)
    a = run(ctx, x_t, n_rows, index, k, params, off, lab, 0.25, 5, 11)
    c = run(ctx, x_t, n_rows, index, k, params, off, lab, 0.25, 5, 11)
    assert np.array_equal(a[0].view(np.int32), c[0].view(np.int32))
    assert np.array_equal(a[1].view(np.int32), c[1].view(np.int32))
    perm = rng.permutation(b)
    p = run(ctx, x_t, n_rows, index[perm], k, params, *_csr([targets[i] for i in perm]), 0.25, 5, 11)
    assert np.array_equal(p[0].view(np.int32), a[0][perm].view(np.int32))
    one = run(ctx, x_t, n_rows, index[3:4], k, params, *_csr(targets[3:4]), 0.25, 5, 11)
    assert one[0].view(np.int32)[0] == a[0].view(np.int32)[3]


# ------------------------------------------------------------------------------------------ 5. memory contract
GUARD = 4096


def _guarded(nbytes, fill):
    buf = torch.full((GUARD + nbytes + GUARD,), fill, dtype=torch.uint8, device="cuda")
    return buf, buf[GUARD:GUARD + nbytes]


def test_memory_contract(ctx):
    k, n_rows, b = 38, 12, 9
    rng = np.random.default_rng(12)
    t = _tensors(k, 12)
    x_t = torch.from_numpy(_x(n_rows, 13)).cuda()
    params = torch.from_numpy(RR.flat(t, k)).cuda()
    off, lab = _csr(_targets(rng, k, b))
    idx = torch.from_numpy(rng.permutation(n_rows)[:b].astype(np.int32)).cuda()
    consts = [a.clone() for a in (x_t, params, off, lab, idx)]
    nbytes = ctx.rnn_train_workspace_bytes(b, k)
    n_grad = params.numel() * 4
    results = []
    for out_fill, ws_fill in ((0x00, 0xFF), (0xFF, 0x00), (0x7B, 0x00)):
        lbuf, loss = _guarded(b * 4, out_fill)
        gbuf, grad = _guarded(n_grad, out_fill)
        wbuf, ws = _guarded(nbytes, ws_fill)
        ctx.rnn_loss_grad(x_t.data_ptr(), n_rows, idx.data_ptr(), b, k, params.data_ptr(), off.data_ptr(),
                          lab.data_ptr(), 0.25, 1, 2, loss.data_ptr(), grad.data_ptr(), ws.data_ptr(), nbytes, _stream())
        for buf in (lbuf, gbuf, wbuf):
            fill = ws_fill if buf is wbuf else out_fill
            assert bool((buf[:GUARD] == fill).all()) and bool((buf[-GUARD:] == fill).all())
        results.append((loss.cpu().numpy().copy(), grad.cpu().numpy().copy()))
        # rejected calls (workspace one byte short, a bad k) and b = 0 write nothing and launch nothing
        snap = [bb.clone() for bb in (lbuf, gbuf, wbuf)]
        n0 = ctx.launch_count()
        for kk, size, bb in ((k, nbytes - 1, b), (1, nbytes, b), (k, nbytes, 0)):
            rc = ctx.lib.b2o_rnn_loss_grad(ctx.handle, x_t.data_ptr(), n_rows, idx.data_ptr(), bb, kk,
                                           params.data_ptr(), off.data_ptr(), lab.data_ptr(), 0.25, 1, 2,
                                           loss.data_ptr(), grad.data_ptr(), ws.data_ptr(), size, None)
            assert (rc == 0) == (bb == 0)
        torch.cuda.synchronize()
        assert ctx.launch_count() == n0
        assert all(bool(torch.equal(a, s)) for a, s in zip((lbuf, gbuf, wbuf), snap))
    for lo, gr in results[1:]:
        assert np.array_equal(lo.view(np.int32), results[0][0].view(np.int32))
        assert np.array_equal(gr.view(np.int32), results[0][1].view(np.int32))
    assert all(bool(torch.equal(a, c)) for a, c in zip((x_t, params, off, lab, idx), consts))
    # b2o_crnn_sequence_features: guarded output, the same values under every prefill
    rec = Recognizer(weights=W.synthetic_crnn_weights(decisive=True))
    crops, _ = _synth(range(74_000_000, 74_000_005))
    xin = _input(rec, crops)
    xin0 = xin.clone()
    cws = rec.ctx.crnn_workspace_bytes(5)
    seen = []
    for fill in (0x00, 0xFF, 0x7B):
        obuf, out = _guarded(5 * 50 * 128 * 2, fill)
        wbuf, w2 = _guarded(cws, 0xFF - fill)
        rec.ctx.crnn_sequence_features(xin.data_ptr(), 5, out.data_ptr(), w2.data_ptr(), cws, _stream())
        assert bool((obuf[:GUARD] == fill).all()) and bool((obuf[-GUARD:] == fill).all())
        assert bool((wbuf[:GUARD] == 0xFF - fill).all()) and bool((wbuf[-GUARD:] == 0xFF - fill).all())
        seen.append(out.cpu().numpy().copy())
        n0 = rec.ctx.launch_count()
        snap = obuf.clone()
        assert rec.ctx.lib.b2o_crnn_sequence_features(rec.ctx.handle, xin.data_ptr(), 5, out.data_ptr(), w2.data_ptr(),
                                                      cws - 1, None) == -4
        assert rec.ctx.lib.b2o_crnn_sequence_features(rec.ctx.handle, xin.data_ptr(), 0, out.data_ptr(), w2.data_ptr(),
                                                      cws, None) == 0
        torch.cuda.synchronize()
        assert rec.ctx.launch_count() == n0 and bool(torch.equal(obuf, snap))
    assert all(np.array_equal(s, seen[0]) for s in seen) and bool(torch.equal(xin, xin0))


# ------------------------------------------------------------------------------------------ 6. end to end
N_TRAIN, N_HELD = 4096, 1024
EPOCHS, LR = 8, 1e-3
TRAIN_SEEDS = range(80_000_000, 80_000_000 + N_TRAIN)           # fit_top's training and held-out seeds
HELD_SEEDS = range(90_000_000, 90_000_000 + N_HELD)
MARGIN = 0.01


@pytest.fixture(scope="module")
def word_crops():
    return _synth(TRAIN_SEEDS), _synth(HELD_SEEDS)


def _rate(rec, crops, words):
    got = rec.recognize_crops(crops)
    return float(np.mean([a == b for a, b in zip(got, words)])), got


def _reinit_second_layer(hw, seed):
    """lstm_11 and lstm_11_back re-drawn as Keras draws them: he_normal kernel (truncated normal, std sqrt(2 / 128)),
    orthogonal recurrent kernel, zero bias with the forget gate's quarter at 1 (unit_forget_bias)."""
    rng = np.random.default_rng(seed)
    out = dict(hw)
    for layer in ("lstm_11", "lstm_11_back"):
        std = np.sqrt(2.0 / 128)
        w = rng.normal(size=(128, 512)) * std
        while np.any(np.abs(w) > 2 * std):
            bad = np.abs(w) > 2 * std
            w[bad] = rng.normal(size=int(bad.sum())) * std
        q, r = np.linalg.qr(rng.normal(size=(512, 128)))
        q = q * np.sign(np.diag(r))
        bias = np.zeros(512)
        bias[128:256] = 1.0
        out[layer + ".kernel"] = (w / 0.87962566103423978).astype(np.float32)   # Keras' truncation correction
        out[layer + ".recurrent_kernel"] = q.T.astype(np.float32)
        out[layer + ".bias"] = bias.astype(np.float32)
    return out


def test_fit_recurrent_recovers_the_second_layer(ctx, word_crops, tmp_path):
    import time
    (tc, tw), (hc, hwords) = word_crops
    hw = W.synthetic_crnn_weights(decisive=True)
    base, _ = _rate(Recognizer(weights=hw), hc, hwords)
    start = _reinit_second_layer(hw, 11)
    before, _ = _rate(Recognizer(weights=start), hc, hwords)
    top = Recognizer(weights=start)
    top.fit_top(tc, tw, epochs=EPOCHS, batch_size=64, learning_rate=LR, seed=3)
    top_rate, _ = _rate(top, hc, hwords)
    rec = Recognizer(weights=start)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    hist = rec.fit_recurrent(tc, tw, epochs=EPOCHS, batch_size=64, learning_rate=LR, seed=3,
                             validation=(hc[:512], hwords[:512]))
    torch.cuda.synchronize()
    secs = time.perf_counter() - t0
    rate, got = _rate(rec, hc, hwords)
    print(f"fit_recurrent, second layer re-initialised: held-out exact reads {before:.4f} before, {rate:.4f} after "
          f"({EPOCHS} epochs of {N_TRAIN} crops, {secs:.2f} s); fit_top from the same start {top_rate:.4f}; the trained "
          f"model {base:.4f}; loss {hist['loss']}; val_loss {hist['val_loss']}")
    assert len(hist["loss"]) == len(hist["val_loss"]) == EPOCHS
    assert hist["val_loss"][-1] < hist["val_loss"][0]
    assert rate >= base - MARGIN
    assert rate > top_rate
    path = str(tmp_path / "fitted.npz")
    rec.save_weights(path)
    loaded = Recognizer(weights=path)
    assert loaded.recognize_crops(hc) == got
    runs = []
    for _ in range(2):                                            # the same run twice: bit-identical weights
        r2 = Recognizer(weights=start)
        r2.fit_recurrent(tc[:1024], tw[:1024], epochs=1, batch_size=64, learning_rate=LR, seed=3)
        runs.append(r2._tensors)
    for name, _ in RR.tensor_names(37):
        assert np.array_equal(runs[0][name].view(np.int32), runs[1][name].view(np.int32)), name


def test_fit_recurrent_does_no_harm(ctx, word_crops):
    (tc, tw), (hc, hwords) = word_crops
    rec = Recognizer(weights=W.synthetic_crnn_weights(decisive=True))
    before, _ = _rate(rec, hc, hwords)
    rec.fit_recurrent(tc[:2048], tw[:2048], epochs=1, batch_size=64, seed=1)
    after, _ = _rate(rec, hc, hwords)
    print(f"fine-tuning the trained BiLSTM: held-out exact reads {before:.4f} -> {after:.4f}")
    assert after >= before


def _logits(rec, crops):
    rec.keep_workspace = True
    rec.predict_device(_input(rec, crops))
    return rec.tap("logits", (len(crops), 48, len(rec.alphabet) + 1), torch.float32).cpu().numpy()


def test_fit_recurrent_is_its_abi_calls(ctx, tmp_path):
    """fit_recurrent, restated as the calls its docstring describes: per epoch a default_rng(seed) permutation, batches
    of batch_size in its order with a short last one (70 = 32 + 32 + 6), dropout keyed on a step counter that runs on
    across epochs, one RMSprop accumulator over the flat parameters carried over, the history as the means of the fp32
    losses, the validation loss without dropout after each epoch.  The 14 tensors and the history bit for bit; the
    reloaded CRNN reads like a recognizer loaded from save_weights."""
    n, bs, epochs, lr, dropout, seed = 70, 32, 2, 1e-3, 0.25, 5
    hw = W.synthetic_crnn_weights(decisive=True)
    crops, words = _synth(range(76_000_000, 76_000_000 + n))
    v_crops, v_words = _synth(range(76_100_000, 76_100_019))
    rec = Recognizer(weights=hw)
    hist = rec.fit_recurrent(crops, words, epochs=epochs, batch_size=bs, learning_rate=lr, dropout=dropout, seed=seed,
                             validation=(v_crops, v_words))
    k = len(rec.alphabet) + 1
    ref = Recognizer(weights=hw)

    def features(c):
        x = _input(ref, c)
        out = torch.empty((len(c), 50, 128), dtype=torch.float16, device="cuda")
        ws = torch.empty(ref.ctx.crnn_workspace_bytes(len(c)), dtype=torch.uint8, device="cuda")
        ref.ctx.crnn_sequence_features(x.data_ptr(), len(c), out.data_ptr(), ws.data_ptr(), ws.numel(), _stream())
        return out
    seq, v_seq = features(crops), features(v_crops)
    labels = [[rec.alphabet.index(c) for c in wd] for wd in words]
    v_labels = [[rec.alphabet.index(c) for c in wd] for wd in v_words]
    params = torch.from_numpy(RR.flat(hw, k)).cuda()
    acc = torch.zeros_like(params)
    rng = np.random.default_rng(seed)
    want = {"loss": [], "val_loss": []}
    step = 0
    for _ in range(epochs):
        perm = rng.permutation(n)
        seen = np.empty(n, np.float32)
        for i in range(0, n, bs):
            idx = perm[i:i + bs]
            loss, grad, _ = run(ctx, seq, n, idx, k, params, *_csr([labels[j] for j in idx]), dropout, seed, step)
            seen[i:i + len(idx)] = loss
            gt = torch.from_numpy(grad).cuda()
            ctx.rmsprop_step(params.data_ptr(), gt.data_ptr(), acc.data_ptr(), params.numel(), lr, 0.9, 1e-7, _stream())
            step += 1
        want["loss"].append(float(seen.astype(np.float64).mean()))
        v_loss = run(ctx, v_seq, len(v_crops), np.arange(len(v_crops)), k, params, *_csr(v_labels), grads=False)[0]
        want["val_loss"].append(float(v_loss.astype(np.float64).mean()))
    assert step == 6 and hist == want, (hist, want)
    trained = RR.unflat(params.cpu().numpy(), k)
    for name, _ in RR.tensor_names(k):
        assert np.array_equal(rec._tensors[name].view(np.int32), trained[name].view(np.int32)), name
    path = str(tmp_path / "recurrent.npz")
    rec.save_weights(path)
    assert np.array_equal(_logits(rec, v_crops).view(np.int32), _logits(Recognizer(weights=path), v_crops).view(np.int32))
    print(f"fit_recurrent as its ABI calls: history {hist}")


# ------------------------------------------------------------------------------------------ 7. argument checks
def test_abi_rejects_bad_arguments(ctx):
    lib, h = ctx.lib, ctx.handle
    k, b = 37, 2
    x = torch.zeros((4, 50, 128), dtype=torch.float16, device="cuda")
    params = torch.zeros(526_336 + 257 * 1025, dtype=torch.float32, device="cuda")
    off, lab = _csr([[1], [2]])
    loss = torch.empty(b, dtype=torch.float32, device="cuda")
    grad = torch.empty_like(params)
    nbytes = ctx.rnn_train_workspace_bytes(b, k)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    P = lambda t: t.data_ptr()                                    # noqa: E731

    def call(kk=k, bb=b, dropout=0.0, n_rows=4, xp=P(x), pp=P(params), lp=P(loss), size=nbytes, wsp=P(ws), gp=P(grad)):
        return lib.b2o_rnn_loss_grad(h, xp, n_rows, None, bb, kk, pp, P(off), P(lab), dropout, 0, 0, lp, gp, wsp, size,
                                     None)
    assert call() == 0
    for kwargs in ({"kk": 1}, {"kk": 1025}, {"dropout": 1.0}, {"dropout": -0.1}, {"dropout": float("nan")},
                   {"bb": -1}, {"n_rows": 0}, {"xp": None}, {"xp": P(x) + 2}, {"pp": None}, {"lp": None}):
        assert call(**kwargs) == -2, kwargs
        assert lib.b2o_last_error(h)
    assert call(size=nbytes - 1) == -4 and call(wsp=None) == -4 and call(gp=None, size=nbytes - 1) == -4
    assert call(gp=None) == 0
    assert lib.b2o_rnn_train_workspace_bytes(2, 1) == 0 and lib.b2o_rnn_train_workspace_bytes(0, 37) == 0
    assert lib.b2o_rnn_train_workspace_bytes(2, 37) == ws_slots(2, 37, ctx)["end"]
    rec = Recognizer(weights=W.synthetic_crnn_weights(decisive=True))
    assert rec.ctx.lib.b2o_crnn_sequence_features(rec.ctx.handle, P(x), 2, None, P(ws), nbytes, None) == -2
    torch.cuda.synchronize()


def test_fit_recurrent_rejects_before_launching():
    rec = Recognizer(weights=W.synthetic_crnn_weights(decisive=True))
    crops = np.full((3, 31, 200), 255, np.uint8)
    n0 = rec.ctx.launch_count()
    for texts in (["ab", "", "c"], ["ab", "A", "c"], ["ab", "x" * 49, "c"], ["ab", "oo" * 13, "c"], ["a", "b"]):
        with pytest.raises(ValueError):
            rec.fit_recurrent(crops, texts)
    for kwargs in ({"epochs": 0}, {"batch_size": 0}, {"learning_rate": -1.0}, {"dropout": 1.0}, {"seed": -1},
                   {"validation": (crops, ["a", "b", ""])}, {"validation": (crops[:2], ["a", "b", "c"])}):
        with pytest.raises(ValueError):
            rec.fit_recurrent(crops, ["a", "b", "c"], **kwargs)
    with pytest.raises(ValueError):
        rec.fit_recurrent(crops[:, :30], ["a", "b", "c"])
    assert rec.ctx.launch_count() == n0
