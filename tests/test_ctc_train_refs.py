"""CPU: the fp64 references of tests/ctc_train_refs.py against independent computations, and the host-side validation
of ``Recognizer.fit_top``'s texts."""
import numpy as np
import pytest
import torch

from keras_ocr_b200.recognition import DEFAULT_ALPHABET, Lexicon, check_texts, encode_csr
from tests import beam_refs as BR
from tests import ctc_train_refs as TR

T = 48


def _torch_loss_grad(lg, labels):
    """Keras' ctc_batch_cost on the softmax output, restated: torch's CTC loss on log(softmax + 1e-7), fp64 autograd."""
    x = torch.tensor(lg, dtype=torch.float64, requires_grad=True)
    lp = torch.log(torch.softmax(x, -1) + 1e-7)
    k = lg.shape[-1]
    loss = torch.nn.functional.ctc_loss(lp[:, None, :], torch.tensor([list(labels)]), torch.tensor([T]),
                                        torch.tensor([len(labels)]), blank=k - 1, reduction="sum")
    loss.backward()
    return float(loss.detach()), x.grad.numpy()


def _cases():
    rng = np.random.default_rng(0)
    out = []
    for k, labels in [(37, (3, 4, 4, 5)), (37, (7,)), (2, (0,)), (2, (0, 0, 0)), (5, (1, 2, 3, 1, 2)),
                      (37, tuple(rng.integers(0, 36, 48))), (5, (2,) * 24), (3, (0, 1) * 24),
                      (38, (1, 1, 2, 2, 3, 3) * 4), (1024, tuple(rng.integers(0, 1023, 20)))]:
        scale = float(rng.choice([0.3, 1.0, 3.0]))
        lg = rng.normal(size=(T, k)) * scale
        out.append((k, labels, lg))
    return out


@pytest.mark.parametrize("case", range(10))
def test_loss_matches_lexicon_score_and_torch(case):
    k, labels, lg = _cases()[case]
    loss, g, info = TR.loss_grad(lg, labels)
    assert np.isfinite(loss)
    assert abs(loss + BR.forward_logprob(BR.log_probs(lg), labels)) <= 1e-9 * max(1.0, abs(loss))
    t_loss, t_grad = _torch_loss_grad(lg, labels)
    assert abs(loss - t_loss) <= 1e-9 * max(1.0, abs(loss))
    assert np.max(np.abs(g - t_grad)) <= 1e-9
    assert np.allclose(info["gamma"].sum(-1), 1.0, atol=1e-12)


def test_gradient_central_differences():
    rng = np.random.default_rng(3)
    for k, labels in [(2, (0,)), (4, (1, 1, 2)), (6, (0, 1, 2, 3, 4))]:
        lg = rng.normal(size=(T, k))
        _, g, _ = TR.loss_grad(lg, labels)
        h = 1e-6
        for _ in range(25):
            t, c = int(rng.integers(0, T)), int(rng.integers(0, k))
            up, dn = lg.copy(), lg.copy()
            up[t, c] += h
            dn[t, c] -= h
            fd = (TR.loss_grad(up, labels)[0] - TR.loss_grad(dn, labels)[0]) / (2 * h)
            assert abs(fd - g[t, c]) <= 1e-6, (k, labels, t, c, fd, g[t, c])


def test_unalignable_and_longest():
    rng = np.random.default_rng(4)
    lg = rng.normal(size=(T, 5))
    loss, g, _ = TR.loss_grad(lg, (2,) * 25)                       # 25 + 24 repeats > 48
    assert loss == np.inf and not g.any()
    loss, _, _ = TR.loss_grad(lg, (2,) * 24)                       # 24 + 23 = 47: aligns
    assert np.isfinite(loss)
    loss, _, _ = TR.loss_grad(lg, tuple(int(c) for c in rng.integers(0, 4, 48) * 0 + np.arange(48) % 4))
    assert np.isfinite(loss)                                        # 48 labels, no repeats: the diagonal path only


def test_weight_gradients_and_dropout_mask():
    rng = np.random.default_rng(5)
    feats = rng.normal(size=(10, T, 256)).astype(np.float16)
    rows = np.array([3, 7, 0])
    x = TR.dropped(feats, rows, 0.25, seed=11, step=2)
    keep = TR.keep_mask(rows, 0.25, 11, 2)
    assert 0.7 < keep.mean() < 0.8
    assert np.array_equal(x == 0, ~keep | (feats[rows] == 0))
    scale = np.float32(1) / (np.float32(1) - np.float32(0.25))
    assert np.array_equal(x[keep], feats[rows][keep].astype(np.float32) * scale)
    assert np.array_equal(TR.dropped(feats, rows, 0.0, 11, 2), feats[rows].astype(np.float32))
    assert not np.array_equal(TR.keep_mask(rows, 0.25, 11, 3), keep)        # a new step draws a new mask
    assert np.array_equal(TR.keep_mask(rows[::-1], 0.25, 11, 2), keep[::-1])  # the mask follows the row
    k = 7
    w, b = rng.normal(size=(256, k)) * 0.05, rng.normal(size=k) * 0.1
    texts = [(1, 2), (3, 3), (5,)]
    gs = np.stack([TR.loss_grad(lg, t)[1] for lg, t in zip(TR.logits(x, w, b), texts)])
    gw, gb = TR.batch_grads(x, gs)
    wt = torch.tensor(w, requires_grad=True)
    bt = torch.tensor(b, requires_grad=True)
    lg = torch.tensor(x, dtype=torch.float64) @ wt + bt
    lp = torch.log(torch.softmax(lg, -1) + 1e-7).permute(1, 0, 2)
    tg = torch.tensor([c for t in texts for c in t])
    loss = torch.nn.functional.ctc_loss(lp, tg, torch.full((3,), T), torch.tensor([len(t) for t in texts]),
                                        blank=k - 1, reduction="sum") / 3
    loss.backward()
    assert np.max(np.abs(gw - wt.grad.numpy())) <= 1e-9 and np.max(np.abs(gb - bt.grad.numpy())) <= 1e-9


def test_rmsprop_reference():
    p, g, a = np.array([1.0, -2.0, 0.5]), np.array([0.1, -0.3, 0.0]), np.zeros(3)
    p1, a1 = TR.rmsprop(p, g, a)
    assert np.allclose(a1, 0.1 * g * g)
    assert np.allclose(p1, p - 1e-3 * g / (np.sqrt(0.1 * g * g) + 1e-7))


# ---------------------------------------------------------------------------------------- host validation of texts
def test_check_texts_accepts_and_encodes():
    off, lab = check_texts(["ab", "ab", "yz" * 24, "a b", "aa" * 12], DEFAULT_ALPHABET + " ")
    assert off.tolist() == [0, 2, 4, 52, 55, 79]
    assert lab[:4].tolist() == [10, 11, 10, 11]
    assert lab.dtype == np.int16 and off.dtype == np.int32
    o2, l2 = encode_csr(["ab", "ab"], {c: i for i, c in enumerate(DEFAULT_ALPHABET)})
    assert np.array_equal(o2, off[:3]) and np.array_equal(l2, lab[:4])
    lex = Lexicon(["ab", "z"])                                      # the lexicon shares the encoding
    assert lex.offsets.tolist() == [0, 2, 3] and lex.labels.tolist() == [10, 11, 35]


@pytest.mark.parametrize("texts, where", [
    (["ok", ""], "text 1"),
    (["ok", 5], "text 1"),
    (["ok", "x" * 49], "text 1 .* longer than 48"),
    (["ok", "aB"], "text 1 .* 'B'"),
    ([" a", "a  b"], "text 1 .* two spaces"),
    (["ok", "aa" * 12 + "a"], "text 1 .* cannot be aligned"),
    (["ok", "o" * 25], "text 1 .* cannot be aligned"),
])
def test_check_texts_rejects(texts, where):
    with pytest.raises(ValueError, match=where):
        check_texts(texts, DEFAULT_ALPHABET + " ")


def test_check_texts_rejects_containers():
    for bad in ("abc", None, [], 3):
        with pytest.raises(ValueError):
            check_texts(bad)
    with pytest.raises(ValueError, match="'A'"):
        check_texts(["A"], alphabet="abc")
    check_texts(["A"], alphabet="A")
