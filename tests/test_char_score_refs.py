"""CPU: the fp64 references for character scores (tests/char_score_refs.py) against brute force and against each
other, the host helper that turns device arrays into word tuples, and the validation of the public flags."""
import numpy as np
import pytest

from keras_ocr_b200 import recognition
from tests import beam_refs as BR
from tests import char_score_refs as CR

T = 48


def _lp(rng, k, t=T, sharp=3.0):
    return BR.log_probs(rng.normal(0.0, sharp, (t, k)))


@pytest.mark.parametrize("t", [3, 4, 5])
def test_definition_matches_brute_force(t):
    """Every edited sequence's F is its exact probability from enumerating all K^T alignments."""
    rng = np.random.default_rng(t)
    k = 3
    lp = _lp(rng, k, t, sharp=1.0)
    exact = BR.brute_force(lp)
    for y in ([], [0], [1], [0, 0], [0, 1], [1, 0, 1], [0, 1, 1]):
        f, logp = CR.definition(lp, y)
        assert logp == pytest.approx(exact.get(tuple(y), -np.inf), abs=1e-12) or (
            logp == -np.inf and tuple(y) not in exact)
        for j in range(len(y)):
            for e, z in enumerate(CR.edits(y, j, k)):
                want = exact.get(tuple(z), -np.inf)
                if np.isfinite(want):
                    assert f[j, e] == pytest.approx(want, abs=1e-12)
                else:
                    assert f[j, e] == -np.inf


def _cases(rng, k):
    """Readings that reach every branch of the recipe: empty, one character, doubled letters, 48-step-tight ones, a
    substitution equal to a neighbour, deletions that make the neighbours equal, unalignable readings."""
    a, b = 0, 1
    return [
        [], [a], [b], [a, a], [a, b, a], [a, a, b, b], [b, a, b, a, b],
        [a] * 24 + [b],                                     # 25 labels + 23 doubles = 48 steps: tight
        [a] * 24,                                           # 47 steps
        [a] * 25,                                           # 49 steps: F(y) = -inf, some edits finite
        [a, b] * 24,                                        # 48 labels, no doubles: tight
        rng.integers(0, k - 1, 12).tolist(),
        rng.integers(0, k - 1, 30).tolist(),
    ]


@pytest.mark.parametrize("k", [3, 5, 12])
def test_recipe_equals_definition(k):
    rng = np.random.default_rng(100 + k)
    for sharp in (1.0, 4.0):
        lp = _lp(rng, k, sharp=sharp)
        for y in _cases(rng, k):
            f_def, lp_def = CR.definition(lp, y)
            f_rec, lp_rec = CR.recipe(lp, y)
            assert np.array_equal(np.isneginf(f_def), np.isneginf(f_rec)), y
            fin = np.isfinite(f_def)
            assert np.abs(f_def[fin] - f_rec[fin]).max(initial=0.0) <= 1e-9, y
            assert (lp_def == lp_rec == -np.inf) or abs(lp_def - lp_rec) <= 1e-9


def test_recipe_on_greedy_readings():
    """Readings the decoder would return: the greedy collapse of peaked logits, at K = 37."""
    rng = np.random.default_rng(7)
    k = 37
    for _ in range(3):
        lg = rng.normal(0.0, 1.0, (T, k))
        lg[np.arange(T), rng.integers(0, k, T)] += 6.0
        lp = BR.log_probs(lg)
        y = list(BR.collapse(lp.argmax(1), k - 1))
        f_def, _ = CR.definition(lp, y)
        f_rec, _ = CR.recipe(lp, y)
        fin = np.isfinite(f_def)
        assert np.abs(f_def[fin] - f_rec[fin]).max(initial=0.0) <= 1e-9
        conf, labels, post, _ = CR.scores(f_rec, y, 8)
        assert np.allclose(np.exp(f_rec - np.logaddexp.reduce(f_rec, axis=1, keepdims=True)).sum(1), 1.0)
        assert ((conf > 0) & (conf <= 1)).all()
        assert (np.diff(post, axis=1) <= 0).all()


def test_scores_rules():
    f = np.array([[-1.0, -1.0, -3.0, -np.inf], [-np.inf] * 4, [-2.0, -np.inf, -np.inf, -np.inf]])
    conf, labels, post, margin = CR.scores(f, [1, 0, 0], 6)
    assert conf[0] == pytest.approx(np.exp(-1) / (2 * np.exp(-1) + np.exp(-3)))
    assert labels[0].tolist() == [0, 1, 2, 3, -1, -1]                  # equal values: the smaller label first
    assert post[0, 3] == 0 and post[0, 4] == 0
    assert margin[0] == 0                                               # a tie in fp64: not comparable
    assert conf[1] == 0 and (labels[1] == -1).all() and (post[1] == 0).all()   # L = -inf
    assert conf[2] == 1 and labels[2].tolist() == [0, 1, 2, 3, -1, -1] and margin[2] == 1.0


def test_host_helper():
    alphabet = "abc"                                                    # K = 4, the deletion is label 3
    conf = np.full((2, T), np.nan, np.float32)
    conf[0, :2] = [0.5, 0.25]
    alt_l = np.full((2, T, 2), -1, np.int32)
    alt_p = np.full((2, T, 2), np.nan, np.float32)
    alt_l[0, 0], alt_p[0, 0] = [0, 3], [0.5, 0.3]
    alt_l[0, 1], alt_p[0, 1] = [1, -1], [0.25, 0.0]
    out = recognition.char_scores_host(conf, ["ab", ""], alphabet)
    assert out[0].dtype == np.float32 and out[0].tolist() == [0.5, 0.25] and out[1].shape == (0,)
    out = recognition.char_scores_host(conf, ["ab", ""], alphabet, alt_l, alt_p)
    c, alts = out[0]
    assert c.tolist() == [0.5, 0.25]
    assert alts == [[("a", 0.5), ("", pytest.approx(0.3))], [("b", 0.25), (None, 0.0)]]
    assert out[1][0].shape == (0,) and out[1][1] == []
    # top_paths = P > 1: one entry per reading
    conf3, l3, p3 = conf[:, None].repeat(2, 1), alt_l[:, None].repeat(2, 1), alt_p[:, None].repeat(2, 1)
    out = recognition.char_scores_host(conf3, [["ab", "a"], ["", "b"]], alphabet, l3, p3)
    assert [len(o[0]) for o in out[0]] == [2, 1] and [len(o[0]) for o in out[1]] == [0, 1]
    assert np.isnan(out[1][1][0][0])                                    # slots past the reading stay NaN


def test_check_char_scores():
    assert recognition.check_char_scores() is None
    assert recognition.check_char_scores(True) == 0
    assert recognition.check_char_scores(True, np.int64(8)) == 8
    for bad in (-1, 9, 1.0, True, "2", None):
        with pytest.raises(ValueError, match="char_alternatives"):
            recognition.check_char_scores(True, bad)
    with pytest.raises(ValueError, match="return_char_scores"):
        recognition.check_char_scores(False, 2)
    with pytest.raises(ValueError, match="return_char_scores"):
        recognition.check_windows(2, char_scores=True)
    assert recognition.check_windows(1, char_scores=True) == 1
