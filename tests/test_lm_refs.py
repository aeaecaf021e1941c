"""CPU: the character language model (``recognition.CharLM``) against tests/lm_refs.py, and the fp64 reference of the
LM-fused beam search against brute force and against ``beam_refs.beam_search``."""
import itertools
import math

import numpy as np
import pytest

from keras_ocr_b200.recognition import LM_BOS, CharLM
from tests import beam_refs as BR
from tests import lm_refs as LR

def _words(seed, n, alphabet="abcdefgh", lo=1, hi=7):
    rng = np.random.default_rng(seed)
    return ["".join(rng.choice(list(alphabet), int(rng.integers(lo, hi + 1)))) for _ in range(n)]


@pytest.mark.parametrize("order", [2, 3, 5])
def test_fit_is_interpolated_kneser_ney(order):
    words = _words(order, 300)
    alphabet = "abcdefgh"
    lm = CharLM.fit(words, alphabet, order=order)
    ref = LR.KneserNey(words, alphabet, order)
    rng = np.random.default_rng(1)
    hists = [()] + [tuple(rng.integers(0, 8, int(rng.integers(1, order)))) for _ in range(40)]
    hists += [(LM_BOS,) + h[:order - 2] for h in hists[1:10]]
    for h in hists:
        for w in range(len(alphabet) + 1):
            got = lm.logp_symbol(w, h)
            want = math.log(ref.prob(w, h))
            assert abs(got - want) <= 1e-12 * max(1.0, abs(want)), (h, w, got, want)


@pytest.mark.parametrize("order", [2, 4, 8])
def test_every_history_sums_to_one(order):
    lm = CharLM.fit(_words(10 + order, 200), "abcdefgh", order=order)
    keys, rows = lm.host_tables()
    hists = [()] + lm._histories
    for h in hists:
        total = sum(math.exp(lm.logp_symbol(w, h)) for w in range(9))
        assert abs(total - 1.0) <= 1e-12, (h, total)
    assert keys[0] == 0 and all(int(a) < int(b) for a, b in zip(keys[:-1], keys[1:]))
    assert np.allclose(np.exp(rows.astype(np.float64)).sum(1), 1.0, atol=1e-5)


def test_hand_computed_bigram():
    """Corpus {"ab", "b"}, order 2.  Bigrams <s>a, ab, b</s>, <s>b, b</s>: raw counts 1, 1, 2, 1 -> D2 = 3/(3+2) = 0.6.
    Unigram continuation counts: a: {<s>} = 1, b: {a, <s>} = 2, </s>: {b} = 1 -> n1 = 2, n2 = 1, D1 = 0.5; total 4,
    gamma = 0.5 * 3 / 4 = 0.375, uniform 1/3 (a, b, </s>): P(a) = 0.5/4 + 0.125 = 0.25, P(b) = 1.5/4 + 0.125 = 0.5,
    P(</s>) = 0.25.  History b: b</s> 2 -> P*(</s>|b) = (2 - 0.6)/2 + 0.3 * 0.25 = 0.775, bo(b) = 0.6 * 1 / 2 = 0.3."""
    lm = CharLM.fit(["ab", "b"], "ab", order=2)
    e = math.exp
    assert abs(e(lm.logp_symbol(0, ())) - 0.25) < 1e-15
    assert abs(e(lm.logp_symbol(1, ())) - 0.5) < 1e-15
    assert abs(e(lm.logp_symbol(2, ())) - 0.25) < 1e-15
    assert abs(e(lm.logp_symbol(2, (1,))) - 0.775) < 1e-15
    assert abs(10 ** lm.backoff10[(1,)] - 0.3) < 1e-15
    assert abs(e(lm.logp_symbol(0, (1,))) - 0.3 * 0.25) < 1e-15          # backed off
    # <s>: <s>a 1, <s>b 1 -> D2 applies, gamma = 0.6 * 2 / 2 = 0.6: P(a|<s>) = 0.4/2 + 0.6 * 0.25 = 0.35
    assert abs(e(lm.logp_symbol(0, (LM_BOS,))) - 0.35) < 1e-15
    assert abs(lm.log_prob("b") - (lm.logp_symbol(1, (LM_BOS,)) + lm.logp_symbol(2, (1,)))) < 1e-15


def test_fit_is_deterministic():
    words = _words(3, 500)
    a, b = CharLM.fit(words, "abcdefgh", 4), CharLM.fit(list(reversed(words)), "abcdefgh", 4)
    assert a.logp10 == b.logp10 and a.backoff10 == b.backoff10
    ka, ra = a.host_tables()
    kb, rb = b.host_tables()
    assert np.array_equal(ka, kb) and np.array_equal(ra.view(np.int32), rb.view(np.int32))
    c = CharLM.fit(["ab", "b"], "ab", 2, counts=[3, 2])
    d = CharLM.fit(["ab"] * 3 + ["b"] * 2, "ab", 2)
    assert c.logp10 == d.logp10


def test_arpa_round_trip_is_exact(tmp_path):
    lm = CharLM.fit(_words(4, 400), "abcdefgh", order=5)
    path = str(tmp_path / "lm.arpa")
    lm.to_arpa(path)
    back = CharLM.from_arpa(path, "abcdefgh")
    assert back.order == 5 and back.logp10 == lm.logp10 and back.backoff10 == lm.backoff10
    text = open(path).read()
    assert CharLM.from_arpa(text, "abcdefgh").logp10 == lm.logp10
    parsed = LR.read_arpa(text)                       # the plain reader sees the same tables
    tok = lambda s: CharLM._token("abcdefgh", s)      # noqa: E731
    assert {tuple(tok(s) for s in g): v for g, v in lm.logp10.items()} == {g: v[0] for g, v in parsed.items()}


def test_from_arpa_drops_unk_and_reads_lmplz_style():
    text = "\n".join(["\\data\\", "ngram 1=5", "ngram 2=3", "", "\\1-grams:", "-1.0\t<unk>\t0", "-99\t<s>\t-0.2",
                      "-0.5\ta\t-0.1", "-0.4\tb", "-0.6\t</s>", "", "\\2-grams:", "-0.3\t<s> a", "-0.2\ta b",
                      "-0.5\t<unk> b", "", "\\end\\", ""])
    lm = CharLM.from_arpa(text, "ab")
    assert lm.order == 2 and (0,) in lm.logp10 and len(lm.logp10) == 6
    ln10 = math.log(10)
    assert abs(lm.logp_symbol(1, (0,)) - (-0.2 * ln10)) < 1e-15
    assert abs(lm.logp_symbol(0, (1,)) - (-0.5 * ln10)) < 1e-15      # b has no backoff: 0
    assert abs(lm.logp_symbol(1, (LM_BOS,)) - (-0.2 - 0.4) * ln10) < 1e-15


def test_folded_rows_equal_the_backoff_recursion():
    for order in (2, 3, 6):
        lm = CharLM.fit(_words(20 + order, 150), "abcdefgh", order=order)
        keys, rows = lm.host_tables()
        where = {int(k): i for i, k in enumerate(keys)}
        for h in [()] + lm._histories:
            r = rows[where[LR.history_key(h)]]
            for w in range(9):
                assert r[w] == np.float32(LR.backoff_logp(lm, w, h)) or \
                    abs(float(r[w]) - LR.backoff_logp(lm, w, h)) <= 2 ** -23 * abs(float(r[w])), (h, w)
        # an unlisted history reads the row of its longest listed suffix
        for prefix in [(0,) * 9, (7, 7, 7, 7), (1, 2, 3, 4, 5, 6, 7)]:
            i = LR.lookup_row(keys, order, prefix)
            h = ((LM_BOS,) + prefix)[-(order - 1):]
            for w in range(9):
                assert abs(float(rows[i, w]) - LR.backoff_logp(lm, w, h)) <= 1e-6 * max(1, abs(float(rows[i, w])))


def test_reference_with_zero_weights_is_plain_beam_search():
    lm = CharLM.fit(_words(5, 100, "ab"), "ab", order=3)
    keys, rows = lm.host_tables()
    rng = np.random.default_rng(0)
    for i in range(6):
        lp = BR.log_probs(rng.normal(size=(12, 3)) * (3 if i % 2 else 1))
        for w in (1, 3, 8):
            paths, a, fend, _ = LR.beam_search_lm(lp, w, keys, rows, 3, 0.0, 0.0)
            ref, score, _ = BR.beam_search(lp, w)
            assert paths == ref and np.array_equal(a, score) and np.array_equal(fend, score)


@pytest.mark.parametrize("alpha,beta", [(0.5, 0.0), (1.5, 0.7), (0.8, -1.0)])
def test_reference_finds_the_exhaustive_maximiser(alpha, beta):
    """With W at least the number of prefixes the search keeps every prefix: its best reading maximises F_end over
    every label sequence (enumerated from the alignments)."""
    lm = CharLM.fit(["ab", "ba", "aab", "b"], "ab", order=3)
    keys, rows = lm.host_tables()
    rng = np.random.default_rng(7)
    for _ in range(5):
        T = 4
        lp = BR.log_probs(rng.normal(size=(T, 3)) * 2)
        paths, _, fend, _ = LR.beam_search_lm(lp, 64, keys, rows, 3, alpha, beta, top_paths=1)
        seqs = {BR.collapse(p, 2) for p in itertools.product(range(3), repeat=T)}
        best = max(seqs, key=lambda s: (LR.fused_score(lp, s, keys, rows, 3, alpha, beta), [-c for c in s]))
        assert paths[0] == best
        assert abs(fend[0] - LR.fused_score(lp, best, keys, rows, 3, alpha, beta)) < 1e-9


def test_value_errors():
    with pytest.raises(ValueError, match="not a non-empty string"):
        CharLM.fit(["ab", ""], "ab")
    with pytest.raises(ValueError, match="not in the alphabet"):
        CharLM.fit(["ax"], "ab")
    with pytest.raises(ValueError, match="order"):
        CharLM.fit(["ab"], "ab", order=1)
    with pytest.raises(ValueError, match="order"):
        CharLM.fit(["ab"], "ab", order=9)
    with pytest.raises(ValueError, match="at most 126"):
        CharLM.fit(["ab"], "".join(chr(0x100 + i) for i in range(127)))
    with pytest.raises(ValueError, match="counts"):
        CharLM.fit(["ab"], "ab", counts=[0])
    lm = CharLM.fit(["ab"], "ab")
    for bad in (float("nan"), float("inf"), "1", None, 1e39, -4e38):     # 1e39 is inf in float32
        with pytest.raises(ValueError, match="finite"):
            lm.weighted(bad, 0.0)
        with pytest.raises(ValueError, match="finite"):
            lm.weighted(0.5, bad)
    w = lm.weighted(2.0, -1.0)
    assert (w.alpha, w.beta, lm.alpha) == (2.0, -1.0, CharLM.ALPHA) and w.logp10 is lm.logp10
    good = ["\\data\\", "ngram 1=4", "ngram 2=1", "", "\\1-grams:", "-99\t<s>\t-0.1", "-0.5\ta", "-0.4\tb",
            "-0.6\t</s>", "", "\\2-grams:", "-0.3\t<s> a", "", "\\end\\"]
    assert CharLM.from_arpa("\n".join(good), "ab").order == 2
    cases = [
        (["-0.5\tx" if ln == "-0.5\ta" else ln for ln in good], "token 'x'"),
        (["ngram 1=3" if ln == "ngram 1=4" else ln for ln in good if ln != "-0.4\tb"], "no unigram"),
        ([ln for ln in good if ln != "-0.4\tb"], "declares 4 1-grams, the file holds 3"),
        (good[:good.index("-0.3\t<s> a")], "declares 1 2-grams, the file holds 0"),      # truncated
        ([ln for ln in good if ln != "\\end\\"], "truncated"),
        ([ln for ln in good if not ln.startswith(("ngram 2", "\\2-", "-0.3"))], "order"),
        (["-0.3\ta <s>" if ln == "-0.3\t<s> a" else ln for ln in good], "may only"),
        (["-0.3\tb a" if ln == "-0.3\t<s> a" else ln for ln in good] + [], None),
        (["-0.3\t<s>" if ln == "-0.3\t<s> a" else ln for ln in good], "fields"),
        (["zz\ta" if ln == "-0.5\ta" else ln for ln in good], "malformed number"),
        (["nan\ta" if ln == "-0.5\ta" else ln for ln in good], "non-finite"),
    ]
    for lines, msg in cases:
        if msg is None:
            assert CharLM.from_arpa("\n".join(lines), "ab").order == 2
            continue
        with pytest.raises(ValueError, match=msg):
            CharLM.from_arpa("\n".join(lines), "ab")
    with pytest.raises(ValueError, match="line"):
        CharLM.from_arpa("\n".join(["-0.3\tb z" if ln == "-0.3\t<s> a" else ln for ln in good]), "ab")
    with pytest.raises(ValueError, match="whitespace"):
        CharLM.from_arpa("\n".join(good), "a b")


def test_history_limit(monkeypatch):
    from keras_ocr_b200 import _lib
    monkeypatch.setattr(_lib, "MAX_LM_HISTORIES", 8)
    with pytest.raises(ValueError, match="histories"):
        CharLM.fit(_words(9, 50), "abcdefgh", order=3)


def test_check_decoder_rules():
    from keras_ocr_b200.recognition import DEFAULT_ALPHABET, check_decoder
    lm = CharLM.fit(["abc"], DEFAULT_ALPHABET, order=2)
    assert check_decoder(4, 2, None, DEFAULT_ALPHABET, lm) is None
    with pytest.raises(ValueError, match="a language model needs beam search: pass beam_width"):
        check_decoder(None, 1, None, DEFAULT_ALPHABET, lm)
    with pytest.raises(ValueError, match="mutually exclusive"):
        check_decoder(None, 1, ["abc"], DEFAULT_ALPHABET, lm)
    with pytest.raises(ValueError, match="alphabet"):
        check_decoder(4, 1, None, "abc", lm)
    with pytest.raises(ValueError, match="top_paths"):
        check_decoder(4, 5, None, DEFAULT_ALPHABET, lm)
    with pytest.raises(ValueError, match="CharLM"):
        check_decoder(4, 1, None, DEFAULT_ALPHABET, "not a model")
