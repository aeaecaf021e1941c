"""CPU: the hotword trie (``recognition.compile_trie``) against a dict trie, the fp64 reference search of
tests/hotword_refs.py against brute force and against plain and LM-fused beam search, and hotword validation."""
import itertools

import numpy as np
import pytest

from keras_ocr_b200 import _lib
from keras_ocr_b200.pipeline import check_records_decoder
from keras_ocr_b200.recognition import CharLM, Hotwords, Lexicon, check_decoder, check_hotwords, check_pattern
from tests import beam_refs as BR
from tests import hotword_refs as HR
from tests import lm_refs as LR


def _words(seed, n, alphabet="abcdefgh", lo=1, hi=7):
    rng = np.random.default_rng(seed)
    out = {"".join(rng.choice(list(alphabet), int(rng.integers(lo, hi + 1)))) for _ in range(n)}
    return sorted(out)


@pytest.mark.parametrize("seed", range(4))
def test_trie_matches_a_dict_trie(seed):
    words = _words(seed, 60 + 40 * seed)
    hw = Hotwords(words, alphabet="abcdefgh")
    keys, child, final = hw.host_tables()
    nodes, fin = HR.dict_trie(HR.encode(words, "abcdefgh"))
    assert keys.dtype == np.uint64 and child.dtype == np.int32 and final.dtype == np.uint8
    assert len(final) == len(nodes) and len(keys) == len(child) == len(nodes) - 1
    assert np.all(keys[1:] > keys[:-1])                                  # sorted, distinct
    parent, label = (keys >> np.uint64(8)).astype(np.int64), (keys & np.uint64(255)).astype(np.int64)
    got = {int(c): (int(p), int(lab)) for p, lab, c in zip(parent, label, child)}
    assert got == {i: (p, c) for i, (p, c, _) in enumerate(nodes) if i}
    assert final.tolist() == [int(f) for f in fin]
    for u in range(len(nodes)):                                          # children contiguous, by label
        at = np.flatnonzero(parent == u)
        if at.size:
            assert np.array_equal(at, np.arange(at[0], at[-1] + 1))
            assert np.all(np.diff(label[at]) > 0)
    assert final.sum() == len(words) and final[0] == 0


def test_trie_is_deterministic_and_empty_list_is_the_root():
    words = _words(9, 300)
    a = Hotwords(words, alphabet="abcdefgh").host_tables()
    b = Hotwords(list(reversed(words)), alphabet="abcdefgh").host_tables()
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    keys, child, final = Hotwords([], alphabet="abcdefgh").host_tables()
    assert keys.size == 0 and child.size == 0 and final.tolist() == [0]
    # a hand-checked trie: "ab", "a", "b", "abc", "ba" -> nodes a=1, b=2, ab=3, ba=4, abc=5
    keys, child, final = Hotwords(["ab", "a", "b", "abc", "ba"], alphabet="abc").host_tables()
    assert keys.tolist() == [0, 1, (1 << 8) | 1, (2 << 8) | 0, (3 << 8) | 2]
    assert child.tolist() == [1, 2, 3, 4, 5] and final.tolist() == [0, 1, 1, 1, 1, 1]


def test_weighted_shares_the_trie():
    hw = Hotwords(["ab"], alphabet="ab", weight=2.0)
    other = hw.weighted(0.5)
    assert other.weight == 0.5 and hw.weight == 2.0 and other.host_tables() is hw.host_tables()


def _model():
    lm = CharLM.fit(["ab", "ba", "aab", "b", "bba"], "ab", order=3)
    keys, rows = lm.host_tables()
    return {"keys": keys, "rows": rows, "order": 3, "alpha": 0.7, "beta": 0.3}


@pytest.mark.parametrize("with_model", [False, True])
@pytest.mark.parametrize("gamma", [0.4, 1.5, 4.0])
def test_reference_finds_the_exhaustive_maximiser(with_model, gamma):
    """With W at least the number of prefixes nothing is pruned: the best reading maximises F_end over every label
    sequence of nonzero probability, whatever the bonus did during the search."""
    model = _model() if with_model else {}
    rng = np.random.default_rng(11)
    for i in range(6):
        T = 4
        lp = BR.log_probs(rng.normal(size=(T, 3)) * 2)
        seqs = HR.encode([["ab", "bab"], ["a", "bb", "aba"], ["b"]][i % 3], "ab")
        paths, a, fend, _ = HR.beam_search_hot(lp, 64, seqs, gamma, top_paths=1, **model)
        best, f = HR.exhaustive_best(lp, seqs, gamma, **model)
        assert paths[0] == best
        assert abs(fend[0] - f) < 1e-9
        assert abs(a[0] - BR.forward_logprob(lp, best)) < 1e-9


def test_reference_with_zero_weight_or_no_words_is_the_plain_and_lm_search():
    model = _model()
    rng = np.random.default_rng(0)
    for i in range(6):
        lp = BR.log_probs(rng.normal(size=(12, 3)) * (3 if i % 2 else 1))
        for w in (1, 3, 8):
            for seqs, gamma in ((HR.encode(["ab", "ba"], "ab"), 0.0), ([], 2.0)):
                paths, a, fend, _ = HR.beam_search_hot(lp, w, seqs, gamma)
                ref, score, _ = BR.beam_search(lp, w)
                assert paths == ref and np.array_equal(a, score) and np.array_equal(fend, score)
                paths, a, fend, _ = HR.beam_search_hot(lp, w, seqs, gamma, **model)
                rp, ra, rf, _ = LR.beam_search_lm(lp, w, model["keys"], model["rows"], 3, 0.7, 0.3)
                assert paths == rp and np.array_equal(a, ra) and np.array_equal(fend, rf)


def test_bonus_is_withdrawn_outside_the_list():
    """A reading that left the trie, or a live prefix that is not a word, ends with no bonus: F_end = A there."""
    rng = np.random.default_rng(5)
    seqs = HR.encode(["abab"], "ab")
    for _ in range(5):
        lp = BR.log_probs(rng.normal(size=(8, 3)))
        paths, a, fend, _ = HR.beam_search_hot(lp, 16, seqs, 1.0)
        for p, ai, fi in zip(paths, a, fend):
            assert fi == (ai + HR.bonus(1.0, 4) if p == (0, 1, 0, 1) else ai)


def test_hotwords_value_errors():
    with pytest.raises(ValueError, match="list or tuple"):
        Hotwords("ab", alphabet="ab")
    with pytest.raises(ValueError, match=r"hotword 1 \(''\)"):
        Hotwords(["ab", ""], alphabet="ab")
    with pytest.raises(ValueError, match=r"hotword 0 \('ax'\) has 'x'"):
        Hotwords(["ax"], alphabet="ab")
    with pytest.raises(ValueError, match="longer than 48"):
        Hotwords(["a" * 49], alphabet="ab")
    with pytest.raises(ValueError, match=r"hotword 2 \('ab'\) is a duplicate"):
        Hotwords(["ab", "b", "ab"], alphabet="ab")
    with pytest.raises(ValueError, match="at most 126"):
        Hotwords(["a"], alphabet="".join(chr(0x100 + i) for i in range(127)))
    for bad in (-0.5, float("inf"), float("nan"), 1e39, True, "1", None):
        with pytest.raises(ValueError, match="weight"):
            Hotwords(["ab"], weight=bad, alphabet="ab")
    with pytest.raises(ValueError, match="weight"):
        Hotwords(["ab"], alphabet="ab").weighted(-1.0)


def test_hotwords_size_limits(monkeypatch):
    monkeypatch.setattr(_lib, "MAX_LEXICON_WORDS", 3)
    with pytest.raises(ValueError, match="at most 3"):
        Hotwords(["a", "b", "ab", "ba"], alphabet="ab")
    monkeypatch.setattr(_lib, "MAX_LEXICON_WORDS", 1 << 20)
    monkeypatch.setattr(_lib, "MAX_LEXICON_LABELS", 5)
    with pytest.raises(ValueError, match=r"hotword 2 \('aba'\) takes the list past 5"):
        Hotwords(["ab", "b", "aba"], alphabet="ab")


def test_check_decoder_rules():
    alpha = "0123456789abcdefghijklmnopqrstuvwxyz"
    lm = CharLM.fit(["ab", "ba"], alpha, order=2)
    assert check_decoder(4, 1, None, alpha, None, None, ["ab"]) is None
    assert check_decoder(4, 2, None, alpha, lm, hotwords=["ab"]) is None
    hw = check_hotwords(["ab", "cd"], 4, 1, None, alpha)
    assert isinstance(hw, Hotwords) and hw.words == ("ab", "cd") and hw.weight == Hotwords.WEIGHT
    assert check_hotwords(hw, 4, 1, None, alpha) is hw
    assert check_hotwords(None, None) is None
    with pytest.raises(ValueError, match="beam search"):
        check_decoder(None, 1, None, alpha, None, None, ["ab"])
    with pytest.raises(ValueError, match="lexicon and hotwords"):
        check_decoder(4, 1, ["ab"], alpha, None, None, ["ab"])
    with pytest.raises(ValueError, match="lexicon and hotwords"):
        check_hotwords(["ab"], 4, 1, Lexicon(["ab"], alpha), alpha)
    with pytest.raises(ValueError, match="pattern and hotwords"):
        check_decoder(4, 1, None, alpha, None, "ab", ["ab"])
    with pytest.raises(ValueError, match="pattern and hotwords"):
        check_pattern("ab", 4, 1, None, alpha, None, ["ab"])
    with pytest.raises(ValueError, match="another alphabet"):
        check_decoder(4, 1, None, alpha, None, None, Hotwords(["ab"], alphabet="ab"))
    with pytest.raises(ValueError, match="Hotwords or a list"):
        check_decoder(4, 1, None, alpha, None, None, "ab")
    with pytest.raises(ValueError, match="top_paths"):
        check_decoder(4, 5, None, alpha, None, None, ["ab"])
    with pytest.raises(ValueError, match="another alphabet"):
        check_decoder(4, 1, None, alpha, CharLM.fit(["ab"], "ab", order=2), None, ["ab"])
    # the records path carries one reading per word
    assert check_records_decoder(4, 1, None, alpha, lm, None, ["ab"]) is None
    with pytest.raises(ValueError, match="top_paths must be 1"):
        check_records_decoder(4, 2, None, alpha, None, None, ["ab"])
    with pytest.raises(ValueError, match="beam search"):
        check_records_decoder(None, 1, None, alpha, None, None, ["ab"])


def test_trie_of_many_words_is_compact():
    words = ["".join(p) for p in itertools.product("abcd", repeat=5)]          # 1024 words, every prefix shared
    keys, child, final = Hotwords(words, alphabet="abcd").host_tables()
    assert len(final) == sum(4 ** d for d in range(6)) and int(final.sum()) == 1024
