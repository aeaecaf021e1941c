"""CPU: the pattern compiler (``keras_ocr_b200.patterns``, ``recognition.Pattern``) against Python's ``re``, the
properties of its automata, its errors, the validation of ``pattern=``, and the fp64 reference search of
tests/pattern_refs.py against plain beam search and brute force."""
import re

import numpy as np
import pytest

from keras_ocr_b200.recognition import DEFAULT_ALPHABET, Pattern
from tests import beam_refs as BR
from tests import pattern_refs as PR

ALPHABETS = (DEFAULT_ALPHABET, "ab", "abc", "0a1b")


def _walk(rng, pat, max_len=12):
    """A string spelt by a random walk of the DFA from its start, stopped at an accepting state or a dead end."""
    q, out = pat.start, []
    for _ in range(max_len):
        if pat.dist[q] == 0 and rng.random() < 0.3:
            break
        nxt = np.nonzero(pat.trans[q] >= 0)[0]
        if nxt.size == 0:
            break
        c = int(rng.choice(nxt))
        out.append(pat.alphabet[c])
        q = int(pat.trans[q, c])
    return "".join(out)


def _mutations(rng, s, alphabet, n=3):
    out = []
    for _ in range(n):
        kind = rng.integers(3)
        i = int(rng.integers(len(s) + 1))
        ch = alphabet[int(rng.integers(len(alphabet)))]
        if kind == 0:
            out.append(s[:i] + ch + s[i:])
        elif s and kind == 1:
            i = min(i, len(s) - 1)
            out.append(s[:i] + s[i + 1:])
        elif s:
            i = min(i, len(s) - 1)
            out.append(s[:i] + ch + s[i + 1:])
    return out


@pytest.mark.parametrize("alphabet", ALPHABETS)
def test_compiler_matches_re_fullmatch(alphabet):
    rng = np.random.default_rng(len(alphabet))
    compiled = checked = 0
    for _ in range(150):
        text = PR.random_pattern(rng, alphabet, depth=int(rng.integers(1, 5)))
        try:
            pat = Pattern(text, alphabet)
        except ValueError as e:                                   # only the size and length limits may refuse these
            assert "states" in str(e) or "longer than" in str(e), (text, str(e))
            continue
        compiled += 1
        rx = re.compile(text)
        strings = ["".join(rng.choice(list(alphabet), size=int(rng.integers(0, 10)))) for _ in range(20)]
        strings += [_walk(rng, pat) for _ in range(20)]
        strings += [m for s in list(strings) for m in _mutations(rng, s, alphabet, 1)]
        for s in strings:
            assert pat.fullmatch(s) == bool(rx.fullmatch(s)), (text, s)
            checked += 1
        assert not pat.fullmatch("\n" + "A")                     # outside the alphabet: never accepted
    assert compiled >= 120 and checked > 10000


def _moore_classes(trans, final):
    cls = final.astype(np.int64)
    while True:
        succ = np.where(trans >= 0, cls[np.maximum(trans, 0)], -1)
        _, new = np.unique(np.concatenate([cls[:, None], succ], 1), axis=0, return_inverse=True)
        new = new.reshape(-1)
        if new.max() == cls.max() and len(np.unique(new)) == len(np.unique(cls)):
            return new
        cls = new


@pytest.mark.parametrize("seed", range(6))
def test_dfa_is_minimal_trimmed_and_dist_is_a_bfs(seed):
    rng = np.random.default_rng(100 + seed)
    done = 0
    while done < 25:
        alphabet = ALPHABETS[int(rng.integers(len(ALPHABETS)))]
        try:
            pat = Pattern(PR.random_pattern(rng, alphabet), alphabet)
        except ValueError:
            continue
        done += 1
        trans, dist, start = pat.host_tables()
        n = pat.n_states
        assert trans.dtype == np.int16 and trans.shape == (n, len(alphabet)) and dist.dtype == np.uint8
        assert start == 0 and trans.min() >= -1 and trans.max() < n
        assert len(np.unique(_moore_classes(trans.astype(np.int64), dist == 0))) == n   # nothing merges
        seen, todo = {start}, [start]                            # every state reachable
        while todo:
            q = todo.pop()
            for t in trans[q][trans[q] >= 0]:
                if int(t) not in seen:
                    seen.add(int(t))
                    todo.append(int(t))
        assert len(seen) == n
        want = np.full(n, -1)                                    # dist: BFS backwards from the accepting states
        want[dist == 0] = 0
        frontier, d = set(np.nonzero(dist == 0)[0].tolist()), 0
        while frontier:
            d += 1
            nxt = set()
            for q in range(n):
                if want[q] < 0 and any(int(t) in frontier for t in trans[q] if t >= 0):
                    want[q] = d
                    nxt.add(q)
            frontier = nxt
        assert (want >= 0).all()                                  # every state co-reachable
        assert np.array_equal(np.minimum(want, 255), dist)


def test_compilation_is_deterministic():
    for text in ("[a-z]{3}[0-9]{4}", "(inv|crn)[0-9]{2,6}", "(a|b)*abb(a|b)?"):
        a, b = Pattern(text), Pattern(text)
        assert all(np.array_equal(x, y) for x, y in zip(a.host_tables()[:2], b.host_tables()[:2]))


def test_hand_cases():
    p = Pattern("[a-z]{3}[0-9]{4}")
    assert p.n_states == 8 and p.dist[p.start] == 7
    assert p.fullmatch("abc1234") and not p.fullmatch("abc123") and not p.fullmatch("ab01234")
    assert Pattern(".*").n_states == 1 and Pattern(".*").dist[0] == 0
    assert Pattern("").fullmatch("") and not Pattern("").fullmatch("a")
    assert Pattern("\\d+").fullmatch("0123") and not Pattern("\\d+").fullmatch("")
    assert Pattern("[^0-9]").fullmatch("q") and not Pattern("[^0-9]").fullmatch("7")
    assert Pattern("a\\.b|c", "abc.").fullmatch("a.b") and not Pattern("a\\.b|c", "abc.").fullmatch("axb")
    assert Pattern("[]a]", "a]").fullmatch("]")


@pytest.mark.parametrize("text, pos", [
    ("^abc", 0), ("abc$", 3), ("a\\b", 1), ("(a)\\1", 3), ("(?=a)b", 1), ("(?!a)b", 1), ("(?<=a)b", 1),
    ("(?i)abc", 1), ("(?P<x>a)", 1), ("a*?", 2), ("a+?", 2), ("a{2}?", 4), ("a*+", 2), ("a**", 2),
    ("(ab", 0), ("ab)", 2), ("a(b(c)", 1), ("[b-a]", 1), ("[a-\\d]", 1), ("[abc", 0), ("A", 0), ("ab!", 2),
    ("[A-Z]", 0), ("a{2,1}", 1), ("a{49}", 1), ("a{1,49}", 1), ("*a", 0), ("a|+", 2), ("a{", 1), ("a{,3}", 1),
    ("\\w", 0), ("\\s", 0), ("\\", 0), ("[^\\d0-9a-z]", 0), ("[[:alpha:]]", 1),
])
def test_rejected_constructs_name_their_position(text, pos):
    with pytest.raises(ValueError, match=f"position {pos}:"):
        Pattern(text)


def test_limits_raise():
    with pytest.raises(ValueError, match="positions 0 to 10: every accepted reading is longer than 48"):
        Pattern("a{30}b{30}")
    with pytest.raises(ValueError, match="at most 4096 are supported"):
        Pattern("[ab]*a[ab]{12}", "ab")                          # the minimal DFA has 2^13 states
    with pytest.raises(ValueError, match=r"position \d+: the repeat expands past"):
        Pattern("((a{48}){48}){48}")
    Pattern("a{48}")                                             # at the limit
    Pattern("[ab]*a[ab]{10}", "ab")                              # 2^11 states


def test_check_pattern_rules():
    from keras_ocr_b200.recognition import CharLM, check_decoder, check_pattern
    p = Pattern("[0-9]+")
    assert check_pattern(None) is None
    assert check_pattern(p, 4, 2) is p and check_pattern("[0-9]+", 4).n_states == p.n_states
    assert check_decoder(4, 2, None, DEFAULT_ALPHABET, None, p) is None
    with pytest.raises(ValueError, match="a pattern needs beam search: pass beam_width"):
        check_pattern(p)
    with pytest.raises(ValueError, match="mutually exclusive"):
        check_pattern(p, 4, 1, ["abc"])
    with pytest.raises(ValueError, match="do not combine"):
        check_pattern(p, 4, 1, None, DEFAULT_ALPHABET, CharLM.fit(["abc"], order=2))
    with pytest.raises(ValueError, match="another alphabet"):
        check_pattern(Pattern("a+", "ab"), 4)
    with pytest.raises(ValueError, match="must be a Pattern or a str"):
        check_pattern(["[0-9]+"], 4)
    with pytest.raises(ValueError):
        check_pattern(p, 4, 5)                                   # top_paths > beam_width
    with pytest.raises(ValueError):
        check_decoder(None, 1, None, DEFAULT_ALPHABET, None, "[0-9]+")


# ------------------------------------------------------------------------------------------ the reference search
def _lp(rng, t, k, sharp=3.0):
    return BR.log_probs(rng.normal(0, sharp, (t, k)))


@pytest.mark.parametrize("k", [3, 5, 12])
def test_universal_pattern_is_plain_beam_search(k):
    rng = np.random.default_rng(k)
    alphabet = "abcdefghijklmnop"[:k - 1]
    u = Pattern(".*", alphabet)
    for w in (1, 3, 8, 32):
        for _ in range(4):
            lp = _lp(rng, 12, k)
            a, sa, ia = PR.beam_search_pattern(lp, w, *u.host_tables())
            b, sb, ib = BR.beam_search(lp, w)
            assert a == b and np.array_equal(sa, sb) and ia == ib


@pytest.mark.parametrize("k, t", [(3, 5), (4, 4)])
def test_reference_finds_the_most_probable_matching_labelling(k, t):
    """With W large enough to keep every prefix, the best reading is the most probable labelling that matches."""
    rng = np.random.default_rng(10 * k + t)
    alphabet = "abc"[:k - 1]
    texts = ["a+", "ab*", "(ab)+", "b?a?b", "[ab]{2}", "", "a{2}", "ba|ab", ".*b"]
    for trial in range(6):
        lp = _lp(rng, t, k, sharp=2.0)
        brute = BR.brute_force(lp)
        for text in texts:
            pat = Pattern(text, alphabet)
            match = {s: v for s, v in brute.items() if re.fullmatch(text, "".join(alphabet[c] for c in s))}
            paths, logp, _ = PR.beam_search_pattern(lp, 10 ** 4, *pat.host_tables(), top_paths=None)
            assert all(pat.fullmatch("".join(alphabet[c] for c in s)) for s in paths)
            if not match:
                assert paths == [], (text, paths)
                continue
            want = BR.ranked(match)
            assert paths[0] == want[0][0], (text, trial, paths[:3], want[:3])
            assert abs(logp[0] - want[0][1]) < 1e-9
            assert sorted(paths) == sorted(match)                 # every matching labelling survives, no other


def test_nothing_survives_an_unreachable_pattern():
    rng = np.random.default_rng(5)
    lp = _lp(rng, 48, 5)
    paths, logp, _ = PR.beam_search_pattern(lp, 16, *Pattern("a{30}", "abcd").host_tables())
    assert paths == [] and logp.size == 0                        # 30 equal letters need 59 steps
