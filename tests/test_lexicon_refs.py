"""CPU: the fp64 lexicon references of tests/lexicon_refs.py, the validation of ``Lexicon`` / ``check_decoder``, and the
lexicon option of the records path through a world-size-2 gloo group."""
import itertools
import multiprocessing as mp
import os
import socket

import numpy as np
import pytest
import torch.distributed as dist

from keras_ocr_b200 import distributed as D
from tests import beam_refs as BR
from tests import lexicon_refs as LR


def _random_lp(rng, t, k, temperature=1.0):
    return BR.log_probs(rng.normal(size=(t, k)) / temperature)


def _random_entries(rng, k, n, hi=12):
    out = set()
    while len(out) < n:
        e = tuple(int(c) for c in rng.integers(0, k - 1, int(rng.integers(1, hi + 1))))
        if len(e) >= 2 and rng.random() < 0.3:
            e = e[:1] + e[:1] + e[2:]                             # a doubled letter
        out.add(e)
    return sorted(out)


# ------------------------------------------------------------------------------------------ 1. the reference
def test_scores_equal_brute_force():
    rng = np.random.default_rng(0)
    for t, k in [(3, 3), (5, 3), (6, 3), (5, 4)]:
        lp = _random_lp(rng, t, k)
        exact = BR.brute_force(lp)
        entries = [e for n in range(1, t + 2) for e in itertools.product(range(k - 1), repeat=n)]
        for got in (LR.scores(lp, entries), LR.scores_many(lp, entries)):
            for e, v in zip(entries, got):
                if e in exact:
                    assert v == pytest.approx(exact[e], rel=1e-12, abs=1e-12), e
                else:                                             # not reachable in t steps
                    assert v == -np.inf and not LR.alignable(e, t), e


def test_scores_many_equals_forward_logprob():
    rng = np.random.default_rng(1)
    for k, temperature in [(3, 1.0), (37, 0.3), (37, 3.0), (301, 1.0)]:
        lp = _random_lp(rng, 48, k, temperature)
        entries = _random_entries(rng, k, 200, hi=30)
        np.testing.assert_allclose(LR.scores_many(lp, entries), LR.scores(lp, entries), rtol=1e-12, atol=1e-9)


def test_unalignable_is_exactly_minus_inf_and_hopeless_is_finite():
    lp = BR.log_probs(np.zeros((48, 37)))
    lp_peaked = BR.log_probs(np.where(np.arange(37) == 36, 40.0, 0.0) * np.ones((48, 1)))   # blank is certain
    entries = [(0,) * 25, (0,) * 24, (0, 1) * 24, (0,) * 2 + (1,) * 23, (5,) * 48, (1, 2) * 24 + (3,)]
    expect_finite = [False, True, True, True, False, False]
    for table in (LR.scores(lp, entries), LR.scores_many(lp, entries), LR.scores_many(lp_peaked, entries)):
        assert [bool(np.isfinite(v)) for v in table] == expect_finite
        assert all(v == -np.inf for v, f in zip(table, expect_finite) if not f)
    hopeless = LR.scores_many(lp_peaked, [(0, 1) * 24])[0]       # every step pays about log(1e-7 / (1 + 37e-7))
    assert -800 < hopeless < -700


def test_scores_do_not_depend_on_the_rest_of_the_lexicon():
    rng = np.random.default_rng(2)
    lp = _random_lp(rng, 48, 37, 0.5)
    entries = _random_entries(rng, 37, 300)
    base = LR.scores_many(lp, entries)
    perm = rng.permutation(len(entries))
    shuffled = LR.scores_many(lp, [entries[i] for i in perm])
    assert np.array_equal(shuffled, base[perm])                  # bit for bit
    extended = LR.scores_many(lp, entries + _random_entries(np.random.default_rng(3), 37, 500, hi=40))
    assert np.array_equal(extended[:len(entries)], base)
    idx, top, _ = LR.top_entries(base, 10)
    idx_s, top_s, _ = LR.top_entries(shuffled, 10)
    assert [entries[i] for i in idx] == [entries[perm[i]] for i in idx_s] and np.array_equal(top, top_s)


def test_ties_rank_by_index():
    lp = BR.log_probs(np.zeros((48, 5)))                          # uniform: entries of one shape score alike
    entries = [(3,), (0,), (2,), (1,)]
    ref = LR.scores(lp, entries)
    assert ref[0] == ref[1] == ref[2] == ref[3]
    idx, _, info = LR.top_entries(ref, 4)
    assert list(idx) == [0, 1, 2, 3] and info["ties"] == 3
    idx, _, _ = LR.top_entries(np.array([-1.0, -np.inf, -1.0, -0.5]), 5)
    assert list(idx) == [3, 0, 2]                                 # -inf entries are never returned


# ------------------------------------------------------------------------------------------ 2. validation
def test_lexicon_compiles_to_csr():
    from keras_ocr_b200.recognition import Lexicon
    lex = Lexicon(["ab", "z", "0a0"])
    assert lex.offsets.dtype == np.int32 and lex.labels.dtype == np.int16
    assert lex.offsets.tolist() == [0, 2, 3, 6]
    assert lex.labels.tolist() == [10, 11, 35, 0, 10, 0]
    assert len(lex) == 3 and Lexicon(("ab",)).words == ("ab",)


BAD_LEXICONS = [([], "empty"), (["ab", ""], "entry 1"), (["a" * 49], "entry 0"), (["ab", "aB"], "entry 1"),
                (["ab", "cd", "ab"], "entry 2"), ("abc", "list"), (["ab", 3], "entry 1")]


@pytest.mark.parametrize("words,where", BAD_LEXICONS)
def test_lexicon_rejects(words, where):
    from keras_ocr_b200.recognition import Lexicon, check_decoder
    with pytest.raises(ValueError, match=where):
        Lexicon(words)
    with pytest.raises(ValueError, match=where):
        check_decoder(lexicon=words)


def test_lexicon_size_limits():
    from keras_ocr_b200.recognition import Lexicon
    with pytest.raises(ValueError, match="at most"):
        Lexicon(["a"] * ((1 << 20) + 1))
    Lexicon(["a" * 48])                                           # 48 characters is the longest entry


def test_check_decoder():
    from keras_ocr_b200.recognition import DEFAULT_ALPHABET, Lexicon, check_decoder
    assert check_decoder() is None and check_decoder(beam_width=5, top_paths=2) is None
    lex = Lexicon(["ab", "cd"])
    assert check_decoder(lexicon=lex) is lex
    assert check_decoder(lexicon=["ab", "cd"], top_paths=128).words == ("ab", "cd")
    assert check_decoder(lexicon=("ab",), top_paths=np.int64(3)).words == ("ab",)
    for kw in (dict(beam_width=5), dict(beam_width=5, top_paths=2), dict(top_paths=0), dict(top_paths=129),
               dict(top_paths=2.0), dict(top_paths=True)):
        with pytest.raises(ValueError):
            check_decoder(lexicon=lex, **kw)
    with pytest.raises(ValueError, match="alphabet"):
        check_decoder(lexicon=Lexicon(["ab"], alphabet="abc"), alphabet=DEFAULT_ALPHABET)
    with pytest.raises(ValueError):
        check_decoder(top_paths=2)                               # no lexicon: check_beam's rules


def _unlaunchable():
    """This package's Pipeline, Detector and Recognizer without a device (any launch would fail)."""
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    from keras_ocr_b200.recognition import DEFAULT_ALPHABET, Recognizer
    pipe = Pipeline.__new__(Pipeline)
    pipe.detector, pipe.recognizer = Detector.__new__(Detector), Recognizer.__new__(Recognizer)
    pipe.recognizer.alphabet = DEFAULT_ALPHABET
    pipe.gpu_decode = False
    return pipe


BAD_CALLS = [dict(lexicon=["ab"], beam_width=5), dict(lexicon=["ab"], top_paths=129), dict(lexicon=[]),
             dict(lexicon=["ab", "ab"]), dict(lexicon=["a-b"])]


@pytest.mark.parametrize("kw", BAD_CALLS)
def test_recognizer_and_pipeline_reject_before_launch(kw):
    from keras_ocr_b200.recognition import Lexicon
    pipe = _unlaunchable()
    rec = pipe.recognizer
    images = np.zeros((1, 32, 32, 3), np.uint8)
    with pytest.raises(ValueError):
        rec.recognize_crops(np.zeros((1, 31, 200), np.uint8), **kw)
    with pytest.raises(ValueError):
        rec.recognize_from_boxes([images[0]], [np.zeros((1, 4, 2), np.float32)], **kw)
    with pytest.raises(ValueError):
        rec.predict_device(None, **kw)
    with pytest.raises(ValueError):
        pipe.recognize(images, recognition_kwargs=kw)
    with pytest.raises(ValueError, match="alphabet"):
        rec.predict_device(None, lexicon=Lexicon(["ab"], alphabet="abc"))


@pytest.mark.parametrize("kw", BAD_CALLS + [dict(lexicon=["ab"], top_paths=2)])
def test_records_paths_reject_before_launch(kw):
    pipe = _unlaunchable()
    images = np.zeros((1, 32, 32, 3), np.uint8)
    with pytest.raises(ValueError):
        pipe.recognize_records(images, **kw)
    with pytest.raises(ValueError):
        D.recognize_sharded(pipe, images, **kw)
    with pytest.raises(ValueError):
        D.ShardedStream(pipe, **kw)


# ------------------------------------------------------------------------------------------ 3. gloo, world size 2
class _FakeStage:
    device = None
    alphabet = "0123456789abcdefghijklmnopqrstuvwxyz"


def _words(images, lexicon):
    """Stands in for the GPU: image v reads as v % 4 words of the lexicon, picked by the image content."""
    out = []
    for im in images:
        v = int(im[0, 0, 0])
        out.append([(lexicon.words[(v + j) % len(lexicon)], np.full((4, 2), float(v) + j, np.float32))
                    for j in range(v % 4)])
    return out


class _FakeLexiconPipeline:
    """``recognize`` only: the lexicon arrives compiled, in ``recognition_kwargs``."""
    detector = _FakeStage()
    recognizer = _FakeStage()

    def recognize(self, images, recognition_kwargs=None):
        from keras_ocr_b200.recognition import Lexicon
        lexicon = recognition_kwargs["lexicon"]
        assert isinstance(lexicon, Lexicon)
        return _words(images, lexicon)


class _FakeLexiconRecordsPipeline(_FakeLexiconPipeline):
    """records_begin / records_end like the real Pipeline; the lexicon arrives in records_begin."""

    def records_begin(self, images, rows=None, rec_boxes=128, lexicon=None):
        return {"images": images, "rows": rows, "rec_boxes": rec_boxes, "lexicon": lexicon}

    def records_counts(self, state):
        return [len(g) for g in _words(state["images"], state["lexicon"])]

    def records_end(self, state, rec_boxes=None):
        return D._host_records(self, _words(state["images"], state["lexicon"]), state["rows"],
                               state["rec_boxes"] if rec_boxes is None else rec_boxes)

    def recognize_records(self, images, rows=None, rec_boxes=128, lexicon=None):
        return self.records_end(self.records_begin(images, rows, rec_boxes, lexicon))


LEXICON = ["cat", "dog", "b00k", "zz9"]


def _lexicon_worker(rank, world, port, images, ret, records, stream, as_list):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from keras_ocr_b200.recognition import Lexicon
        pipe = _FakeLexiconRecordsPipeline() if records else _FakeLexiconPipeline()
        lexicon = list(LEXICON) if as_list else Lexicon(LEXICON)
        if stream:
            s = D.ShardedStream(pipe, max_boxes=8, lexicon=lexicon)
            outs = [s.submit(images[rank * 3:(rank + 1) * 3]), s.flush()]
            res = outs[1]
            if rank == 0:
                assert outs[0] is None
        else:
            res = D.recognize_sharded(pipe, images, max_boxes=8, lexicon=lexicon)
        if rank == 0:
            ret.put([[(t, b.tolist()) for t, b in g] for g in res])
        else:
            assert res is None
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("records,stream,as_list", [(False, False, True), (True, False, False), (False, True, False),
                                                    (True, True, True)])
def test_lexicon_through_the_sharded_paths(records, stream, as_list):
    from keras_ocr_b200.recognition import Lexicon
    images = np.zeros((6, 4, 4, 3), np.uint8)
    images[:, 0, 0, 0] = np.arange(6) + 1
    s = socket.socket(); s.bind(("127.0.0.1", 0)); port = s.getsockname()[1]; s.close()
    ctx = mp.get_context("spawn")
    ret = ctx.Queue()
    procs = [ctx.Process(target=_lexicon_worker, args=(r, 2, port, images, ret, records, stream, as_list))
             for r in range(2)]
    for p in procs:
        p.start()
    got = ret.get(timeout=120)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    expect = [[(t, b.tolist()) for t, b in g] for g in _words(images, Lexicon(LEXICON))]
    assert got == expect and all(t in LEXICON for g in got for t, _ in g)
