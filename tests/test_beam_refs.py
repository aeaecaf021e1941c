"""CPU: the fp64 beam-search references of tests/beam_refs.py, and the argument checks of the beam-search options."""
import numpy as np
import pytest
import torch

from tests import beam_refs as BR


def _random_lp(rng, t, k, temperature=1.0):
    return BR.log_probs(rng.normal(size=(t, k)) / temperature)


# ------------------------------------------------------------------------------------------ 1. exact sequence logp
def test_forward_logprob_equals_ctc_loss():
    rng = np.random.default_rng(0)
    for t, k in [(48, 37), (48, 3), (20, 301), (12, 5)]:
        lp = _random_lp(rng, t, k, 0.7)
        for length in (0, 1, 3, 7):
            labels = rng.integers(0, k - 1, length)
            if length >= 3:
                labels[1] = labels[0]                             # a doubled letter needs a blank between
            loss = torch.nn.functional.ctc_loss(torch.from_numpy(lp)[:, None, :], torch.from_numpy(labels)[None].long(),
                                                torch.tensor([t]), torch.tensor([length]), blank=k - 1,
                                                reduction="none")
            assert BR.forward_logprob(lp, labels) == pytest.approx(-float(loss[0]), rel=1e-12, abs=1e-12)


def test_forward_logprob_equals_brute_force():
    rng = np.random.default_rng(1)
    for t, k in [(1, 2), (3, 3), (5, 4), (6, 3), (6, 4)]:
        lp = _random_lp(rng, t, k)
        exact = BR.brute_force(lp)
        for seq, v in exact.items():
            assert BR.forward_logprob(lp, seq) == pytest.approx(v, rel=1e-12, abs=1e-12), seq
        # the distributions sum to the mass of the floored softmax, (1 + K 1e-7)^T
        assert np.logaddexp.reduce(list(exact.values())) == pytest.approx(t * np.log1p(k * 1e-7), abs=1e-12)


# ------------------------------------------------------------------------------------------ 2. the reference beam search
def test_beam_without_pruning_is_exact():
    """W above the number of distinct prefixes: nothing is pruned, so the P paths are the P most probable sequences."""
    rng = np.random.default_rng(2)
    for t, k in [(4, 3), (5, 3), (6, 3), (4, 4), (5, 4)]:
        for temperature in (0.3, 1.0, 3.0):
            lp = _random_lp(rng, t, k, temperature)
            best = BR.ranked(BR.brute_force(lp))
            paths, logp, _ = BR.beam_search(lp, 128, top_paths=20)
            assert paths == [s for s, _ in best[:20]]
            np.testing.assert_allclose(logp, [v for _, v in best[:20]], rtol=0, atol=1e-12)


def test_beam_peaked_top1_is_greedy():
    rng = np.random.default_rng(3)
    for k in (3, 37, 301):
        for w in (1, 2, 5, 100):
            logits = rng.normal(size=(48, k))
            arg = rng.integers(0, k, 48)
            arg[5:9] = arg[4]                                     # runs of one label collapse
            logits[np.arange(48), arg] += 30.0
            paths, logp, _ = BR.beam_search(BR.log_probs(logits), w, top_paths=1)
            assert paths[0] == BR.collapse(arg, k - 1)
            assert logp[0] <= 1e-5


def test_beam_uniform_follows_the_tie_rule():
    for t, k, w in [(4, 3, 128), (5, 4, 128), (6, 3, 4), (6, 4, 7), (48, 37, 10)]:
        lp = BR.log_probs(np.zeros((t, k)))
        paths, logp, info = BR.beam_search(lp, w)
        assert info["ties"] > 0
        for i in range(len(paths) - 1):                          # equal scores: ascending label sequence
            assert logp[i] > logp[i + 1] or (logp[i] == logp[i + 1] and paths[i] < paths[i + 1])
        if t <= 6 and w == 128:
            # sequences of different shapes can have equal exact probabilities (e.g. "0" and "00" for T = 5, K = 4);
            # their fp64 sums then differ in the last bits and rank by those, so only the values are compared here
            exact = BR.brute_force(lp)
            np.testing.assert_allclose(logp, [exact[p] for p in paths], rtol=0, atol=1e-12)
            np.testing.assert_allclose(logp, sorted(exact.values(), reverse=True)[:len(paths)], rtol=0, atol=1e-12)


def test_beam_paths_distinct_and_non_increasing():
    rng = np.random.default_rng(4)
    for k, w in [(3, 5), (37, 10), (37, 100), (301, 20), (1024, 128)]:
        lp = _random_lp(rng, 48, k, 0.5)
        paths, logp, info = BR.beam_search(lp, w)
        assert len(paths) == len(set(paths)) == min(w, len(paths))
        assert np.all(np.diff(logp) <= 0)
        for p, v in zip(paths[:3], logp[:3]):                    # a beam score is a lower bound of the exact logp
            assert v <= BR.forward_logprob(lp, p) + 1e-9
        assert info["prune_margin"] > 0


# ------------------------------------------------------------------------------------------ 3. argument checks
BAD = [dict(beam_width=0), dict(beam_width=129), dict(beam_width=2.0), dict(beam_width=True),
       dict(beam_width=5, top_paths=6), dict(beam_width=5, top_paths=0), dict(top_paths=2)]


@pytest.mark.parametrize("kw", BAD)
def test_check_beam_rejects(kw):
    from keras_ocr_b200 import recognition
    with pytest.raises(ValueError):
        recognition.check_beam(**kw)


def test_check_beam_accepts():
    from keras_ocr_b200 import recognition
    for kw in (dict(), dict(beam_width=1), dict(beam_width=128, top_paths=128), dict(beam_width=np.int64(10))):
        recognition.check_beam(**kw)


def _unlaunchable():
    """This package's Pipeline, Detector and Recognizer without a device: any launch would fail, so a ValueError
    shows that the arguments were refused first."""
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    from keras_ocr_b200.recognition import Recognizer
    pipe = Pipeline.__new__(Pipeline)
    pipe.detector, pipe.recognizer = Detector.__new__(Detector), Recognizer.__new__(Recognizer)
    pipe.gpu_decode = False
    return pipe


@pytest.mark.parametrize("kw", BAD)
def test_recognizer_and_pipeline_reject_before_launch(kw):
    pipe = _unlaunchable()
    rec = pipe.recognizer
    crops = np.zeros((1, 31, 200), np.uint8)
    images = np.zeros((1, 32, 32, 3), np.uint8)
    with pytest.raises(ValueError):
        rec.recognize_crops(crops, **kw)
    with pytest.raises(ValueError):
        rec.recognize_from_boxes([images[0]], [np.zeros((1, 4, 2), np.float32)], **kw)
    with pytest.raises(ValueError):
        rec.predict_device(None, **kw)
    with pytest.raises(ValueError):
        pipe.recognize(images, recognition_kwargs=kw)


@pytest.mark.parametrize("kw", BAD + [dict(beam_width=5, top_paths=2)])
def test_records_paths_reject_before_launch(kw):
    from keras_ocr_b200 import distributed as D
    pipe = _unlaunchable()
    images = np.zeros((1, 32, 32, 3), np.uint8)
    with pytest.raises(ValueError):
        pipe.recognize_records(images, **kw)
    with pytest.raises(ValueError):
        D.recognize_sharded(pipe, images, **kw)
    with pytest.raises(ValueError):
        D.ShardedStream(pipe, **kw)
