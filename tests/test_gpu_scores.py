"""Detection scores and word confidences on the GPU.

* Path log-probability S = sum_t log(max_c softmax(l_t)_c + 1e-7), stage by stage: the device's own ``l2`` tap gives the
  fp64 logits l = l2[:, 2:] @ w + b and from them S_ref in fp64.  The device's fp32 logits are within
  L_t = GAMMA(257) * max_c(|l2| @ |w| + |b|) of l (tests/test_gpu_crnn_stages.py), and log max softmax is 2-Lipschitz in
  the max-norm of the logits (the max moves by <= L_t, the log-sum-exp by <= L_t; the 1e-7 floor only flattens it), so
  |S_gpu - S_ref| <= sum_t (2 L_t + e_t).  e_t is the fp32 slack of the kernel's own arithmetic on its logits, u = 2^-24:
  the sum-exp of step t is built from K exponentials and at most ceil(K/32) + 5 rescalings (online per lane, then the
  five butterfly levels), each a subtraction, an expf (<= 2 ulp) and a product or sum -- at most 6u relative each, since
  the sum is >= 1 and an argument x <= 0 contributes |x| e^x u <= u / e; the reciprocal and the + 1e-7 add 2u, logf one
  ulp of the term (2u |term_t|).  The 48 terms are summed in fp32: gamma(48) * sum_t |term_t| more.
* Detection scores are exact: the max of channel 0 over the component of every box, in box order.
* C3 (256 crops, decisive weights) against the oracle's logits, C4 geometry (768 x 768 pages at scale 2) end to end.
Worst ratios to the bounds are printed; DESIGN.md section 2 records the measured ones.
"""
import math
import os

import numpy as np
import pytest
import torch

from keras_ocr_b200 import weights as W
from tests import score_refs as S, stage_refs as R

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _terms(logits):
    """Per-step log(max softmax + 1e-7) in fp64, (B,48)."""
    lg = np.asarray(logits, np.float64)
    m = lg.max(-1, keepdims=True)
    lse = np.log(np.exp(lg - m).sum(-1))
    return np.log(np.exp(-lse) + 1e-7)


def _slack(k, terms):
    """sum_t e_t + the fp32 summation of the 48 terms (module docstring), per crop."""
    per_step = 6 * U * (k + math.ceil(k / 32) + 5) + 2 * U + 2 * U * np.abs(terms)
    return per_step.sum(-1) + R.gamma(48) * np.abs(terms).sum(-1)


def _input(rec, crops):
    t = torch.from_numpy(np.ascontiguousarray(crops)).to(rec.device)
    x = torch.empty((len(crops), 200, 31), dtype=torch.float16, device=rec.device)
    rec.ctx.crops_to_input(t.data_ptr(), len(crops), x.data_ptr(), _stream())
    return x


def _crops(b, seed):
    rng = np.random.default_rng(seed)
    crops = rng.integers(0, 256, (b, 31, 200), dtype=np.uint8)
    crops[:, :, 120 + 7 * (seed % 5):] = 0
    return crops


# ------------------------------------------------------------------------------------------ 1. S, stage by stage
@pytest.mark.parametrize("k", [3, 37, 301, 1024])
def test_logp_stage_vs_fp64_from_device_l2(cuda_device, k):
    from keras_ocr_b200.recognition import Recognizer
    alphabet = "0123456789abcdefghijklmnopqrstuvwxyz" if k == 37 else (
        "ab" if k == 3 else "".join(chr(0x4E00 + i) for i in range(k - 1)))
    w = W.synthetic_crnn_weights(seed=5, alphabet=alphabet)
    rec = Recognizer(weights=w, alphabet=alphabet)
    rec.keep_workspace = True
    wk, bk = np.asarray(w["fc_12.kernel"], np.float64), np.asarray(w["fc_12.bias"], np.float64)
    worst = 0.0
    for b in (1, 7, 17):
        x = _input(rec, _crops(b, seed=k + b))
        plain = rec.predict_device(x).cpu().numpy()
        labels, logp = rec.predict_device(x, with_scores=True)
        labels, logp = labels.cpu().numpy(), logp.cpu().numpy().astype(np.float64)
        assert np.array_equal(labels, plain)                               # the scored run decodes the same labels
        l2 = rec.tap("l2", (b, 50, 256), torch.float16).double().cpu().numpy()[:, 2:]
        terms = _terms(l2 @ wk + bk)
        ref = terms.sum(-1)
        big_l = R.gamma(257) * (np.abs(l2) @ np.abs(wk) + np.abs(bk)).max(-1)   # (B,48)
        bound = (2 * big_l).sum(-1) + _slack(k, terms)
        assert np.all(np.isfinite(logp)) and np.all(logp <= 48 * np.log1p(1e-7) + 1e-6)
        r = float((np.abs(logp - ref) / bound).max())
        worst = max(worst, r)
        assert r <= 1.0, (b, r)
        if b == 17:                                                        # a crop alone == the same crop in a batch
            crops = _crops(17, seed=k + 17)
            for i in range(17):
                _, alone = rec.predict_device(_input(rec, crops[i:i + 1]), with_scores=True)
                assert alone.cpu().numpy().view(np.int32)[0] == logp.astype(np.float32).view(np.int32)[i], i
    print(f"S stage K={k}: worst |S_gpu - S_ref| / bound = {worst:.3g}")


# ------------------------------------------------------------------------------------------ 2. detection scores
@pytest.fixture(scope="module")
def detector(cuda_device):
    from keras_ocr_b200.detection import Detector
    return Detector(weights=W.synthetic_craft_weights(seed=3))


def _check_box_scores(detector, maps, **thr):
    t = torch.from_numpy(np.ascontiguousarray(maps)).to(detector.device)
    state = detector.boxes_enqueue(t, with_scores=True, **thr)
    boxes, counts = detector.boxes_finish(state)
    got = state["box_scores"].cpu().numpy()
    plain_boxes, plain_counts = detector.boxes_device(t, **thr)
    assert np.array_equal(counts, plain_counts)
    boxes, plain_boxes = boxes.cpu().numpy(), plain_boxes.cpu().numpy()
    det_thr = thr.get("detection_threshold", 0.7)
    n = 0
    for i, scores in enumerate(maps):
        assert np.array_equal(boxes[i, :counts[i]], plain_boxes[i, :counts[i]])       # the scored run's boxes
        _, ref = S.box_scores(scores, **thr)
        assert int(counts[i]) == len(ref)
        assert np.array_equal(got[i, :counts[i]], ref), i           # exact, box order
        assert np.all(got[i, :counts[i]] >= np.float32(det_thr))
        n += len(ref)
    return n


@pytest.mark.parametrize("thr", [None, 0.5, 0.9])
def test_detection_scores_golden_maps(detector, golden_dir, thr):
    g = np.load(os.path.join(golden_dir, "boxes.npz"))
    kw = {} if thr is None else {"detection_threshold": thr}
    for tag in ("grid32", "rot12", "dense", "blank", "refmaps"):
        _check_box_scores(detector, g[f"boxes_{tag}_scores"], **kw)


def test_detection_scores_large_and_adversarial(detector):
    from oracle import synth
    maps = synth.score_maps(101, 2, 768, 768, 32)
    adv = np.zeros((1, 160, 200, 2), np.float32)
    adv[0, 10:13, 10:13, 0] = 0.9
    adv[0, 10:12, 30:35, 0] = 0.9
    adv[0, 20:25, 60:70, 0] = 0.699                     # below the detection threshold: dropped
    adv[0, 20:25, 90:100, 0] = 0.701                    # kept, score 0.701
    adv[0, 0:8, 150:200, 0] = 0.8
    adv[0, 60:70, 20:120, 0] = 0.8
    adv[0, 60:70, 60:80, 1] = 0.9
    adv[0, 100:130, 40:70, 0] = 0.85
    adv[0, 112, 55, 0] = 0.97                           # one hot pixel sets its component's score
    yy, xx = np.mgrid[0:160, 0:200]
    adv[0, ..., 0] = np.maximum(adv[0, ..., 0], 0.9 * (np.abs(yy - 120) + np.abs(xx - 150) < 18))
    big = np.zeros((1, 1000, 1000, 2), np.float32)      # second quads pass and the global planes
    big[0, 10:340, 50:950, 0] = 0.9
    big[0, 420:750, 40:940, 0] = 0.85
    big[0, 500:600, 300:500, 1] = 0.9
    big[0, 830:990, 100:400, 0] = 0.9
    big[0, 900:910, 500:560, 0] = 0.8
    big[0, 200, 600, 0] = 0.93
    for scores in (maps, adv, big):
        assert _check_box_scores(detector, scores) > 0


def test_detection_scores_overflow_retry(detector):
    from oracle import synth
    maps = synth.score_maps(7, 1, 256, 256, 40)
    detector.max_boxes = 4                               # the count > max_boxes retry keeps the scores
    try:
        _check_box_scores(detector, maps)
        assert detector.max_boxes >= 32
    finally:
        detector.max_boxes = 256


def test_detect_return_scores(detector):
    img = np.random.default_rng(0).integers(0, 256, (2, 96, 128, 3), dtype=np.uint8)
    plain = detector.detect(img)
    scored = detector.detect(img, return_scores=True)
    assert len(scored) == len(plain)
    for p, (b, s) in zip(plain, scored):
        assert np.array_equal(p, b) and s.shape == (len(p),) and s.dtype == np.float32


# ------------------------------------------------------------------------------------------ 3. C3
def test_c3_logp_vs_oracle(cuda_device, golden_dir):
    from keras_ocr_b200.recognition import Recognizer
    from oracle import crnn
    g = np.load(os.path.join(golden_dir, "c3_crops.npz"))
    crops = g["crops"]
    wts = W.synthetic_crnn_weights(2, decisive=True)
    rec = Recognizer(weights=wts)
    rec.keep_workspace = True
    labels, logp = rec.predict_device(_input(rec, crops), with_scores=True)
    logp = logp.cpu().numpy().astype(np.float64)
    logits = rec.tap("logits", (256, 48, 37), torch.float32).double().cpu().numpy()
    ref_logits = []
    with torch.no_grad():
        for i in range(0, 256, 64):
            _, inter = crnn.crnn_logits(wts, crops[i:i + 64].astype(np.float32) / 255, return_intermediates=True)
            ref_logits.append(inter["logits"].double())
    ref_logits = torch.cat(ref_logits)
    s_oracle = S.path_logprob(torch.softmax(ref_logits, -1))
    bound = (2 * np.abs(logits - ref_logits.numpy()).max(-1)).sum(-1) + _slack(37, _terms(logits))
    ratio = np.abs(logp - s_oracle) / bound
    print(f"C3: worst |S_gpu - S_oracle| / bound = {ratio.max():.3g}; confidences median "
          f"{np.median(np.exp(logp)):.3f}, min {np.exp(logp).min():.3g}")
    assert ratio.max() <= 1.0
    assert np.array_equal(labels.cpu().numpy(), g["labels"])
    texts = rec.recognize_crops(crops, return_scores=True)
    assert [t for t, _ in texts] == crnn.labels_to_text(g["labels"])
    assert np.array_equal(np.array([c for _, c in texts]), np.minimum(np.exp(logp.astype(np.float32)), np.float32(1)))


# ------------------------------------------------------------------------------------------ 4. chained pages
def test_chained_pages_scores(cuda_device):
    from keras_ocr_b200 import distributed as D
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    from keras_ocr_b200.recognition import Recognizer
    from oracle import synth
    from oracle.pipeline import OraclePipeline

    cw, rw = W.synthetic_craft_weights(3, textlike=True), W.synthetic_crnn_weights(2, decisive=True)
    rng = np.random.default_rng(1000)
    pages = np.stack([synth.text_image(rng, 768, 768, 32, return_layout=True)[0] for _ in range(2)])
    det, rec = Detector(weights=cw), Recognizer(weights=rw)
    pipe = Pipeline(detector=det, recognizer=rec, scale=2)
    plain = pipe.recognize(pages)
    scored = pipe.recognize(pages, return_scores=True)
    pipe2 = Pipeline(detector=det, recognizer=rec, scale=2, inflight=2)
    pipe2.min_chunk = 1                                   # two pages -> two in-flight sub-batches
    scored2 = pipe2.recognize(pages, return_scores=True)

    def key(res):
        return [[(w[0], np.asarray(w[1]).view(np.int32).tolist()) + tuple(np.float32(v).view(np.int32).item() for v in w[2:])
                 for w in g] for g in res]
    assert [[(t, b.view(np.int32).tolist()) for t, b in g] for g in plain] == [[k[:2] for k in g] for g in key(scored)]
    assert key(scored2) == key(scored)
    assert sum(len(g) for g in scored) >= 60

    # detection scores: exactly the maxima over the GPU's own score map; near the oracle chain's
    batch, _ = pipe.prepare_device(pages)
    gmaps = det.predict_device(batch).cpu().numpy()
    oracle = OraclePipeline(cw, rw, scale=2)
    omaps = oracle.detect_scores(oracle.prepare(pages)[0])
    span = max(float(np.abs(omaps).max()), 1.0)
    worst = 0.0
    for i, g in enumerate(scored):
        s = np.array([w[2] for w in g], np.float32)
        _, own = S.box_scores(gmaps[i])
        assert np.array_equal(s, own)
        _, ref = S.box_scores(omaps[i])
        assert len(ref) == len(s)
        worst = max(worst, float(np.abs(s - ref).max() / span))
        conf = np.array([w[3] for w in g])
        assert np.all(np.isfinite(conf)) and np.all(conf > 0) and np.all(conf <= 1)
    print(f"C4: detection scores vs oracle chain: worst |diff| / map range = {worst:.3g} (bound 2e-2)")
    assert worst <= 2e-2

    records = pipe.recognize_records(pages, scores=True)
    assert records.shape == (2, det.ctx.record_floats_scored(128))
    decoded = D._decode_blocks([records.cpu()], 128, rec.alphabet, scores=True)
    assert key(decoded) == key(scored)
