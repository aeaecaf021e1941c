"""Cost and usefulness of character scores (``return_char_scores``, ``b2o_ctc_char_scores``).

Timing.  The kernel alone: ``b2o_ctc_char_scores`` on 1024 crops of seeded logits (K = 37) with the readings the beam
decoder returns for them (``b2o_ctc_beam_decode``, W = 8), P in {1, 8}, A in {0, 8}; CUDA events around 10 calls after
a warm-up, median and spread over R rounds.  End to end: ``Pipeline.recognize`` on bench.py's 32 pages, greedy and
``beam_width=16``, without and with ``return_char_scores`` (A = 8; greedy also A = 0), alternated in one process;
median ms per call and its spread (min-max) over R rounds.

Usefulness.  On the degraded pseudo-language pages of tests/test_gpu_lm.py (``pseudo_pages``, ``SEVERITY``, its test
seeds), greedy readings of the true length, character by character against the rendered word: the ROC AUC of the
character confidence as a detector of misread characters, against the baseline of the largest softmax probability of
the read label over the character's Viterbi span (``b2o_ctc_align`` on the same logits, tapped from the recognizer's
workspace); and how often the true character of a misread one is the top 1, among the top 4 and among the top 8
alternatives.  The card's name and power limit are read in the same run.  Writes the JSON line to stdout and, with
--out, to a file."""
import argparse
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def auc(pos, neg):
    """P(a positive scores below a negative) + P(tie) / 2: how well a low score singles out the positives."""
    import numpy as np
    from scipy.stats import rankdata
    pos, neg = np.asarray(pos, np.float64), np.asarray(neg, np.float64)
    r = rankdata(-np.concatenate([pos, neg]))        # high rank = low score
    return float((r[:len(pos)].sum() - len(pos) * (len(pos) + 1) / 2) / (len(pos) * len(neg)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import cv2
    import numpy as np
    import torch

    import bench
    from keras_ocr_b200 import weights as W
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    from keras_ocr_b200.recognition import Recognizer
    from scripts.bench_lm import report
    from scripts.bench_polygons import card
    from tests.test_gpu_beam import crafted
    from tests.test_gpu_lm import SEVERITY, TEST_SEEDS, pseudo_pages

    assert torch.cuda.is_available(), "bench_char_scores measures on the GPU"
    pipe = Pipeline(detector=Detector(weights=W.synthetic_craft_weights(3, textlike=True), device=0),
                    recognizer=Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True), device=0),
                    scale=bench.SCALE, max_size=2048)
    rec = pipe.recognizer
    line = {"card": None, "power_limit": None, "rounds": args.rounds}

    # ---- the kernel alone
    ctx, stream = rec.ctx, torch.cuda.current_stream().cuda_stream
    n, k = 1024, 37
    x = torch.from_numpy(crafted(k, n, seed=5)).cuda()
    labels = torch.empty((n, 8, 48), dtype=torch.int32, device="cuda")
    logp = torch.empty((n, 8), dtype=torch.float32, device="cuda")
    ctx.ctc_beam_decode(x.data_ptr(), n, k, 8, 8, labels.data_ptr(), logp.data_ptr(), stream)
    lens = (labels >= 0).sum(-1).float()
    line["kernel_readings_mean_length"] = {"P=1": round(float(lens[:, 0].mean()), 2), "P=8": round(float(lens.mean()), 2)}

    def timed(call):
        call()
        reps = []
        for _ in range(args.rounds):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(10):
                call()
            b.record()
            b.synchronize()
            reps.append(a.elapsed_time(b) / 10)
        return {"median_ms": round(statistics.median(reps), 3), "min_ms": round(min(reps), 3),
                "max_ms": round(max(reps), 3)}

    kernel = {}
    for p in (1, 8):
        lab = labels[:, :p].contiguous()
        for a in (0, 8):
            conf = torch.empty((n, p, 48), dtype=torch.float32, device="cuda")
            al = torch.empty((n, p, 48, max(a, 1)), dtype=torch.int32, device="cuda")
            post = torch.empty((n, p, 48, max(a, 1)), dtype=torch.float32, device="cuda")
            kernel[f"P={p},A={a}"] = timed(lambda p=p, a=a, lab=lab, conf=conf, al=al, post=post: ctx.ctc_char_scores(
                x.data_ptr(), n, k, lab.data_ptr(), p, a, conf.data_ptr(), al.data_ptr() if a else None,
                post.data_ptr() if a else None, None, stream))
    line["kernel_1024_crops_k37"] = kernel

    # ---- end to end on bench.py's pages
    pages = bench.make_pages(0)
    modes = {"greedy": ({}, {}), "greedy+conf": ({}, {"return_char_scores": True}),
             "greedy+scores": ({}, {"return_char_scores": True, "char_alternatives": 8}),
             "beam16": ({"beam_width": 16}, {}),
             "beam16+scores": ({"beam_width": 16}, {"return_char_scores": True, "char_alternatives": 8})}
    for kw, flags in modes.values():                           # warm up every shape
        pipe.recognize(pages, recognition_kwargs=kw, **flags)
    times = {m: [] for m in modes}
    for _ in range(args.rounds):
        for m, (kw, flags) in modes.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pipe.recognize(pages, recognition_kwargs=kw, **flags)
            torch.cuda.synchronize()
            times[m].append((time.perf_counter() - t0) * 1e3)
    line["bench_pages"] = {m: {"median_ms": round(statistics.median(v), 2), "min_ms": round(min(v), 2),
                               "max_ms": round(max(v), 2)} for m, v in times.items()}

    # ---- usefulness on the degraded pages: one sub-batch, so the recognizer's workspace keeps every word's logits
    pg, items = pseudo_pages(TEST_SEEDS, SEVERITY)
    rec.keep_workspace = True
    res = pipe.recognize(pg, return_char_scores=True, char_alternatives=8)
    words = [w for g in res for w in g]
    logits = rec.tap("logits", (len(words), 48, k), torch.float32)
    rec.keep_workspace = False
    lab = np.full((len(words), 1, 48), -1, np.int32)
    for i, w in enumerate(words):
        lab[i, 0, :len(w[0])] = [rec.alphabet.index(ch) for ch in w[0]]
    spans = torch.empty((len(words), 1, 48, 2), dtype=torch.int32, device="cuda")
    lab_t = torch.from_numpy(lab).cuda()
    ctx.ctc_align(logits.data_ptr(), len(words), k, lab_t.data_ptr(), 1, spans.data_ptr(), None, stream)
    prob = torch.softmax(logits.double(), -1).cpu().numpy()
    spans = spans.cpu().numpy()
    conf_right, conf_wrong, base_right, base_wrong, ranks = [], [], [], [], []
    start = 0
    for g, it in zip(res, items):
        for q, word in enumerate(g):
            i = start + q
            box = np.asarray(word[1], np.float32).reshape(-1, 1, 2)
            inside = [t for t, c in it if cv2.pointPolygonTest(box, (float(c[0]), float(c[1])), False) >= 0]
            if len(inside) != 1 or len(inside[0]) != len(word[0]):
                continue
            conf, alts = word[-1]
            for j, (r, t) in enumerate(zip(word[0], inside[0])):
                f, l = spans[i, 0, j]
                base = float(prob[i, f:l + 1, lab[i, 0, j]].max()) if f >= 0 else 0.0
                if r == t:
                    conf_right.append(float(conf[j]))
                    base_right.append(base)
                else:
                    conf_wrong.append(float(conf[j]))
                    base_wrong.append(base)
                    chars = [ch for ch, _ in alts[j]]
                    ranks.append(chars.index(t) if t in chars else None)
        start += len(g)
    m = len(conf_wrong)
    line["degraded_pages"] = {
        "severity": SEVERITY, "seeds": list(TEST_SEEDS), "words": sum(len(it) for it in items),
        "characters_scored": len(conf_right) + m, "misread": m,
        "mean_confidence_right": round(float(np.mean(conf_right)), 4),
        "mean_confidence_misread": round(float(np.mean(conf_wrong)), 4) if m else None,
        "auc_confidence": round(auc(conf_wrong, conf_right), 4) if m else None,
        "auc_span_max_softmax": round(auc(base_wrong, base_right), 4) if m else None,
        "true_char_top1": sum(r == 0 for r in ranks), "true_char_top4": sum(r is not None and r < 4 for r in ranks),
        "true_char_top8": sum(r is not None for r in ranks)}
    report(line, args.out, card)


if __name__ == "__main__":
    main()
