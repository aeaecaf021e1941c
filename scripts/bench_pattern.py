"""Cost and effect of pattern-constrained decoding (``pattern=``, ``b2o_crnn_forward_beam_pattern``).

Timing.  The decoder alone: ``b2o_ctc_beam_pattern_decode`` against ``b2o_ctc_beam_decode`` on 1024 crops of seeded
logits (K = 37), W in {4, 16, 64, 128}, with four patterns: ``.*``, ``[0-9]+``, a plate format and a large automaton
(an alternation of 300 seeded random words); CUDA events around 10 calls after a warm-up, median and spread over R
rounds.  End to end: ``Pipeline.recognize`` on bench.py's 32 pages with ``beam_width=16``, with and without ``.*``,
alternated in one process; median ms per call and its spread (min-max) over R rounds.

Accuracy.  Exact reads (``window_refs.exact_reads``) on degraded pages of formatted codes (tests/test_gpu_pattern.py:
plates, invoice numbers and dates, rendered and degraded as tests/test_gpu_lm.py renders its pages, at its
``SEVERITY``): greedy, beam 16 and beam 16 + the alternation of the three formats, on the tuning seeds (100..103) and
on the tests' test seeds.  The card's name and power limit are read in the same run.  Writes the JSON line to stdout
and, with --out, to a file."""
import argparse
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TUNING_SEEDS = (100, 101, 102, 103)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import torch

    import bench
    from keras_ocr_b200 import weights as W
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    from keras_ocr_b200.recognition import Pattern, Recognizer
    from scripts.bench_lm import report
    from scripts.bench_polygons import card
    from tests import window_refs as R
    from tests.test_gpu_beam import crafted
    from tests.test_gpu_lm import SEVERITY
    from tests.test_gpu_pattern import CODES, TEST_SEEDS, code_pages

    assert torch.cuda.is_available(), "bench_pattern measures on the GPU"
    pipe = Pipeline(detector=Detector(weights=W.synthetic_craft_weights(3, textlike=True), device=0),
                    recognizer=Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True), device=0), scale=2)
    rec = pipe.recognizer
    rng = np.random.default_rng(11)
    words = sorted({"".join(rng.choice(list("abcdefghijklmnopqrstuvwxyz0123456789"), int(rng.integers(4, 11))))
                    for _ in range(300)})
    t0 = time.perf_counter()
    large = Pattern("|".join(words))
    compile_ms = (time.perf_counter() - t0) * 1e3
    patterns = {"any": Pattern(".*"), "digits": Pattern("[0-9]+"), "plate": Pattern("[a-z]{3}[0-9]{4}"),
                "words300": large}
    line = {"card": None, "power_limit": None, "rounds": args.rounds,
            "states": {k: p.n_states for k, p in patterns.items()}, "words300_compile_ms": round(compile_ms, 1)}

    # ---- the decoder alone
    ctx, stream = rec.ctx, torch.cuda.current_stream().cuda_stream
    x = torch.from_numpy(crafted(37, 1024, seed=5)).cuda()
    labels = torch.empty((1024, 4, 48), dtype=torch.int32, device="cuda")
    logp = torch.empty((1024, 4), dtype=torch.float32, device="cuda")

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
    for w in (4, 16, 64, 128):
        entry = {"beam": timed(lambda w=w: ctx.ctc_beam_decode(x.data_ptr(), 1024, 37, w, 4, labels.data_ptr(),
                                                               logp.data_ptr(), stream))}
        for name, pat in patterns.items():
            desc = pat.descriptor("cuda:0")
            entry[name] = timed(lambda w=w, desc=desc: ctx.ctc_beam_pattern_decode(
                x.data_ptr(), 1024, 37, w, 4, desc, labels.data_ptr(), logp.data_ptr(), stream))
        kernel[f"W={w}"] = entry
    line["decoder_1024_crops_k37"] = kernel

    # ---- end to end on bench.py's pages
    pages = bench.make_pages(0)
    modes = {"beam16": {"beam_width": 16}, "beam16+any": {"beam_width": 16, "pattern": patterns["any"]}}
    for kw in modes.values():                                   # warm up every shape
        pipe.recognize(pages, recognition_kwargs=kw)
    times = {m: [] for m in modes}
    for _ in range(args.rounds):
        for m, kw in modes.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pipe.recognize(pages, recognition_kwargs=kw)
            torch.cuda.synchronize()
            times[m].append((time.perf_counter() - t0) * 1e3)
    line["bench_pages"] = {m: {"median_ms": round(statistics.median(v), 2), "min_ms": round(min(v), 2),
                               "max_ms": round(max(v), 2)} for m, v in times.items()}

    # ---- degraded code pages: tuning seeds, then the test seeds
    codes = Pattern(CODES)
    line["severity"] = SEVERITY
    for name, seeds in (("tuning_pages", TUNING_SEEDS), ("test_pages", TEST_SEEDS)):
        pg, items = code_pages(seeds)
        entry = {"codes": sum(len(it) for it in items)}
        for m, kw in (("greedy", {}), ("beam16", {"beam_width": 16}),
                      ("beam16+pattern", {"beam_width": 16, "pattern": codes})):
            res = pipe.recognize(pg, recognition_kwargs=kw)
            entry[m] = sum(R.exact_reads(g, it) for g, it in zip(res, items))
            if "pattern" in kw:
                entry["no_matching_reading"] = sum(t == "" for g in res for t, _ in g)
                entry["all_match"] = all(t == "" or codes.fullmatch(t) for g in res for t, _ in g)
        line[name] = entry
    report(line, args.out, card)


if __name__ == "__main__":
    main()
