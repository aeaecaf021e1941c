"""Cost of wide-word windows: Pipeline.recognize with and without recognition_kwargs={"max_windows": 4}, alternated in
one process, and b2o_stitch_windows alone.

Step time, two workloads: the bench pages (bench.py's 32 pages of 768 x 768 at scale 2, no box wider than the crop at
full height) and 32 long-word pages (tests/window_refs.py's long_word_page: one 14- to 30-letter word or a merged pair
per line).  Each round times one call of each mode (host clock around a call that ends in a device synchronise); the
report is the median ms per call and its spread (min-max) over R rounds, and the words read exactly on the long-word
pages.  Kernel time: b2o_stitch_windows on 32 x 256 seeded wide words (window_refs.stitch_case), CUDA events around
50 calls.  The card's name and power limit are read in the same run.  Writes the JSON line to stdout and, with --out,
to a file."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import torch

    import bench
    from keras_ocr_b200 import weights as W
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    from keras_ocr_b200.recognition import Recognizer
    from scripts.bench_polygons import card
    from tests import window_refs as R

    pipe = Pipeline(detector=Detector(weights=W.synthetic_craft_weights(3, textlike=True), device=0),
                    recognizer=Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True), device=0), scale=2)
    long_pages = [R.long_word_page(100 + s) for s in range(32)]
    workloads = {"bench_pages": bench.make_pages(0), "long_word_pages": np.stack([p for p, _ in long_pages])}
    modes = {"default": {}, "max_windows=4": {"recognition_kwargs": {"max_windows": 4}}}
    line = {"card": None, "power_limit": None, "rounds": args.rounds}
    for name, pages in workloads.items():
        results = {m: pipe.recognize(pages, **kw) for m, kw in modes.items()}      # warm up every shape
        times = {m: [] for m in modes}
        for _ in range(args.rounds):
            for m, kw in modes.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                pipe.recognize(pages, **kw)
                torch.cuda.synchronize()
                times[m].append((time.perf_counter() - t0) * 1e3)
        entry = {m: {"median_ms": round(statistics.median(v), 2), "min_ms": round(min(v), 2),
                     "max_ms": round(max(v), 2)} for m, v in times.items()}
        base = entry["default"]["median_ms"]
        entry["extra_pct"] = round(100 * (entry["max_windows=4"]["median_ms"] - base) / base, 2)
        if name == "long_word_pages":
            entry["items"] = sum(len(i) for _, i in long_pages)
            for m in modes:
                entry[m]["exact"] = sum(R.exact_reads(r, i) for r, (_, i) in zip(results[m], long_pages))
        line[name] = entry

    # stitch_kernel alone on 32 x 256 wide words
    ctx = pipe.recognizer.ctx
    quads, m, words, start, lg, th = R.stitch_case(7, 32 * 256)
    dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (lg, th, quads, words, start)]
    labels = torch.empty((len(quads), 48 * m), dtype=torch.int32, device="cuda")
    logp = torch.empty((len(quads),), dtype=torch.float32, device="cuda")
    stream = torch.cuda.current_stream().cuda_stream

    def call():
        ctx.stitch_windows(dev[0].data_ptr(), 37, dev[1].data_ptr(), dev[2].data_ptr(), dev[3].data_ptr(),
                           dev[4].data_ptr(), len(words), m, labels.data_ptr(), logp.data_ptr(), stream)

    for _ in range(5):
        call()
    reps, per = [], 50
    for _ in range(args.rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(per):
            call()
        b.record()
        b.synchronize()
        reps.append(a.elapsed_time(b) / per)
    line["stitch_kernel"] = {"words": int(len(words)), "windows": int(start[-1]), "max_windows": m,
                             "median_ms": round(statistics.median(reps), 4), "min_ms": round(min(reps), 4),
                             "max_ms": round(max(reps), 4)}
    line["card"], line["power_limit"] = card()
    text = json.dumps(line)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
