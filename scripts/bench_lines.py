"""Cost of text lines: Pipeline.recognize with and without return_lines=True, alternated in one process, and the
b2o_group_lines kernels alone.

Step time: the bench pages (bench.py's 32 pages of 768 x 768 at scale 2, textlike CRAFT weights, the decisive CRNN);
each round times one call of each mode (host clock around a call that ends in a device synchronise), and the report
is the median ms per call and its spread (min-max) over R rounds.  Kernel time: b2o_group_lines (its three launches)
on seeded random layouts at 32 images x 256 words and at 1 image x 8192 words, CUDA events around 50 calls, the two
sizes alternated per round.  The card's name and power limit are read in the same run.  Writes the JSON line to
stdout and, with --out, to a file."""
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
    from tests import test_gpu_lines as T

    pipe = Pipeline(detector=Detector(weights=W.synthetic_craft_weights(3, textlike=True), device=0),
                    recognizer=Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True), device=0), scale=2)
    pages = bench.make_pages(0)
    pipe.recognize(pages)                                        # warm up every shape
    pipe.recognize(pages, return_lines=True)
    times = {"default": [], "lines": []}
    for _ in range(args.rounds):
        for mode in times:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pipe.recognize(pages, return_lines=mode == "lines")
            torch.cuda.synchronize()
            times[mode].append(1e3 * (time.perf_counter() - t0))

    ctx = pipe.detector.ctx
    rng = np.random.default_rng(0)
    cases = {}
    for name, n, m in (("32x256", 32, 256), ("1x8192", 1, 8192)):
        t, counts = T.table([T.random_page(rng, m) for _ in range(n)], m)
        outs = [torch.empty(s, dtype=d, device="cuda") for s, d in
                (((n,), torch.int32), ((n, m), torch.int32), ((n, m + 1), torch.int32), ((n, m, 4, 2), torch.float32))]
        nbytes = ctx.lines_workspace_bytes(n, m)
        cases[name] = (torch.from_numpy(t).cuda(), torch.from_numpy(counts).cuda(), n, m, outs,
                       torch.empty(nbytes, dtype=torch.uint8, device="cuda"), nbytes)
    params = T._params({})

    def launch(case):
        boxes, counts, n, m, outs, ws, nbytes = case
        ctx.group_lines(boxes.data_ptr(), counts.data_ptr(), n, m, *params, *[o.data_ptr() for o in outs],
                        ws.data_ptr(), nbytes, torch.cuda.current_stream().cuda_stream)

    kernel = {name: [] for name in cases}
    for case in cases.values():
        launch(case)
    for _ in range(args.rounds):
        for name, case in cases.items():
            start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            for _ in range(50):
                launch(case)
            stop.record()
            stop.synchronize()
            kernel[name].append(start.elapsed_time(stop) / 50)

    name, limit = card()
    res = {"gpu": name, "power_limit": limit, "rounds": args.rounds, "pages": len(pages)}
    for mode, v in times.items():
        res[f"bench_pages.{mode}.median_ms"] = round(statistics.median(v), 2)
        res[f"bench_pages.{mode}.spread_ms"] = [round(min(v), 2), round(max(v), 2)]
    res["bench_pages.overhead_pct"] = round(100 * (res["bench_pages.lines.median_ms"] /
                                                   res["bench_pages.default.median_ms"] - 1), 2)
    for case, v in kernel.items():
        res[f"group_lines.{case}.median_ms"] = round(statistics.median(v), 4)
        res[f"group_lines.{case}.spread_ms"] = [round(min(v), 4), round(max(v), 4)]
    got = pipe.recognize(pages[:4], return_lines=True)
    res["bench_pages.lines_per_page"] = [len(g) for g in got]
    res["bench_pages.words_per_page"] = [sum(len(l[2]) for l in g) for g in got]
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
