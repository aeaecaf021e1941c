"""Cost of text blocks: Pipeline.recognize with and without return_blocks=True, alternated in one process, and the
b2o_group_blocks kernel alone.

Step time: the bench pages (bench.py's 32 pages of 768 x 768 at scale 2, textlike CRAFT weights, the decisive CRNN);
each round times one call of each mode (host clock around a call that ends in a device synchronise), and the report
is the median ms per call and its spread (min-max) over R rounds.  Kernel time: b2o_group_blocks (one launch) on
seeded random column layouts at 32 images x 256 lines and 1 image x 8192 lines, and on the 1024-line spiral
(tests/block_refs.py, one cut per tree level); CUDA events around a number of calls, the cases alternated per round.
The card's name and power limit are read in the same run.  Writes the JSON line to stdout and, with --out, to a
file."""
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
    from tests import block_refs as R
    from tests import test_gpu_blocks as T

    pipe = Pipeline(detector=Detector(weights=W.synthetic_craft_weights(3, textlike=True), device=0),
                    recognizer=Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True), device=0), scale=2)
    pages = bench.make_pages(0)
    pipe.recognize(pages)                                        # warm up every shape
    pipe.recognize(pages, return_blocks=True)
    times = {"default": [], "blocks": []}
    for _ in range(args.rounds):
        for mode in times:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pipe.recognize(pages, return_blocks=mode == "blocks")
            torch.cuda.synchronize()
            times[mode].append(1e3 * (time.perf_counter() - t0))

    ctx = pipe.detector.ctx
    rng = np.random.default_rng(0)
    cases = {}
    for name, pages_, m, reps in (("32x256", [R.random_page(rng, 256) for _ in range(32)], 256, 50),
                                  ("1x8192", [R.random_page(rng, 8192, tilt=3.0)], 8192, 10),
                                  ("spiral1024", [R.spiral(1024)], 1024, 3)):
        n = len(pages_)
        ins = [torch.from_numpy(a).cuda() for a in T.table(pages_, m)]
        outs = [torch.empty(s, dtype=d, device="cuda") for s, d in
                (((n,), torch.int32), ((n, m), torch.int32), ((n, m + 1), torch.int32), ((n, m, 4, 2), torch.float32))]
        nbytes = ctx.blocks_workspace_bytes(n, m)
        cases[name] = (ins, n, m, outs, torch.empty(nbytes, dtype=torch.uint8, device="cuda"), nbytes, reps)
    params = T._params({})

    def launch(case):
        ins, n, m, outs, ws, nbytes, _ = case
        ctx.group_blocks(*[t.data_ptr() for t in ins], n, m, *params, *[o.data_ptr() for o in outs], ws.data_ptr(),
                         nbytes, torch.cuda.current_stream().cuda_stream)

    kernel = {name: [] for name in cases}
    for case in cases.values():
        launch(case)
    for _ in range(args.rounds):
        for name, case in cases.items():
            start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            for _ in range(case[-1]):
                launch(case)
            stop.record()
            stop.synchronize()
            kernel[name].append(start.elapsed_time(stop) / case[-1])
    blocks_found = {name: int(case[3][0].cpu().max()) for name, case in cases.items()}

    name, limit = card()
    res = {"gpu": name, "power_limit": limit, "rounds": args.rounds, "pages": len(pages)}
    for mode, v in times.items():
        res[f"bench_pages.{mode}.median_ms"] = round(statistics.median(v), 2)
        res[f"bench_pages.{mode}.spread_ms"] = [round(min(v), 2), round(max(v), 2)]
    res["bench_pages.overhead_pct"] = round(100 * (res["bench_pages.blocks.median_ms"] /
                                                   res["bench_pages.default.median_ms"] - 1), 2)
    for case, v in kernel.items():
        res[f"group_blocks.{case}.median_ms"] = round(statistics.median(v), 4)
        res[f"group_blocks.{case}.spread_ms"] = [round(min(v), 4), round(max(v), 4)]
        res[f"group_blocks.{case}.max_blocks"] = blocks_found[case]
    got = pipe.recognize(pages[:4], return_blocks=True)
    res["bench_pages.blocks_per_page"] = [len(g) for g in got]
    res["bench_pages.lines_per_page"] = [sum(len(b[2]) for b in g) for g in got]
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
