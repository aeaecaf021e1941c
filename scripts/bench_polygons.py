"""Cost of reading along polygons: Pipeline.recognize with and without return_polygons=True, alternated in one process.

Two workloads: the bench pages (bench.py's 32 pages of 768 x 768 at scale 2, textlike CRAFT weights, the decisive
CRNN) and the curved pages of tests/test_gpu_polygons.py (24 pages, bends 30 to 120 degrees).  Each round times one
call of each mode per workload (host clock around a call that ends in a device synchronise); the report is the median
ms per call and its spread (min-max) over R rounds, with the card's name and power limit read in the same run.
Writes the JSON line to stdout and, with --out, to a file."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [x.strip() for x in q.split(",")]
        return name, limit
    except Exception as e:  # noqa: BLE001 - reported, not hidden
        return f"unknown ({e})", "unknown"


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
    from keras_ocr_b200.recognition import Recognizer
    from tests import test_gpu_polygons as T

    pipe = Pipeline(detector=Detector(weights=W.synthetic_craft_weights(3, textlike=True), device=0),
                    recognizer=Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True), device=0), scale=2)
    curved = [T.curved_pages(b, n=6) for b in T.BENDS]
    workloads = {"bench_pages": bench.make_pages(0),
                 "curved_pages": np.concatenate([c[0] for c in curved])}
    times = {(w, m): [] for w in workloads for m in ("default", "polygons")}
    for images in workloads.values():                            # warm up every shape
        pipe.recognize(images)
        pipe.recognize(images, return_polygons=True)
    for _ in range(args.rounds):
        for w, images in workloads.items():
            for mode in ("default", "polygons"):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                pipe.recognize(images, return_polygons=mode == "polygons")
                torch.cuda.synchronize()
                times[(w, mode)].append(1e3 * (time.perf_counter() - t0))
    name, limit = card()
    res = {"gpu": name, "power_limit": limit, "rounds": args.rounds, "pages": {w: len(v) for w, v in workloads.items()}}
    for (w, mode), v in times.items():
        res[f"{w}.{mode}.median_ms"] = round(statistics.median(v), 2)
        res[f"{w}.{mode}.spread_ms"] = [round(min(v), 2), round(max(v), 2)]
    for w in workloads:
        res[f"{w}.overhead_pct"] = round(100 * (res[f"{w}.polygons.median_ms"] / res[f"{w}.default.median_ms"] - 1), 2)
    words = {}
    for b, (images, ws) in zip(T.BENDS, curved):
        words[b] = (T._read(pipe.recognize(images), ws), T._read(pipe.recognize(images, return_polygons=True), ws),
                    sum(len(x) for x in ws))
    res["curved_words_read_default_polygons_of"] = words
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
