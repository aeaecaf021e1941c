"""bench_scores.py -- what detection scores, word confidences and beam-search decoding cost: ``Pipeline.recognize``
with and without ``return_scores=True``, and with ``recognition_kwargs={"beam_width": W}`` for every W given, on the
workload of bench.py (32 pages 768x768, scale 2 -> 1536x1536, sources resident in HBM).

    python scripts/bench_scores.py [--steps K] [--warmup W] [--rounds R] [--beam-width W [W ...]]

The calls are timed alternately, R rounds of K steps each (CUDA events around K steps bracketed by a device
synchronise), so that drifting clocks and other work on the host hit all alike; prints one JSON line with the medians,
the spread over the rounds, the rendered words each call reads correctly (``bench.words_read``) and the card's name
and power limit.  Writes nothing.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card_info(device_index):
    """Name and power limit (W) of the measured card (read-only nvidia-smi query)."""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits",
                              "-i", str(device_index)], capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [p.strip() for p in out.split(",")[:2]]
        return {"gpu": name, "power_limit_w": float(limit)}
    except (OSError, ValueError, subprocess.SubprocessError):
        return {"gpu": None, "power_limit_w": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--beam-width", type=int, nargs="+", default=[])
    args = ap.parse_args()

    import torch

    import bench
    from keras_ocr_b200 import weights as W
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    from keras_ocr_b200.recognition import Recognizer

    assert torch.cuda.is_available(), "bench_scores.py needs a CUDA device; there is no CPU fallback"
    device = torch.device("cuda", 0)
    det = Detector(weights=W.synthetic_craft_weights(3, textlike=True), device=0)
    rec = Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True), device=0)
    pipe = Pipeline(detector=det, recognizer=rec, scale=bench.SCALE, max_size=2048)
    pages_host, page_words, page_rects = bench.make_pages(0, with_layout=True)
    pages = torch.from_numpy(pages_host).to(device)
    calls = {"default": lambda: pipe.recognize(pages), "scored": lambda: pipe.recognize(pages, return_scores=True)}
    for w in args.beam_width:
        calls[f"beam{w}"] = lambda w=w: pipe.recognize(pages, recognition_kwargs={"beam_width": w})

    def timed(fn):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    for _ in range(max(args.warmup, 1)):
        for fn in calls.values():
            fn()
    ms = {k: [] for k in calls}
    for _ in range(args.rounds):
        for k, fn in calls.items():
            ms[k].append(timed(fn))
    words = sum(len(g) for g in calls["default"]())
    line = dict(card_info(0), **{
        "workload": bench.workload_config(1)["workload"], "steps_per_round": args.steps, "rounds": args.rounds,
        "words_per_step": words,
        "default_ms_per_step": statistics.median(ms["default"]), "scored_ms_per_step": statistics.median(ms["scored"]),
        "default_ms_spread": [min(ms["default"]), max(ms["default"])],
        "scored_ms_spread": [min(ms["scored"]), max(ms["scored"])],
        "overhead": statistics.median(ms["scored"]) / statistics.median(ms["default"]) - 1.0})
    default_words = [t for g in calls["default"]() for t, _ in g]
    for k, fn in calls.items():
        if k == "scored":
            continue
        result = fn()
        hit, rendered = bench.words_read(result, page_words, page_rects)
        line[f"{k}_words_read"] = [hit, rendered]
        if k != "default":
            line[f"{k}_ms_per_step"] = statistics.median(ms[k])
            line[f"{k}_ms_spread"] = [min(ms[k]), max(ms[k])]
            line[f"{k}_overhead"] = statistics.median(ms[k]) / statistics.median(ms["default"]) - 1.0
            line[f"{k}_words_differing_from_default"] = sum(a != b for a, b in zip([t for g in result for t, _ in g],
                                                                                  default_words))
    print(json.dumps(line))


if __name__ == "__main__":
    main()
