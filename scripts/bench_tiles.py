"""Tiled detection (DESIGN.md section 1, "Tiles"): cost on large pages, and the seam error against the whole-page
forward at each margin.

perf: 4 pages of 3072 x 3072 (oracle.synth.text_images, 512 words each: the glyph size of bench.py's pages) through
Pipeline(scale=2, max_size=6144), a 6144 x 6144 detector input tiled at 2048.  Reports the median ms per page end to end
(host clock around calls that end in a device synchronise), the cut / CRAFT / stitch / getBoxes times from CUDA events
around each launch of one tiled forward and its getBoxes, the overlap overhead, how many pages had more boxes than the
first box table holds (a rerun of getBoxes in boxes_finish), and the peak allocated memory of the detect stage, tiled
and whole-page where the whole page is allowed.

margins: 4 pages of 1536 x 1536 (128 words each) at scale 2, a 3072 x 3072 detector input, through the whole-page
forward and through tiles of 2048 with margins 0, 64, 128 and 256: the largest |score difference| (every score is a
core score of one tile), the boxes matched one to one (axis-aligned IoU >= 0.5) and their smallest IoU, and the words
whose text is the same in both runs.

The card's name and power limit are read in the same run.  Writes the JSON line to stdout and, with --out, to a file."""
import argparse
import collections
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _iou(a, b):
    ax0, ay0, ax1, ay1 = a[:, 0].min(), a[:, 1].min(), a[:, 0].max(), a[:, 1].max()
    bx0, by0, bx1, by1 = b[:, 0].min(), b[:, 1].min(), b[:, 0].max(), b[:, 1].max()
    iw, ih = max(0.0, min(ax1, bx1) - max(ax0, bx0)), max(0.0, min(ay1, by1) - max(ay0, by0))
    inter = iw * ih
    union = (ax1 - ax0) * (ay1 - ay0) + (bx1 - bx0) * (by1 - by0) - inter
    return float(inter / union) if union > 0 else 0.0


def _match(ref, got):
    """Greedy one-to-one matching of two box lists at IoU >= 0.5: (matched, smallest IoU of a match)."""
    used, ious = set(), []
    for a in ref:
        best, j = 0.0, -1
        for k, b in enumerate(got):
            if k not in used:
                v = _iou(a, b)
                if v > best:
                    best, j = v, k
        if best >= 0.5:
            used.add(j)
            ious.append(best)
    return len(ious), (min(ious) if ious else None)


def perf(pipe, rounds):
    import numpy as np
    import torch

    from keras_ocr_b200 import _lib, detection
    from oracle import synth

    det = pipe.detector
    pages, _ = synth.text_images(seed=77, n=4, h=3072, w=3072, n_words=512)
    pipe.recognize(pages)                                        # warm up every shape
    times = []
    for _ in range(rounds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pipe.recognize(pages)
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3 / len(pages))
    out = {"pages": len(pages), "page": [3072, 3072], "detector_input": None,
           "ms_per_page": {"median": round(statistics.median(times), 2), "min": round(min(times), 2),
                           "max": round(max(times), 2)}}
    batch, _ = pipe.prepare_device(pages)
    n, hp, wp, _ = batch.shape
    out["detector_input"] = [hp, wp]
    plan = _lib.tile_plan(hp, wp, detection.DEFAULT_TILE_SIZE, detection.TILE_MARGIN)
    total = n * plan.n_h * plan.n_w
    out["tiles"] = {"per_page": plan.n_h * plan.n_w, "tile": [plan.t_h, plan.t_w], "margin": detection.TILE_MARGIN,
                    "nominal_overhead_(t/s)^2": round((plan.t_h / plan.s_h) * (plan.t_w / plan.s_w), 3),
                    "tile_pixels_over_page_pixels": round(plan.n_h * plan.n_w * plan.t_h * plan.t_w / (hp * wp), 3)}
    # one tiled forward launch by launch, events around each
    stream = torch.cuda.current_stream().cuda_stream
    per = min(total, max(1, detection.TILE_CHUNK_PIXELS // (plan.t_h * plan.t_w)))
    tiles = torch.empty((per, plan.t_h, plan.t_w, 3), dtype=torch.uint8, device="cuda")
    tile_scores = torch.empty((per, plan.t_h // 2, plan.t_w // 2, 2), dtype=torch.float32, device="cuda")
    scores = torch.empty((n, hp // 2, wp // 2, 2), dtype=torch.float32, device="cuda")
    ws, nbytes = det._workspace(per, plan.t_h, plan.t_w)
    stage = collections.defaultdict(list)

    def timed(name, fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        stage[name].append((a, b))

    for rep in range(rounds):
        for first in range(0, total, per):
            k = min(per, total - first)
            timed(f"cut_{rep}", lambda: det.ctx.cut_tiles(batch.data_ptr(), n, plan, first, k, tiles.data_ptr(), stream))
            timed(f"craft_{rep}", lambda: det.ctx.craft_forward(tiles.data_ptr(), k, plan.t_h, plan.t_w,
                                                                tile_scores.data_ptr(), ws.data_ptr(), nbytes, stream))
            timed(f"stitch_{rep}", lambda: det.ctx.stitch_tiles(tile_scores.data_ptr(), n, plan, first, k,
                                                                scores.data_ptr(), stream))
        timed(f"getboxes_{rep}", lambda: det.boxes_enqueue(scores))
    torch.cuda.synchronize()
    ms = {}
    for name in ("cut", "craft", "stitch", "getboxes"):
        per_rep = [sum(a.elapsed_time(b) for a, b in stage[f"{name}_{r}"]) for r in range(rounds)]
        ms[name] = round(statistics.median(per_rep), 3)
    ms["cut+stitch_share_of_craft_pct"] = round(100 * (ms["cut"] + ms["stitch"]) / ms["craft"], 3)
    out["stage_ms_per_batch"] = ms
    state = det.boxes_enqueue(scores)
    _, counts = det.boxes_finish(state)
    out["boxes_per_page"] = [int(c) for c in counts]
    out["pages_over_256_boxes"] = int((counts > 256).sum())
    # peak allocated memory of the detect stage
    peak = {}
    for label, b, tile in (("tiled_6144", batch, detection.DEFAULT_TILE_SIZE),):
        det._ws = None
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        det.predict_device(b, tile_size=tile)
        torch.cuda.synchronize()
        peak[label] = round((torch.cuda.max_memory_allocated() - base) / 2**30, 3)
    peak["whole_6144"] = "refused: more than 2^25 pixels per image"
    small = batch[:, :3072, :3072].contiguous()
    for label, tile in (("tiled_3072", detection.DEFAULT_TILE_SIZE), ("whole_3072", None)):
        det._ws = None
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        det.predict_device(small, tile_size=tile)
        torch.cuda.synchronize()
        peak[label] = round((torch.cuda.max_memory_allocated() - base) / 2**30, 3)
    out["detect_peak_gib_4_pages"] = peak
    return out


def margins(pipe):
    import numpy as np
    import torch

    from oracle import synth

    det = pipe.detector
    pages, _ = synth.text_images(seed=55, n=4, h=1536, w=1536, n_words=128)
    batch, _ = pipe.prepare_device(pages)
    whole = det.predict_device(batch)
    wb, wc = det.boxes_device(whole)
    wb = wb.cpu().numpy()
    orig = det.predict_device
    det.predict_device = lambda b, tile_size=None, margin=None: orig(b)
    try:
        ref_words = pipe.recognize(pages)
    finally:
        det.predict_device = orig
    rows = []
    for m in (0, 64, 128, 256):
        tiled = det.predict_device(batch, tile_size=2048, margin=m)
        diff = float((tiled - whole).abs().max())
        tb, tc = det.boxes_device(tiled)
        tb = tb.cpu().numpy()
        matched, worst = 0, 1.0
        for i in range(len(pages)):
            k, lo = _match(wb[i, :wc[i]], tb[i, :tc[i]])
            matched += k
            worst = min(worst, lo if lo is not None else 1.0)
        det.predict_device = lambda b, tile_size=None, margin=None, m=m: orig(b, tile_size=2048, margin=m)
        try:
            words = pipe.recognize(pages)
        finally:
            det.predict_device = orig
        same = 0
        for a, b in zip(ref_words, words):
            same += sum((collections.Counter(t for t, _ in a) & collections.Counter(t for t, _ in b)).values())
        rows.append({"margin": m, "max_abs_score_diff": diff, "boxes_whole": int(np.sum(wc)), "boxes_tiled": int(np.sum(tc)),
                     "matched": matched, "min_iou": round(worst, 4),
                     "words_whole": sum(len(a) for a in ref_words), "same_texts": same})
        torch.cuda.synchronize()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--part", choices=("perf", "margins", "all"), default="all")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    from keras_ocr_b200 import weights as W
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    from keras_ocr_b200.recognition import Recognizer
    from scripts.bench_polygons import card

    det = Detector(weights=W.synthetic_craft_weights(3, textlike=True), device=0)
    rec = Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True), device=0)
    line = {"card": None, "power_limit": None, "weights": "synthetic textlike CRAFT, decisive CRNN"}
    if args.part in ("margins", "all"):
        line["margins"] = margins(Pipeline(detector=det, recognizer=rec, scale=2, max_size=3072))
    if args.part in ("perf", "all"):
        line["perf"] = perf(Pipeline(detector=det, recognizer=rec, scale=2, max_size=6144), args.rounds)
    line["card"], line["power_limit"] = card()
    text = json.dumps(line)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
