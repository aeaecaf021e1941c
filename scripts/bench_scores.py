"""bench_scores.py -- what detection scores, word confidences, beam-search, lexicon decoding and quarter-turn reading
cost: ``Pipeline.recognize`` with and without ``return_scores=True``, with ``recognition_kwargs={"beam_width": W}`` for
every W given, with ``recognition_kwargs={"lexicon": L}`` for every lexicon size N given and with
``recognition_kwargs={"rotations": T, "rotation_vote": V}`` for every turn list T and vote V given, on the workload of
bench.py (32 pages 768x768, scale 2 -> 1536x1536, sources resident in HBM).  A size-N lexicon is the bench pages'
rendered words plus seeded distractors (``oracle.synth.random_word``) up to N entries.

    python scripts/bench_scores.py [--steps K] [--warmup W] [--rounds R] [--beam-width W [W ...]]
                                   [--lexicon-size N [N ...]] [--decoder-lexicon-size N [N ...]] [--decoder-calls C]
                                   [--rotations 02 0123 ...] [--rotation-vote word page] [--rotation-beam-width W ...]

``--rotations``: turn lists as digit strings (``02`` = (0, 2)), each timed with every ``--rotation-vote`` (default
page), greedy and with every ``--rotation-beam-width``.  Besides the words read on the upright pages, the line then reports ``words_read`` of the default call and of
every rotation leg on the pages turned by np.rot90(page, k), k = 1, 2, 3 (outside the timed region).

``--char-boxes``: also ``recognize(return_char_boxes=True)`` (leg ``char_boxes``) and every rotation leg with it
(``<leg>_char_boxes``): the cost of locating every character (alignment, cells, and the greedy forward's logits).

``--decoder-lexicon-size``: the lexicon decoder alone (``b2o_ctc_lexicon_decode``, top_paths 1) on the fc_12 logits
of one bench step's crops, C launches between CUDA events after a warm-up, in ms per call.

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


def rot90_rect(rect, k, h, w):
    """(x0, y0, x1, y1) of an (h, w) page on np.rot90(page, k): (x, y) -> (y, w - 1 - x), applied k times."""
    x0, y0, x1, y1 = rect
    for _ in range(k):
        x0, y0, x1, y1 = y0, w - 1 - x1, y1, w - 1 - x0
        h, w = w, h
    return x0, y0, x1, y1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--beam-width", type=int, nargs="+", default=[])
    ap.add_argument("--lexicon-size", type=int, nargs="+", default=[])
    ap.add_argument("--decoder-lexicon-size", type=int, nargs="+", default=[])
    ap.add_argument("--decoder-calls", type=int, default=20)
    ap.add_argument("--rotations", nargs="+", default=[], help="turn lists as digit strings, e.g. 02 0123")
    ap.add_argument("--rotation-vote", nargs="+", default=["page"], choices=["word", "page"])
    ap.add_argument("--rotation-beam-width", type=int, nargs="+", default=[],
                    help="also time every rotation leg with beam search of these widths")
    ap.add_argument("--char-boxes", action="store_true", help="also time return_char_boxes=True")
    args = ap.parse_args()

    import numpy as np
    import torch

    import bench
    from keras_ocr_b200 import weights as W
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    from keras_ocr_b200.recognition import Lexicon, Recognizer
    from oracle import synth

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

    def lexicon(n):
        words = list(dict.fromkeys(w for page in page_words for w in page))[:n]
        seen, rng = set(words), np.random.default_rng(n)
        while len(words) < n:
            w = synth.random_word(rng)
            if w not in seen:
                seen.add(w)
                words.append(w)
        return Lexicon(words, rec.alphabet)

    lexicons = {n: lexicon(n) for n in sorted(set(args.lexicon_size) | set(args.decoder_lexicon_size))}
    for n in args.lexicon_size:
        calls[f"lexicon{n}"] = lambda n=n: pipe.recognize(pages, recognition_kwargs={"lexicon": lexicons[n]})
    rotation_kwargs = {}
    for spec in args.rotations:
        for vote in args.rotation_vote:
            rotation_kwargs[f"rot{spec}_{vote}"] = {"rotations": tuple(int(c) for c in spec), "rotation_vote": vote}
            for w in args.rotation_beam_width:
                rotation_kwargs[f"rot{spec}_{vote}_beam{w}"] = dict(rotation_kwargs[f"rot{spec}_{vote}"], beam_width=w)
    for name, kw in rotation_kwargs.items():
        calls[name] = lambda kw=kw, imgs=pages: pipe.recognize(imgs, recognition_kwargs=kw)
    with_cells = set()
    if args.char_boxes:
        calls["char_boxes"] = lambda: pipe.recognize(pages, return_char_boxes=True)
        with_cells.add("char_boxes")
        for name, kw in rotation_kwargs.items():
            calls[f"{name}_char_boxes"] = lambda kw=kw: pipe.recognize(pages, recognition_kwargs=kw, return_char_boxes=True)
            with_cells.add(f"{name}_char_boxes")

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
        if k in with_cells:                              # (text, box, cells) -> (text, box)
            result = [[w[:2] for w in g] for g in result]
        hit, rendered = bench.words_read(result, page_words, page_rects)
        line[f"{k}_words_read"] = [hit, rendered]
        if k != "default":
            line[f"{k}_ms_per_step"] = statistics.median(ms[k])
            line[f"{k}_ms_spread"] = [min(ms[k]), max(ms[k])]
            line[f"{k}_overhead"] = statistics.median(ms[k]) / statistics.median(ms["default"]) - 1.0
            line[f"{k}_words_differing_from_default"] = sum(a != b for a, b in zip([t for g in result for t, _ in g],
                                                                                  default_words))
    if rotation_kwargs:                                  # accuracy on the pages turned by np.rot90(page, k), untimed
        for k in (1, 2, 3):
            turned = torch.from_numpy(np.ascontiguousarray(np.rot90(pages_host, k, axes=(1, 2)))).to(device)
            rects = [[rot90_rect(r, k, bench.PAGE_H, bench.PAGE_W) for r in page] for page in page_rects]
            legs = {"default": {}, **rotation_kwargs}
            for name, kw in legs.items():
                hit, rendered = bench.words_read(pipe.recognize(turned, recognition_kwargs=kw), page_words, rects)
                line[f"{name}_words_read_rot90_k{k}"] = [hit, rendered]
    if args.decoder_lexicon_size:
        rec.keep_workspace = True
        n_crops = sum(len(g) for g in pipe.recognize(pages))
        logits = rec.tap("logits", (n_crops, 48, len(rec.alphabet) + 1), torch.float32)
        rec.keep_workspace = False
        line["decoder_crops"] = n_crops
        for n in args.decoder_lexicon_size:
            off, lab = lexicons[n].device_arrays(device)
            out = torch.empty((n_crops, 1, 48), dtype=torch.int32, device=device)
            logp = torch.empty((n_crops, 1), dtype=torch.float32, device=device)
            nbytes = rec.ctx.lexicon_workspace_bytes(n_crops, n, 1)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
            stream = torch.cuda.current_stream(device).cuda_stream

            def call():
                rec.ctx.ctc_lexicon_decode(logits.data_ptr(), n_crops, logits.shape[2], off.data_ptr(), lab.data_ptr(), n,
                                           1, out.data_ptr(), logp.data_ptr(), ws.data_ptr(), nbytes, stream)
            for _ in range(3):
                call()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.decoder_calls):
                call()
            e1.record()
            torch.cuda.synchronize()
            line[f"decoder_lexicon{n}_ms_per_call"] = e0.elapsed_time(e1) / args.decoder_calls
    print(json.dumps(line))


if __name__ == "__main__":
    main()
