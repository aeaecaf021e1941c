"""Cost and effect of hotwords (``hotwords=``, ``b2o_crnn_forward_beam_hotword``).

Timing.  The decoder alone: ``b2o_ctc_beam_hotword_decode`` without and with a language model against
``b2o_ctc_beam_decode`` and ``b2o_ctc_beam_lm_decode`` on 1024 crops of seeded logits (K = 37), W in {16, 128}, lists
of 100 and 10^5 pseudo-language words, CUDA events around 10 calls after a warm-up.  End to end: ``Pipeline.recognize``
on bench.py's 32 pages with ``beam_width=16``, with and without hotwords (a list of the page words and a distractor
list of 10^5 words that matches none of them), alternated in one process; median ms per call and its spread (min-max)
over R rounds.

Accuracy.  Exact reads (``window_refs.exact_reads``) on the degraded pseudo-language pages of tests/test_gpu_lm.py at
its ``SEVERITY``, split into listed and unlisted words.  The list ("names") is the page words that are not in the
language model's 20k-word corpus.  Modes: beam 16, + hotwords, + the model, + the model and hotwords, a hard lexicon of
the names, and beam 16 + a distractor list of 10^5 words that are not on the pages.  Tuning: the weight sweep on the
tuning seeds (100..103) that picks ``Hotwords.WEIGHT``; the report is on the tests' held-out seeds.  Clean bench.py
pages: rendered words read exactly with and without a list of their words.  The card's name and power limit are read
in the same run.  Writes the JSON line to stdout and, with --out, to a file."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TUNING_SEEDS = (100, 101, 102, 103)
WEIGHTS = (0.25, 0.5, 1.0, 1.5, 2.0, 3.0, 5.0)


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
    from keras_ocr_b200.recognition import DEFAULT_ALPHABET as A, CharLM, Hotwords, Lexicon, Recognizer
    from scripts.bench_polygons import card
    from tests import window_refs as R
    from tests.test_gpu_beam import crafted
    from tests.test_gpu_lm import SEVERITY, TEST_SEEDS, pseudo_pages, pseudo_words

    assert torch.cuda.is_available(), "bench_hotwords measures on the GPU"
    pipe = Pipeline(detector=Detector(weights=W.synthetic_craft_weights(3, textlike=True), device=0),
                    recognizer=Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True), device=0), scale=2)
    rec = pipe.recognizer
    corpus = pseudo_words(77, 20000, A[10:], sample_seed=1)
    seen = set(corpus)
    lm = CharLM.fit(corpus, A, order=5)
    line = {"card": None, "power_limit": None, "rounds": args.rounds}
    tune, test = pseudo_pages(TUNING_SEEDS), pseudo_pages(TEST_SEEDS)
    on_pages = {w for pg in (tune, test) for it in pg[1] for w, _ in it}
    rng = np.random.default_rng(3)                  # 10^5 random letter strings of 4..8 characters, none on a page
    draws = {"".join(A[10 + c] for c in rng.integers(0, 26, int(n))) for n in rng.integers(4, 9, 120000)}
    distractors = sorted(draws - on_pages)[:100000]
    far = Hotwords(distractors, alphabet=A)

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

    # ---- the decoder alone
    ctx, stream = rec.ctx, torch.cuda.current_stream().cuda_stream
    x = torch.from_numpy(crafted(37, 1024, seed=5)).cuda()
    labels = torch.empty((1024, 4, 48), dtype=torch.int32, device="cuda")
    logp = torch.empty((1024, 4), dtype=torch.float32, device="cuda")
    lmd = lm.descriptor("cuda:0")
    lists = {"100": Hotwords(sorted(set(pseudo_words(5, 100, A[10:], sample_seed=4))), alphabet=A), "1e5": far}
    kernel = {}
    for w in (16, 128):
        entry = {"beam": timed(lambda: ctx.ctc_beam_decode(x.data_ptr(), 1024, 37, w, 4, labels.data_ptr(),
                                                           logp.data_ptr(), stream)),
                 "beam_lm": timed(lambda: ctx.ctc_beam_lm_decode(x.data_ptr(), 1024, 37, w, 4, lmd, labels.data_ptr(),
                                                                 logp.data_ptr(), None, stream))}
        for name, hw in lists.items():
            hd = hw.descriptor("cuda:0")
            entry[f"hotwords_{name}"] = timed(lambda: ctx.ctc_beam_hotword_decode(
                x.data_ptr(), 1024, 37, w, 4, None, hd, labels.data_ptr(), logp.data_ptr(), None, stream))
            entry[f"lm+hotwords_{name}"] = timed(lambda: ctx.ctc_beam_hotword_decode(
                x.data_ptr(), 1024, 37, w, 4, lmd, hd, labels.data_ptr(), logp.data_ptr(), None, stream))
        kernel[f"W={w}"] = entry
    line["decoder_1024_crops_k37"] = kernel

    # ---- end to end on bench.py's pages
    laid, page_words, page_rects = bench.make_pages(0, with_layout=True)
    pages = bench.make_pages(0)
    mine = Hotwords(sorted({w for ws in page_words for w in ws}), alphabet=A)      # every rendered word, listed
    modes = {"beam16": {"beam_width": 16}, "beam16+hotwords_page_words": {"beam_width": 16, "hotwords": mine},
             "beam16+hotwords_1e5_distractors": {"beam_width": 16, "hotwords": far}}
    for kw in modes.values():
        pipe.recognize(pages, recognition_kwargs=kw)
    times = {m: [] for m in modes}
    for _ in range(args.rounds):
        for m, kw in modes.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pipe.recognize(pages, recognition_kwargs=kw)
            torch.cuda.synchronize()
            times[m].append((time.perf_counter() - t0) * 1e3)
    line["bench_pages_ms"] = {m: {"median_ms": round(statistics.median(v), 2), "min_ms": round(min(v), 2),
                                  "max_ms": round(max(v), 2)} for m, v in times.items()}
    clean = {}
    for m, kw in modes.items():
        clean[m], clean["rendered"] = bench.words_read(pipe.recognize(laid, recognition_kwargs=kw), page_words,
                                                        page_rects)
    line["bench_pages_exact"] = clean

    # ---- degraded pseudo-language pages
    def split(pg, names, kw):
        res = pipe.recognize(pg[0], recognition_kwargs=kw)
        out = {"unlisted": 0, "listed": 0}
        for g, it in zip(res, pg[1]):
            out["listed"] += R.exact_reads(g, [(w, c) for w, c in it if w in names])
            out["unlisted"] += R.exact_reads(g, [(w, c) for w, c in it if w not in names])
        return out

    def table(pg, weight):
        names = sorted({w for it in pg[1] for w, _ in it if w not in seen})
        hw = Hotwords(names, weight=weight, alphabet=A)
        return {"words": sum(len(it) for it in pg[1]), "names": len(names),
                "listed_on_pages": sum(w in set(names) for it in pg[1] for w, _ in it),
                "beam16": split(pg, set(names), {"beam_width": 16}),
                "beam16+hotwords": split(pg, set(names), {"beam_width": 16, "hotwords": hw}),
                "beam16+lm": split(pg, set(names), {"beam_width": 16, "language_model": lm}),
                "beam16+lm+hotwords": split(pg, set(names), {"beam_width": 16, "language_model": lm, "hotwords": hw}),
                "lexicon_of_names": split(pg, set(names), {"lexicon": Lexicon(names, A)}),
                "beam16+distractors_1e5": split(pg, set(names), {"beam_width": 16, "hotwords": far.weighted(weight)})}

    sweep = {}
    for wt in WEIGHTS:
        names = sorted({w for it in tune[1] for w, _ in it if w not in seen})
        hw = Hotwords(names, weight=wt, alphabet=A)
        sweep[str(wt)] = {"beam16+hotwords": split(tune, set(names), {"beam_width": 16, "hotwords": hw}),
                          "beam16+lm+hotwords": split(tune, set(names), {"beam_width": 16, "language_model": lm,
                                                                         "hotwords": hw})}
    line["severity"] = SEVERITY
    line["tuning_sweep"] = sweep
    line["tuning_default_weight"] = table(tune, Hotwords.WEIGHT)
    line["held_out_default_weight"] = table(test, Hotwords.WEIGHT)
    report(line, args.out, card)


def report(line, out, card):
    line["card"], line["power_limit"] = card()
    text = json.dumps(line)
    print(text)
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
