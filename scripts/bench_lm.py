"""Cost and effect of the character language model (``language_model=``, ``b2o_crnn_forward_beam_lm``).

Timing.  The decoder alone: ``b2o_ctc_beam_lm_decode`` against ``b2o_ctc_beam_decode`` on 1024 crops of seeded logits
(K = 37), W in {4, 16, 64, 128}, an order-5 model of 20k pseudo-language words, CUDA events around 10 calls after a
warm-up.  End to end: ``Pipeline.recognize`` on bench.py's 32 pages with ``beam_width=16``, with and without the model,
alternated in one process; median ms per call and its spread (min-max) over R rounds.

Accuracy.  Exact reads (``window_refs.exact_reads``) on degraded pages of the seeded pseudo-language of
tests/test_gpu_lm.py (words of a random character trigram chain, rendered as ``window_refs.long_word_page`` renders,
blurred, faded and noised at the tests' ``SEVERITY``): greedy, beam 16, beam 16 + the model, and a lexicon of the
model's 20k-word corpus, which cannot read a word outside it.  Clean bench.py pages with a model fitted on unrelated
words (another chain): rendered words read exactly, as bench.py counts them, for greedy, beam 16 and beam 16 + that
model.  Tuning: the alpha, beta sweep on the tuning seeds (100..103, disjoint from the tests' test seeds) that picks
``CharLM.ALPHA`` / ``CharLM.BETA``.  ``--scan s1,s2,...``: only beam 16 and the sweep on the tuning seeds at each of
those severities, to choose one where beam search alone misreads words.  The card's name and power limit are read in
the same run.  Writes the JSON line to stdout and, with --out, to a file."""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TUNING_SEEDS = (100, 101, 102, 103)
ALPHAS, BETAS = (0.25, 0.5, 1.0, 1.5, 2.0), (0.0, 0.5, 1.0, 2.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    ap.add_argument("--scan", default=None, help="comma-separated severities: the tuning sweep at each, nothing else")
    args = ap.parse_args()
    import numpy as np
    import torch

    import bench
    from keras_ocr_b200 import weights as W
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    from keras_ocr_b200.recognition import DEFAULT_ALPHABET as A, CharLM, Lexicon, Recognizer
    from scripts.bench_polygons import card
    from tests import window_refs as R
    from tests.test_gpu_beam import crafted
    from tests.test_gpu_lm import SEVERITY, TEST_SEEDS, pseudo_pages, pseudo_words

    assert torch.cuda.is_available(), "bench_lm measures on the GPU"
    pipe = Pipeline(detector=Detector(weights=W.synthetic_craft_weights(3, textlike=True), device=0),
                    recognizer=Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True), device=0), scale=2)
    rec = pipe.recognizer
    corpus = pseudo_words(77, 20000, A[10:], sample_seed=1)
    lm = CharLM.fit(corpus, A, order=5)
    line = {"card": None, "power_limit": None, "rounds": args.rounds, "histories": int(lm.host_tables()[0].shape[0])}

    def exact(pages_items, kw):
        pg, items = pages_items
        res = pipe.recognize(pg, recognition_kwargs=kw)
        return sum(R.exact_reads(g, it) for g, it in zip(res, items))

    def sweep(tune):
        return {f"{a},{b}": exact(tune, {"beam_width": 16, "language_model": lm.weighted(a, b)})
                for a in ALPHAS for b in BETAS}

    if args.scan:
        for sev in (float(v) for v in args.scan.split(",")):
            tune = pseudo_pages(TUNING_SEEDS, severity=sev)
            line[f"severity={sev}"] = {"words": sum(len(it) for it in tune[1]), "beam16": exact(tune, {"beam_width": 16}),
                                       "sweep": sweep(tune)}
        return report(line, args.out, card)

    # ---- the decoder alone
    ctx, stream = rec.ctx, torch.cuda.current_stream().cuda_stream
    x = torch.from_numpy(crafted(37, 1024, seed=5)).cuda()
    labels = torch.empty((1024, 4, 48), dtype=torch.int32, device="cuda")
    logp = torch.empty((1024, 4), dtype=torch.float32, device="cuda")
    desc = lm.descriptor("cuda:0")
    kernel = {}
    for w in (4, 16, 64, 128):
        calls = {"beam": lambda w=w: ctx.ctc_beam_decode(x.data_ptr(), 1024, 37, w, 4, labels.data_ptr(),
                                                         logp.data_ptr(), stream),
                 "beam_lm": lambda w=w: ctx.ctc_beam_lm_decode(x.data_ptr(), 1024, 37, w, 4, desc, labels.data_ptr(),
                                                               logp.data_ptr(), None, stream)}
        entry = {}
        for name, call in calls.items():
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
            entry[name] = {"median_ms": round(statistics.median(reps), 3), "min_ms": round(min(reps), 3),
                           "max_ms": round(max(reps), 3)}
        kernel[f"W={w}"] = entry
    line["decoder_1024_crops_k37_order5"] = kernel

    # ---- end to end on bench.py's pages
    pages = bench.make_pages(0)
    modes = {"beam16": {"beam_width": 16}, "beam16+lm": {"beam_width": 16, "language_model": lm}}
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

    # ---- clean bench pages, read against the rendered words, with a model of unrelated words
    laid, page_words, page_rects = bench.make_pages(0, with_layout=True)
    other = CharLM.fit(pseudo_words(991, 20000, A[10:], sample_seed=2), A, order=5)
    clean = {}
    for m, kw in (("greedy", {}), ("beam16", {"beam_width": 16}),
                  ("beam16+unrelated_lm", {"beam_width": 16, "language_model": other}),
                  ("beam16+unrelated_lm_alpha0.5_beta0", {"beam_width": 16, "language_model": other.weighted(0.5, 0.0)})):
        clean[m], clean["rendered"] = bench.words_read(pipe.recognize(laid, recognition_kwargs=kw), page_words,
                                                        page_rects)
    line["clean_pages_exact"] = clean

    # ---- degraded pseudo-language pages: tuning sweep, then the test seeds
    tune = pseudo_pages(TUNING_SEEDS)
    sw = sweep(tune)
    line["severity"] = SEVERITY
    line["tuning_sweep_exact"] = sw
    line["tuning_beam16_exact"] = exact(tune, {"beam_width": 16})
    best = max(sw, key=lambda k: (sw[k], k == f"{CharLM.ALPHA},{CharLM.BETA}"))
    line["tuning_best"] = best
    test = pseudo_pages(TEST_SEEDS)
    words = sum(len(it) for it in test[1])
    lex = Lexicon(sorted(set(corpus)), A)
    line["degraded_test_pages"] = {
        "words": words, "unseen": sum(w not in set(corpus) for it in test[1] for w, _ in it),
        "greedy": exact(test, {}), "beam16": exact(test, {"beam_width": 16}),
        "beam16+lm_defaults": exact(test, {"beam_width": 16, "language_model": lm}),
        "beam16+lm_tuned": exact(test, {"beam_width": 16, "language_model": lm.weighted(*map(float, best.split(",")))}),
        "lexicon_of_corpus": exact(test, {"lexicon": lex})}
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
