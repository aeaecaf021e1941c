"""Measure training the recognizer's output layer on the GPU: the features pass (``b2o_crnn_features``) in crops/s and
the optimizer step (``b2o_ctc_loss_grad`` with dropout 0.25 + two ``b2o_rmsprop_step``) in steps/s at batch 256, for
K = 38 and K = 1024 classes.  Timed with CUDA events after warm-up; prints the card's name and power limit, read in the
same run, and one JSON line.

    python scripts/bench_fit_top.py [--iters 50]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from keras_ocr_b200 import weights as W  # noqa: E402
from keras_ocr_b200.recognition import Recognizer  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return name, limit


def timed(fn, iters, warmup=5):
    for _ in range(warmup):
        fn()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) / iters / 1e3            # seconds per call


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    b, rows = 256, 4096
    stream = lambda: torch.cuda.current_stream().cuda_stream      # noqa: E731
    out = {"batch": b}
    for k in (38, 1024):
        alphabet = "".join(chr(0x4E00 + i) for i in range(k - 1))
        rec = Recognizer(alphabet=alphabet, weights=W.synthetic_crnn_weights(seed=1))
        ctx = rec.ctx
        crnn_in = torch.rand((b, 200, 31), device="cuda").half()
        feats = torch.empty((rows, 48, 256), dtype=torch.float16, device="cuda")
        nbytes = ctx.crnn_workspace_bytes(b)
        ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
        sec = timed(lambda: ctx.crnn_features(crnn_in.data_ptr(), b, feats.data_ptr(), ws.data_ptr(), nbytes, stream()),
                    args.iters)
        out[f"features_crops_per_s_k{k}"] = b / sec
        feats.copy_(torch.tanh(torch.randn_like(feats, dtype=torch.float32)).half())
        rng = np.random.default_rng(0)
        lengths = rng.integers(3, 11, b)
        off = torch.from_numpy(np.concatenate([[0], np.cumsum(lengths)]).astype(np.int32)).cuda()
        lab = torch.from_numpy(rng.integers(0, k - 1, int(lengths.sum())).astype(np.int16)).cuda()
        index = torch.from_numpy(rng.permutation(rows)[:b].astype(np.int32)).cuda()
        w = torch.randn((256, k), device="cuda") * 0.05
        bias = torch.zeros(k, device="cuda")
        acc_w, acc_b = torch.zeros_like(w), torch.zeros_like(bias)
        gw, gb = torch.empty_like(w), torch.empty_like(bias)
        loss = torch.empty(b, device="cuda")
        tb = ctx.ctc_train_workspace_bytes(b, k)
        tws = torch.empty(tb, dtype=torch.uint8, device="cuda")
        step = [0]

        def opt_step():
            ctx.ctc_loss_grad(feats.data_ptr(), rows, index.data_ptr(), b, k, w.data_ptr(), bias.data_ptr(),
                              off.data_ptr(), lab.data_ptr(), 0.25, 0, step[0], loss.data_ptr(), gw.data_ptr(),
                              gb.data_ptr(), None, tws.data_ptr(), tb, stream())
            ctx.rmsprop_step(w.data_ptr(), gw.data_ptr(), acc_w.data_ptr(), w.numel(), 1e-3, 0.9, 1e-7, stream())
            ctx.rmsprop_step(bias.data_ptr(), gb.data_ptr(), acc_b.data_ptr(), k, 1e-3, 0.9, 1e-7, stream())
            step[0] += 1
        sec = timed(opt_step, args.iters)
        out[f"optimizer_steps_per_s_k{k}"] = 1.0 / sec
        out[f"optimizer_step_ms_k{k}"] = sec * 1e3
        assert np.isfinite(loss.cpu().numpy()).all()
    name, limit = card()
    out["gpu"], out["power_limit"] = name, limit
    print(f"{name}, power limit {limit}: " + ", ".join(f"{k} {v:.4g}" if isinstance(v, float) else f"{k} {v}"
                                                       for k, v in out.items() if k not in ("gpu", "power_limit")))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
