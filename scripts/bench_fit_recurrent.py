"""Measure fine-tuning the recognizer's recurrent head on the GPU: the sequence-features pass
(``b2o_crnn_sequence_features``) in crops/s at batch 256, and one optimizer step (``b2o_rnn_loss_grad`` with dropout 0.25
+ one ``b2o_rmsprop_step`` over all 14 tensors) at batch 64 and 256, K = 38.  Timed with CUDA events after warm-up;
prints the card's name and power limit, read in the same run, and one JSON line.

    python scripts/bench_fit_recurrent.py [--iters 50]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from keras_ocr_b200 import weights as W  # noqa: E402
from keras_ocr_b200.recognition import Recognizer  # noqa: E402
from scripts.bench_fit_top import card, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    k, rows = 38, 4096
    stream = lambda: torch.cuda.current_stream().cuda_stream      # noqa: E731
    rec = Recognizer(alphabet="".join(chr(0x4E00 + i) for i in range(k - 1)), weights=W.synthetic_crnn_weights(seed=1))
    ctx = rec.ctx
    out = {"k": k}
    b = 256
    crnn_in = torch.rand((b, 200, 31), device="cuda").half()
    seq = torch.empty((rows, 50, 128), dtype=torch.float16, device="cuda")
    nbytes = ctx.crnn_workspace_bytes(b)
    ws = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    sec = timed(lambda: ctx.crnn_sequence_features(crnn_in.data_ptr(), b, seq.data_ptr(), ws.data_ptr(), nbytes,
                                                   stream()), args.iters)
    out["sequence_features_crops_per_s"] = b / sec
    seq.copy_(torch.relu(torch.randn_like(seq, dtype=torch.float32)).half())
    names = rec._rnn_tensor_names()
    params = torch.from_numpy(np.concatenate([np.asarray(rec._tensors[n], np.float32).reshape(-1)
                                              for n, _ in names])).cuda()
    acc, grad = torch.zeros_like(params), torch.empty_like(params)
    rng = np.random.default_rng(0)
    for b in (64, 256):
        lengths = rng.integers(3, 11, b)
        off = torch.from_numpy(np.concatenate([[0], np.cumsum(lengths)]).astype(np.int32)).cuda()
        lab = torch.from_numpy(rng.integers(0, k - 1, int(lengths.sum())).astype(np.int16)).cuda()
        index = torch.from_numpy(rng.permutation(rows)[:b].astype(np.int32)).cuda()
        loss = torch.empty(b, device="cuda")
        tb = ctx.rnn_train_workspace_bytes(b, k)
        tws = torch.empty(tb, dtype=torch.uint8, device="cuda")
        step = [0]

        def opt_step():
            ctx.rnn_loss_grad(seq.data_ptr(), rows, index.data_ptr(), b, k, params.data_ptr(), off.data_ptr(),
                              lab.data_ptr(), 0.25, 0, step[0], loss.data_ptr(), grad.data_ptr(), tws.data_ptr(), tb,
                              stream())
            ctx.rmsprop_step(params.data_ptr(), grad.data_ptr(), acc.data_ptr(), params.numel(), 1e-3, 0.9, 1e-7,
                             stream())
            step[0] += 1
        sec = timed(opt_step, args.iters)
        out[f"optimizer_step_ms_b{b}"] = sec * 1e3
        out[f"workspace_mb_b{b}"] = tb / 2 ** 20
        assert np.isfinite(loss.cpu().numpy()).all()
    name, limit = card()
    out["gpu"], out["power_limit"] = name, limit
    print(f"{name}, power limit {limit}: " + ", ".join(f"{k} {v:.4g}" if isinstance(v, float) else f"{k} {v}"
                                                       for k, v in out.items() if k not in ("gpu", "power_limit")))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
