"""Development timing probe (not the benchmark): CRAFT / CRNN forward times on one GPU."""
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from keras_ocr_b200 import _lib, weights as W
from keras_ocr_b200.detection import Detector
from keras_ocr_b200.recognition import Recognizer


def timeit(fn, warm=2, iters=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def main():
    n, h, w = int(os.environ.get("N", 4)), int(os.environ.get("H", 768)), int(os.environ.get("W", 768))
    iters = int(os.environ.get("ITERS", 5))
    det = Detector(weights=W.synthetic_craft_weights(3))
    rng = np.random.default_rng(0)
    img = torch.from_numpy(rng.integers(0, 256, (n, h, w, 3), dtype=np.uint8)).cuda()
    for name, eng in (("tc", _lib.CONV_AUTO),) + ((("simt", _lib.CONV_SIMT),) if os.environ.get("SIMT") else ()):
        det.ctx.set_conv_engine(eng)
        try:
            ms = timeit(lambda: det.predict_device(img), 2, iters)
            flop = W.CRAFT_FLOP_PER_PIXEL * n * h * w
            print(f"CRAFT {name}: {n}x{h}x{w}: {ms:.3f} ms  -> {flop / ms / 1e9:.1f} TFLOP/s, {n / ms * 1e3:.1f} img/s")
        except Exception as e:  # noqa
            print(f"CRAFT {name} FAILED: {e}")
    det.ctx.set_conv_engine(_lib.CONV_AUTO)
    rec = Recognizer(weights=W.synthetic_crnn_weights(2))
    b = int(os.environ.get("B", 256))
    x = torch.rand((b, 200, 31), device="cuda").half()
    try:
        ms = timeit(lambda: rec.predict_device(x), 2, iters)
        print(f"CRNN: {b} crops: {ms:.3f} ms -> {W.CRNN_FLOP_PER_CROP * b / ms / 1e9:.1f} TFLOP/s, {b / ms * 1e3:.0f} crops/s")
    except Exception as e:  # noqa
        print(f"CRNN FAILED: {e}")


if __name__ == "__main__":
    main()
