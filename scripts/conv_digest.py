"""conv_digest.py -- SHA-256 digests of what the convolutions compute on bench.py's 32 seeded pages.

    python scripts/conv_digest.py

Prints one JSON line with digests of the detector's score maps (``Detector.predict_device`` on the step's resized and
padded batch), of the recognizer's fc_12 logits for the step's crops (``Recognizer.tap("logits")``) and of the arrays
``bench.py --dump-outputs`` writes.  Two builds that compute the same bits print the same digests.  Writes nothing.
"""
import hashlib
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def sha(a):
    return hashlib.sha256(a.tobytes()).hexdigest()


def main():
    import numpy as np
    import torch

    import bench
    from keras_ocr_b200 import weights as W
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    from keras_ocr_b200.recognition import STEPS, Recognizer

    assert torch.cuda.is_available(), "conv_digest.py needs a CUDA device"
    det = Detector(weights=W.synthetic_craft_weights(3, textlike=True), device=0)
    rec = Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True), device=0)
    pipe = Pipeline(detector=det, recognizer=rec, scale=bench.SCALE, max_size=2048)
    pages = torch.from_numpy(bench.make_pages(0)).to(torch.device("cuda", 0))

    batch, _ = pipe.prepare_device(pages)
    scores = det.predict_device(batch).cpu().numpy()
    result = pipe.recognize(pages)
    rec.keep_workspace = True
    again = pipe.recognize(pages)
    crops = sum(len(g) for g in result)
    logits = rec.tap("logits", (crops, STEPS, len(rec.alphabet) + 1), torch.float32).cpu().numpy()
    rec.keep_workspace = False
    out = {"scores": sha(scores), "scores_shape": list(scores.shape), "logits": sha(logits),
           "logits_shape": list(logits.shape),
           "same_words_with_logits_kept": [t for g in again for t, _ in g] == [t for g in result for t, _ in g]}
    with tempfile.TemporaryDirectory() as tmp:
        bench.dump_outputs(result, tmp)
        for name in sorted(os.listdir(tmp)):
            out["dump/" + name] = sha(np.load(os.path.join(tmp, name)))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
