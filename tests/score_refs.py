"""References for detection scores and word confidences, built on the oracle's own outputs.

* ``box_scores``: the oracle's ``getBoxes`` (``imageops.get_boxes_single``) keeps a component when its largest text score
  reaches the detection threshold (reference detection.py:240-241); the score of each kept box is that maximum, read
  from the component labels and the kept label ids the oracle reports through its ``debug`` dict, in box order.
* ``path_logprob``: the greedy CTC path's log-probability S = sum_t log(max_c p[t,c] + 1e-7) in float64 from a softmax
  (B,T,K) such as ``oracle.crnn.crnn_logits`` returns.  Per TensorFlow's documentation S is minus the second output of
  ``keras.backend.ctc_decode(greedy=True)``, which the reference's ``CTCDecoder`` drops (recognition.py:175); that link
  is not pinned against TensorFlow.
"""
import numpy as np
import torch


def box_scores(scores, **thresholds):
    """(quads, (n,) float32 detection score of each box) of the oracle's getBoxes on one (h, w, 2) map."""
    from oracle import imageops
    debug = {}
    quads = imageops.get_boxes_single(scores, debug=debug, **thresholds)
    text, labels = scores[..., 0], debug["labels"]
    return quads, np.array([text[labels == cid].max() for cid in debug["kept"]], dtype=np.float32)


def path_logprob(probs):
    """(B,) float64 log-probability of the greedy path of a (B,T,K) softmax."""
    p = torch.as_tensor(probs).double()
    return torch.log(p.max(-1).values + 1e-7).sum(-1).numpy()
