"""Detector: drop-in for ``keras_ocr.detection.Detector`` (reference detection.py:661-785).

``detect`` keeps the reference signature and return type; the work is done by the CUDA library:
compute_input + CRAFT forward (``b2o_craft_forward``) and getBoxes (``b2o_get_boxes``).
"""
import typing

import numpy as np
import torch

from . import _lib, tools, weights as weights_mod

PRETRAINED_WEIGHTS = {   # same files as reference detection.py:647-658
    ("clovaai_general", True): {
        "filename": "craft_mlt_25k.pth",
        "sha256": "4a5efbfb48b4081100544e75e1e2b57f8de3d84f213004b14b85fd4b3748db17",
    },
}


def _as_device_images(images, device):
    """list / ndarray / tensor of HxWx3 uint8 -> (N,H,W,3) uint8 CUDA tensor."""
    if isinstance(images, torch.Tensor):
        t = images
    else:
        arr = np.ascontiguousarray(np.array([tools.read(image) for image in images]))
        t = torch.from_numpy(arr)
    assert t.dim() == 4 and t.shape[-1] == 3, "images must be (N, H, W, 3)"
    assert t.dtype == torch.uint8, "images must be uint8 RGB"
    if not t.is_cuda:
        t = t.pin_memory().to(device, non_blocking=True)
    return t.contiguous()


class Detector:
    """A text detector using the CRAFT architecture, running as sm_90a CUDA kernels.

    Args:
        weights: ``"clovaai_general"`` (reads ``craft_mlt_25k.pth`` from the keras-ocr cache dir),
            a path to a ``.pth`` / ``.npz`` file, or a dict of tensors keyed like the ``.pth``
            (see ``weights.py``).
        load_from_torch, optimizer, backbone_name: accepted for signature compatibility; only the
            ``vgg`` backbone exists (reference detection.py:363 raises NotImplementedError otherwise).
        device: CUDA device index (default: current device).
    """

    def __init__(self, weights="clovaai_general", load_from_torch=False, optimizer="adam",
                 backbone_name="vgg", device=None):
        if backbone_name != "vgg":
            raise NotImplementedError
        if not torch.cuda.is_available():
            raise _lib.B2OError("keras-ocr_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        self.device_index = torch.cuda.current_device() if device is None else int(device)
        self.device = torch.device("cuda", self.device_index)
        if isinstance(weights, dict):
            tensors = weights
        elif isinstance(weights, str) and weights.endswith(".pth"):
            tensors = weights_mod.load_craft_pth(weights)
        elif isinstance(weights, str) and weights.endswith(".npz"):
            tensors = weights_mod.load_npz(weights)
        elif weights == "clovaai_general":
            cfg = PRETRAINED_WEIGHTS[("clovaai_general", True)]
            tensors = weights_mod.load_craft_pth(tools.find_cached(cfg["filename"], cfg["sha256"]))
        else:
            raise NotImplementedError(f"Cannot load weights from {weights}")
        self.ctx = _lib.Context(self.device_index)
        self.ctx.load_craft(tensors)
        self.max_boxes = 256
        self._ws = None                  # reusable CRAFT workspace (grown on demand)
        self._box_ws = None

    # ------------------------------------------------------------------ device-resident API
    def predict_device(self, images_t):
        """CRAFT forward.  images_t: (N,H,W,3) uint8 CUDA tensor -> (N,H/2,W/2,2) float32 scores."""
        n, h, w, _ = images_t.shape
        stream = torch.cuda.current_stream(self.device).cuda_stream
        scores = torch.empty((n, h // 2, w // 2, 2), dtype=torch.float32, device=self.device)
        nbytes = self.ctx.craft_workspace_bytes(n, h, w)
        assert nbytes > 0, "image too small for CRAFT (needs H, W >= 32)"
        if self._ws is None or self._ws.numel() < nbytes:
            self._ws = None
            self._ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        ws = self._ws
        self.ctx.craft_forward(images_t.data_ptr(), n, h, w, scores.data_ptr(), ws.data_ptr(), nbytes, stream)
        return scores

    def boxes_enqueue(self, scores, detection_threshold=0.7, text_threshold=0.4, link_threshold=0.4,
                      size_threshold=10, with_scores=False):
        """getBoxes on the device, asynchronously: launches the kernels and the copy of the per-image counts into
        pinned memory, records an event and returns at once (``boxes_finish`` waits for that event only, so work
        enqueued afterwards keeps the GPU busy while the host reads the counts).  ``with_scores``: the state also
        holds ``box_scores`` (N,M) float32 CUDA, each box's detection score (``b2o_get_boxes_scored``)."""
        n, hs, ws_, _ = scores.shape
        stream = torch.cuda.current_stream(self.device)
        scores = scores.contiguous()
        m = self.max_boxes
        boxes = torch.empty((n, m, 4, 2), dtype=torch.float32, device=self.device)
        counts = torch.empty((n,), dtype=torch.int32, device=self.device)
        nbytes = self.ctx.boxes_workspace_bytes(n, hs, ws_, m)
        if self._box_ws is None or self._box_ws.numel() < nbytes:
            self._box_ws = None
            self._box_ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        wsp = self._box_ws
        thr = (float(detection_threshold), float(text_threshold), float(link_threshold), int(size_threshold))
        box_scores = None
        if with_scores:
            box_scores = torch.empty((n, m), dtype=torch.float32, device=self.device)
            self.ctx.get_boxes_scored(scores.data_ptr(), n, hs, ws_, *thr, boxes.data_ptr(), counts.data_ptr(),
                                      box_scores.data_ptr(), m, wsp.data_ptr(), nbytes, stream.cuda_stream)
        else:
            self.ctx.get_boxes(scores.data_ptr(), n, hs, ws_, *thr, boxes.data_ptr(), counts.data_ptr(), m,
                               wsp.data_ptr(), nbytes, stream.cuda_stream)
        counts_pin = torch.empty((n,), dtype=torch.int32, pin_memory=True)
        counts_pin.copy_(counts, non_blocking=True)
        event = torch.cuda.Event()
        event.record(stream)
        # recognize_from_boxes' bookkeeping (dense box list + image index, recognition.py:511-521) is queued
        # behind the counts copy: it needs no host knowledge, so it runs while the host still waits for the event
        flat = torch.empty((n * m, 4, 2), dtype=torch.float32, device=self.device)
        image_index = torch.empty((n * m,), dtype=torch.int32, device=self.device)
        self.ctx.compact_boxes(boxes.data_ptr(), counts.data_ptr(), n, m, flat.data_ptr(), image_index.data_ptr(),
                               stream.cuda_stream)
        return {"scores": scores, "boxes": boxes, "counts": counts, "counts_pin": counts_pin, "event": event, "m": m,
                "thr": thr, "flat": flat, "image_index": image_index, "box_scores": box_scores}

    def boxes_finish(self, state):
        """Wait for ``boxes_enqueue``.  Returns (boxes (N,M,4,2) float32 CUDA, counts ndarray (N,)); re-runs
        getBoxes with a larger box table in the (rare) case an image had more boxes than the table holds (the state's
        ``box_scores``, when asked for, then come from that run too)."""
        state["event"].synchronize()                     # the one synchronisation of the detector half
        counts_host = state["counts_pin"].numpy().copy()
        while counts_host.size and int(counts_host.max()) > state["boxes"].shape[1]:
            self.max_boxes = int(2 ** np.ceil(np.log2(int(counts_host.max()))))
            d, t, l, s = state["thr"]
            again = self.boxes_enqueue(state["scores"], d, t, l, s, with_scores=state["box_scores"] is not None)
            again["event"].synchronize()
            state.update(again)
            counts_host = state["counts_pin"].numpy().copy()
        return state["boxes"], counts_host

    def boxes_device(self, scores, detection_threshold=0.7, text_threshold=0.4, link_threshold=0.4,
                     size_threshold=10):
        """getBoxes on the device.  Returns (boxes (N,M,4,2) float32 CUDA, counts ndarray (N,))."""
        return self.boxes_finish(self.boxes_enqueue(scores, detection_threshold, text_threshold, link_threshold,
                                                    size_threshold))

    def detect_device(self, images_t, **thresholds):
        return self.boxes_device(self.predict_device(images_t), **thresholds)

    # ------------------------------------------------------------------ reference API
    def detect(self, images: typing.List[typing.Union[np.ndarray, str]], detection_threshold=0.7,
               text_threshold=0.4, link_threshold=0.4, size_threshold=10, return_scores=False, **kwargs):
        """Same contract as reference detection.py:745-785: a list with one array of boxes
        ``(n_i, 4, 2)`` float32 per image (``np.array([])`` when there is none).  ``kwargs`` are the
        keras ``predict`` arguments of the reference (batch_size, verbose, ...) and are ignored.

        ``return_scores=True``: one ``(boxes, scores)`` pair per image instead, ``scores`` (n_i,) float32 the
        detection score of each box -- the largest text score over its connected component, the value compared
        with ``detection_threshold`` (so every score is >= it)."""
        images_t = _as_device_images(images, self.device)
        state = self.boxes_enqueue(self.predict_device(images_t), detection_threshold, text_threshold, link_threshold,
                                   size_threshold, with_scores=return_scores)
        boxes, counts = self.boxes_finish(state)
        boxes_host = boxes.cpu().numpy()
        groups = [boxes_host[i, :c].copy() if c else np.array([]) for i, c in enumerate(counts)]
        if not return_scores:
            return groups
        scores_host = state["box_scores"].cpu().numpy()
        return [(g, scores_host[i, :c].copy()) for i, (g, c) in enumerate(zip(groups, counts))]
