"""Detector: drop-in for ``keras_ocr.detection.Detector`` (reference detection.py:661-785).

``detect`` keeps the reference signature and return type; the work is done by the CUDA library:
compute_input + CRAFT forward (``b2o_craft_forward``) and getBoxes (``b2o_get_boxes``).
"""
import math
import numbers
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


# Tiled detection (DESIGN.md section 1, "Tiles").  TILE_MARGIN: detector pixels of context kept on each inner side of a
# tile's core, the smallest margin at which the tiled forward's boxes and texts matched the whole page's (DESIGN.md
# section 5).  DEFAULT_TILE_SIZE: tile_size=None tiles a batch whose padded height is over it -- the batches the
# whole-page forward cannot take, as getBoxes once refused their score maps.  TILE_CHUNK_PIXELS: tiles per CRAFT launch
# are as many as fit this pixel count, which bounds the forward's workspace whatever the page size.
TILE_MARGIN = 64
DEFAULT_TILE_SIZE = 2048
MAX_TILE_SIZE = 2048
TILE_CHUNK_PIXELS = 8 * 2048 * 2048


def check_tiles(tile_size=None):
    """Validate ``tile_size`` (DESIGN.md section 1, "Tiles") and return it as an int, or None for the default rule: a
    multiple of 32 with 4 * TILE_MARGIN <= tile_size <= 2048.  Bools, non-integers and other values raise
    ``ValueError``."""
    if tile_size is None:
        return None
    if isinstance(tile_size, bool) or not isinstance(tile_size, numbers.Integral):
        raise ValueError(f"tile_size must be an integer or None, got {tile_size!r}")
    t = int(tile_size)
    if t % 32 or not 4 * TILE_MARGIN <= t <= MAX_TILE_SIZE:
        raise ValueError(f"tile_size must be a multiple of 32 in [{4 * TILE_MARGIN}, {MAX_TILE_SIZE}], got {t}")
    return t


def tile_size_for(hp, wp, tile_size=None):
    """The tile size a padded (hp, wp) batch is detected with, or None for the whole-page forward.  ``tile_size`` as
    ``check_tiles`` returns it: None tiles at DEFAULT_TILE_SIZE only a batch taller than that; a size tiles a batch
    larger than it in either dimension."""
    if tile_size is None:
        return DEFAULT_TILE_SIZE if hp > DEFAULT_TILE_SIZE else None
    return tile_size if hp > tile_size or wp > tile_size else None


LINE_DEFAULTS = {"angle_tolerance": 15.0, "height_ratio": 0.5, "offset_ratio": 0.5, "gap_ratio": 1.5}


def check_lines(**kw):
    """Validate the text-line parameters (DESIGN.md section 1, "Text lines") and return all four as floats, defaults
    filled in.  ``angle_tolerance`` in (0, 90] degrees, ``height_ratio`` in (0, 1], ``offset_ratio`` > 0,
    ``gap_ratio`` >= 0; unknown keys and values that are not finite real numbers raise ``ValueError``."""
    unknown = sorted(set(kw) - set(LINE_DEFAULTS))
    if unknown:
        raise ValueError(f"unknown line parameters {unknown}; expected some of {sorted(LINE_DEFAULTS)}")
    out = dict(LINE_DEFAULTS)
    for k, v in kw.items():
        if isinstance(v, bool) or not isinstance(v, numbers.Real) or not math.isfinite(float(v)):
            raise ValueError(f"{k} must be a finite number, got {v!r}")
        out[k] = float(v)
    if not 0 < out["angle_tolerance"] <= 90:
        raise ValueError(f"angle_tolerance must be in (0, 90] degrees, got {out['angle_tolerance']}")
    if not 0 < out["height_ratio"] <= 1:
        raise ValueError(f"height_ratio must be in (0, 1], got {out['height_ratio']}")
    if not out["offset_ratio"] > 0:
        raise ValueError(f"offset_ratio must be > 0, got {out['offset_ratio']}")
    if not out["gap_ratio"] >= 0:
        raise ValueError(f"gap_ratio must be >= 0, got {out['gap_ratio']}")
    return out


def lines_from_csr(line_count, word_order, line_start, line_boxes):
    """One image's rows of b2o_group_lines (host arrays) -> [(line_box (4,2) float32, word indices int32), ...]."""
    return [(line_boxes[l].copy(), word_order[line_start[l]:line_start[l + 1]].copy()) for l in range(int(line_count))]


BLOCK_DEFAULTS = {"row_gap": 1.5, "col_gap": 1.0}


def check_blocks(**kw):
    """Validate the text-block parameters (DESIGN.md section 1, "Text blocks") and return both as floats, defaults
    filled in.  ``row_gap`` and ``col_gap`` > 0, in units of the median line height; unknown keys and values that are
    not finite real numbers raise ``ValueError``."""
    unknown = sorted(set(kw) - set(BLOCK_DEFAULTS))
    if unknown:
        raise ValueError(f"unknown block parameters {unknown}; expected some of {sorted(BLOCK_DEFAULTS)}")
    out = dict(BLOCK_DEFAULTS)
    for k, v in kw.items():
        if isinstance(v, bool) or not isinstance(v, numbers.Real) or not math.isfinite(float(v)):
            raise ValueError(f"{k} must be a finite number, got {v!r}")
        if not float(v) > 0:
            raise ValueError(f"{k} must be > 0, got {v!r}")
        out[k] = float(v)
    return out


def blocks_from_csr(block_count, line_order, block_start, block_boxes):
    """One image's rows of b2o_group_blocks (host arrays) -> [(block_box (4,2) float32, line indices int32), ...]."""
    return [(block_boxes[b].copy(), line_order[block_start[b]:block_start[b + 1]].copy())
            for b in range(int(block_count))]


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
        self._line_ws = None
        self._block_ws = None

    # ------------------------------------------------------------------ device-resident API
    def _workspace(self, n, h, w):
        nbytes = self.ctx.craft_workspace_bytes(n, h, w)
        assert nbytes > 0, "image too small for CRAFT (needs H, W >= 32)"
        if self._ws is None or self._ws.numel() < nbytes:
            self._ws = None
            self._ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        return self._ws, nbytes

    def predict_device(self, images_t, tile_size=None, margin=TILE_MARGIN):
        """CRAFT forward.  images_t: (N,H,W,3) uint8 CUDA tensor -> (N,H/2,W/2,2) float32 scores.

        ``tile_size`` None: the whole page in one forward.  Otherwise (``check_tiles``) a batch larger than one tile
        runs over overlapping tiles (DESIGN.md section 1, "Tiles"): cut (``b2o_cut_tiles``), CRAFT on chunks of at
        most TILE_CHUNK_PIXELS pixels of tiles, each tile's core stitched into the page map (``b2o_stitch_tiles``),
        all queued on the current stream without a host wait; a batch that fits one tile takes the whole-page
        forward.  ``margin`` (a multiple of 16) is the context around each core; other values than TILE_MARGIN are
        for measuring the seams."""
        n, h, w, _ = images_t.shape
        stream = torch.cuda.current_stream(self.device).cuda_stream
        scores = torch.empty((n, h // 2, w // 2, 2), dtype=torch.float32, device=self.device)
        plan = None
        if tile_size is not None:
            tile_size = check_tiles(tile_size)
            plan = _lib.tile_plan(h, w, tile_size, margin)
            if plan is None:
                raise ValueError(f"no tile grid for a ({h}, {w}) batch with tile_size={tile_size}, margin={margin}")
        if plan is None or plan.n_h * plan.n_w == 1:
            ws, nbytes = self._workspace(n, h, w)
            self.ctx.craft_forward(images_t.data_ptr(), n, h, w, scores.data_ptr(), ws.data_ptr(), nbytes, stream)
            return scores
        images_t = images_t.contiguous()
        total = n * plan.n_h * plan.n_w
        per = min(total, max(1, TILE_CHUNK_PIXELS // (plan.t_h * plan.t_w)))
        tiles = torch.empty((per, plan.t_h, plan.t_w, 3), dtype=torch.uint8, device=self.device)
        tile_scores = torch.empty((per, plan.t_h // 2, plan.t_w // 2, 2), dtype=torch.float32, device=self.device)
        ws, nbytes = self._workspace(per, plan.t_h, plan.t_w)
        for first in range(0, total, per):
            k = min(per, total - first)
            self.ctx.cut_tiles(images_t.data_ptr(), n, plan, first, k, tiles.data_ptr(), stream)
            self.ctx.craft_forward(tiles.data_ptr(), k, plan.t_h, plan.t_w, tile_scores.data_ptr(), ws.data_ptr(), nbytes,
                                   stream)
            self.ctx.stitch_tiles(tile_scores.data_ptr(), n, plan, first, k, scores.data_ptr(), stream)
        return scores

    def boxes_enqueue(self, scores, detection_threshold=0.7, text_threshold=0.4, link_threshold=0.4,
                      size_threshold=10, with_scores=False, with_polygons=False, max_windows=1):
        """getBoxes on the device, asynchronously: launches the kernels and the copy of the per-image counts into
        pinned memory, records an event and returns at once (``boxes_finish`` waits for that event only, so work
        enqueued afterwards keeps the GPU busy while the host reads the counts).  ``with_scores``: the state also
        holds ``box_scores`` (N,M) float32 CUDA, each box's detection score (``b2o_get_boxes_scored``).
        ``with_polygons``: the state also holds every box's polygon (``b2o_get_boxes_poly``), ``polys`` (N,M,18,2)
        float32 and ``points`` (N,M) int32 CUDA, and their dense lists ``flat_polys`` / ``flat_points`` in the order
        of ``flat``; boxes and scores are those of the call without polygons.  ``max_windows`` > 1: the state also holds
        ``windows_pin`` (N,M) int32 pinned, every box's window count K (``b2o_window_counts``, see
        ``recognition.check_windows``), copied with the counts and valid once ``boxes_finish`` returns, for the first
        count boxes of each image."""
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
        box_scores = polys = points = None
        if with_scores:
            box_scores = torch.empty((n, m), dtype=torch.float32, device=self.device)
        if with_polygons:
            polys = torch.empty((n, m, _lib.POLY_POINTS, 2), dtype=torch.float32, device=self.device)
            points = torch.empty((n, m), dtype=torch.int32, device=self.device)
            self.ctx.get_boxes_poly(scores.data_ptr(), n, hs, ws_, *thr, boxes.data_ptr(), counts.data_ptr(),
                                    box_scores.data_ptr() if with_scores else None, polys.data_ptr(), points.data_ptr(),
                                    m, wsp.data_ptr(), nbytes, stream.cuda_stream)
        elif with_scores:
            self.ctx.get_boxes_scored(scores.data_ptr(), n, hs, ws_, *thr, boxes.data_ptr(), counts.data_ptr(),
                                      box_scores.data_ptr(), m, wsp.data_ptr(), nbytes, stream.cuda_stream)
        else:
            self.ctx.get_boxes(scores.data_ptr(), n, hs, ws_, *thr, boxes.data_ptr(), counts.data_ptr(), m,
                               wsp.data_ptr(), nbytes, stream.cuda_stream)
        counts_pin = torch.empty((n,), dtype=torch.int32, pin_memory=True)
        counts_pin.copy_(counts, non_blocking=True)
        windows_pin = None
        if max_windows > 1:                              # read back with the counts: no synchronisation of its own
            windows = torch.empty((n, m), dtype=torch.int32, device=self.device)
            self.ctx.window_counts(boxes.data_ptr(), counts.data_ptr(), n, m, int(max_windows), windows.data_ptr(),
                                   stream.cuda_stream)
            windows_pin = torch.empty((n, m), dtype=torch.int32, pin_memory=True)
            windows_pin.copy_(windows, non_blocking=True)
        event = torch.cuda.Event()
        event.record(stream)
        # recognize_from_boxes' bookkeeping (dense box list + image index, recognition.py:511-521) is queued
        # behind the counts copy: it needs no host knowledge, so it runs while the host still waits for the event
        flat = torch.empty((n * m, 4, 2), dtype=torch.float32, device=self.device)
        image_index = torch.empty((n * m,), dtype=torch.int32, device=self.device)
        self.ctx.compact_boxes(boxes.data_ptr(), counts.data_ptr(), n, m, flat.data_ptr(), image_index.data_ptr(),
                               stream.cuda_stream)
        flat_polys = flat_points = None
        if with_polygons:
            flat_polys = torch.empty((n * m, _lib.POLY_POINTS, 2), dtype=torch.float32, device=self.device)
            flat_points = torch.empty((n * m,), dtype=torch.int32, device=self.device)
            self.ctx.compact_polys(polys.data_ptr(), points.data_ptr(), counts.data_ptr(), n, m, flat_polys.data_ptr(),
                                   flat_points.data_ptr(), image_index.data_ptr(), stream.cuda_stream)
        return {"scores": scores, "boxes": boxes, "counts": counts, "counts_pin": counts_pin, "event": event, "m": m,
                "thr": thr, "flat": flat, "image_index": image_index, "box_scores": box_scores, "polys": polys,
                "points": points, "flat_polys": flat_polys, "flat_points": flat_points, "max_windows": max_windows,
                "windows_pin": windows_pin}

    def boxes_finish(self, state):
        """Wait for ``boxes_enqueue``.  Returns (boxes (N,M,4,2) float32 CUDA, counts ndarray (N,)); re-runs
        getBoxes with a larger box table in the (rare) case an image had more boxes than the table holds (the state's
        ``box_scores`` and polygons, when asked for, then come from that run too)."""
        state["event"].synchronize()                     # the one synchronisation of the detector half
        counts_host = state["counts_pin"].numpy().copy()
        while counts_host.size and int(counts_host.max()) > state["boxes"].shape[1]:
            self.max_boxes = int(2 ** np.ceil(np.log2(int(counts_host.max()))))
            d, t, l, s = state["thr"]
            again = self.boxes_enqueue(state["scores"], d, t, l, s, with_scores=state["box_scores"] is not None,
                                       with_polygons=state.get("polys") is not None,
                                       max_windows=state.get("max_windows", 1))
            again["event"].synchronize()
            state.update(again)
            counts_host = state["counts_pin"].numpy().copy()
        return state["boxes"], counts_host

    def boxes_device(self, scores, detection_threshold=0.7, text_threshold=0.4, link_threshold=0.4,
                     size_threshold=10):
        """getBoxes on the device.  Returns (boxes (N,M,4,2) float32 CUDA, counts ndarray (N,))."""
        return self.boxes_finish(self.boxes_enqueue(scores, detection_threshold, text_threshold, link_threshold,
                                                    size_threshold))

    def group_lines_device(self, boxes, counts_dev, **line_kwargs):
        """Text lines in reading order on the device (``b2o_group_lines``), queued on the current stream.
        ``boxes`` (N,M,4,2) float32 CUDA and ``counts_dev`` (N,) int32 CUDA as ``boxes_enqueue`` makes them (box[0] ->
        box[1] the reading direction); ``line_kwargs`` as ``check_lines`` takes them.  Returns (line_counts (N,),
        word_order (N,M), line_start (N,M+1) int32, line_boxes (N,M,4,2) float32), all CUDA: the words of line l of
        image i are ``word_order[i, line_start[i, l]:line_start[i, l + 1]]``, lines in page order.  Slots past an
        image's word / line count are not written."""
        p = check_lines(**line_kwargs)
        n, m = int(boxes.shape[0]), int(boxes.shape[1])
        assert boxes.is_cuda and boxes.dtype == torch.float32 and tuple(boxes.shape[2:]) == (4, 2)
        assert counts_dev.is_cuda and counts_dev.dtype == torch.int32 and tuple(counts_dev.shape) == (n,)
        boxes = boxes.contiguous()
        dev = boxes.device
        line_counts = torch.empty((n,), dtype=torch.int32, device=dev)
        word_order = torch.empty((n, m), dtype=torch.int32, device=dev)
        line_start = torch.empty((n, m + 1), dtype=torch.int32, device=dev)
        line_boxes = torch.empty((n, m, 4, 2), dtype=torch.float32, device=dev)
        if n == 0:
            return line_counts, word_order, line_start, line_boxes
        nbytes = self.ctx.lines_workspace_bytes(n, m)
        if self._line_ws is None or self._line_ws.numel() < nbytes:
            self._line_ws = None
            self._line_ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        self.ctx.group_lines(boxes.data_ptr(), counts_dev.data_ptr(), n, m, math.cos(math.radians(p["angle_tolerance"])),
                             p["height_ratio"], p["offset_ratio"], p["gap_ratio"], line_counts.data_ptr(),
                             word_order.data_ptr(), line_start.data_ptr(), line_boxes.data_ptr(),
                             self._line_ws.data_ptr(), nbytes, torch.cuda.current_stream(dev).cuda_stream)
        return line_counts, word_order, line_start, line_boxes

    def group_lines(self, box_groups, **line_kwargs):
        """Text lines of host box groups, as ``detect`` returns them (``np.array([])`` for an image without boxes) or
        from any other detector: per image a list of (line_box (4,2) float32, word_indices int32) in reading order,
        the indices into that image's boxes.  box[0] -> box[1] of every box must be its reading direction."""
        check_lines(**line_kwargs)
        groups = [np.asarray(g, np.float32).reshape(-1, 4, 2) for g in box_groups]
        if not groups:
            return []
        counts = np.array([len(g) for g in groups], np.int32)
        m = max(1, int(counts.max()))
        table = np.zeros((len(groups), m, 4, 2), np.float32)
        for i, g in enumerate(groups):
            table[i, :len(g)] = g
        out = self.group_lines_device(torch.from_numpy(table).to(self.device), torch.from_numpy(counts).to(self.device),
                                      **line_kwargs)
        lc, wo, ls, lb = (t.cpu().numpy() for t in out)
        return [lines_from_csr(lc[i], wo[i], ls[i], lb[i]) for i in range(len(groups))]

    def group_blocks_device(self, line_counts, line_start, line_boxes, **block_kwargs):
        """Text blocks in reading order on the device (``b2o_group_blocks``), queued on the current stream: recursive
        XY-cut over the lines ``group_lines_device`` returns (``line_counts`` (N,), ``line_start`` (N,M+1) int32,
        ``line_boxes`` (N,M,4,2) float32, all CUDA); ``block_kwargs`` as ``check_blocks`` takes them.  Returns
        (block_counts (N,), line_order (N,M), block_start (N,M+1) int32, block_boxes (N,M,4,2) float32), all CUDA: the
        lines of block b of image i, in page order, are ``line_order[i, block_start[i, b]:block_start[i, b + 1]]``,
        blocks in reading order.  Slots past an image's line / block count are not written."""
        p = check_blocks(**block_kwargs)
        n, m = int(line_boxes.shape[0]), int(line_boxes.shape[1])
        assert line_boxes.is_cuda and line_boxes.dtype == torch.float32 and tuple(line_boxes.shape[2:]) == (4, 2)
        assert line_counts.is_cuda and line_counts.dtype == torch.int32 and tuple(line_counts.shape) == (n,)
        assert line_start.is_cuda and line_start.dtype == torch.int32 and tuple(line_start.shape) == (n, m + 1)
        line_counts, line_start, line_boxes = line_counts.contiguous(), line_start.contiguous(), line_boxes.contiguous()
        dev = line_boxes.device
        block_counts = torch.empty((n,), dtype=torch.int32, device=dev)
        line_order = torch.empty((n, m), dtype=torch.int32, device=dev)
        block_start = torch.empty((n, m + 1), dtype=torch.int32, device=dev)
        block_boxes = torch.empty((n, m, 4, 2), dtype=torch.float32, device=dev)
        if n == 0:
            return block_counts, line_order, block_start, block_boxes
        nbytes = self.ctx.blocks_workspace_bytes(n, m)
        if self._block_ws is None or self._block_ws.numel() < nbytes:
            self._block_ws = None
            self._block_ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        self.ctx.group_blocks(line_counts.data_ptr(), line_start.data_ptr(), line_boxes.data_ptr(), n, m, p["row_gap"],
                              p["col_gap"], block_counts.data_ptr(), line_order.data_ptr(), block_start.data_ptr(),
                              block_boxes.data_ptr(), self._block_ws.data_ptr(), nbytes,
                              torch.cuda.current_stream(dev).cuda_stream)
        return block_counts, line_order, block_start, block_boxes

    def group_blocks(self, line_groups, **block_kwargs):
        """Text blocks of host lines, as ``group_lines`` returns them (per image a list of (line_box (4,2),
        word_indices)) or from any other source in page order: per image a list of (block_box (4,2) float32,
        line_indices int32) in reading order, the indices into that image's lines.  box[0] -> box[1] of every line box
        must be its reading direction."""
        check_blocks(**block_kwargs)
        if not line_groups:
            return []
        n = len(line_groups)
        counts = np.array([len(g) for g in line_groups], np.int32)
        m = max(1, int(counts.max()))
        boxes = np.zeros((n, m, 4, 2), np.float32)
        starts = np.zeros((n, m + 1), np.int32)
        for i, g in enumerate(line_groups):
            if len(g):
                boxes[i, :len(g)] = np.stack([np.asarray(b, np.float32).reshape(4, 2) for b, _ in g])
                starts[i, 1:len(g) + 1] = np.cumsum([len(w) for _, w in g])
        dev = self.device
        out = self.group_blocks_device(torch.from_numpy(counts).to(dev), torch.from_numpy(starts).to(dev),
                                       torch.from_numpy(boxes).to(dev), **block_kwargs)
        bc, lo, bs, bb = (t.cpu().numpy() for t in out)
        return [blocks_from_csr(bc[i], lo[i], bs[i], bb[i]) for i in range(n)]

    def detect_device(self, images_t, tile_size=None, **thresholds):
        tile_size = check_tiles(tile_size)
        return self.boxes_device(self.predict_device(images_t, tile_size_for(images_t.shape[1], images_t.shape[2],
                                                                             tile_size)), **thresholds)

    # ------------------------------------------------------------------ reference API
    def detect(self, images: typing.List[typing.Union[np.ndarray, str]], detection_threshold=0.7,
               text_threshold=0.4, link_threshold=0.4, size_threshold=10, return_scores=False, return_polygons=False,
               tile_size=None, **kwargs):
        """Same contract as reference detection.py:745-785: a list with one array of boxes
        ``(n_i, 4, 2)`` float32 per image (``np.array([])`` when there is none).  ``kwargs`` are the
        keras ``predict`` arguments of the reference (batch_size, verbose, ...) and are ignored.

        ``return_scores=True``: one ``(boxes, scores)`` pair per image instead, ``scores`` (n_i,) float32 the
        detection score of each box -- the largest text score over its connected component, the value compared
        with ``detection_threshold`` (so every score is >= it).

        ``return_polygons=True``: every image also gives the polygon of each box, last in its tuple -- ``(boxes,
        polygons)`` or ``(boxes, scores, polygons)`` -- a list of (p,2) float32 arrays in detector-input pixels: the box
        itself (p = 4) for a straight word, otherwise 2 (s + 1) points along a curved word's centre line, the top edge
        left to right then the bottom edge right to left, clockwise from the top-left (``b2o_get_boxes_poly``).  Boxes
        and scores are those of the default call.

        ``tile_size`` (``check_tiles``): the batch runs CRAFT over overlapping tiles of that size when it is larger than
        one in either dimension; None (the default) tiles at 2048 a batch taller than 2048 only (``tile_size_for``).
        Everything after the score map is unchanged."""
        tile_size = check_tiles(tile_size)
        images_t = _as_device_images(images, self.device)
        scores = self.predict_device(images_t, tile_size_for(images_t.shape[1], images_t.shape[2], tile_size))
        state = self.boxes_enqueue(scores, detection_threshold, text_threshold, link_threshold,
                                   size_threshold, with_scores=return_scores, with_polygons=return_polygons)
        boxes, counts = self.boxes_finish(state)
        boxes_host = boxes.cpu().numpy()
        groups = [boxes_host[i, :c].copy() if c else np.array([]) for i, c in enumerate(counts)]
        if not (return_scores or return_polygons):
            return groups
        out = [(g,) for g in groups]
        if return_scores:
            scores_host = state["box_scores"].cpu().numpy()
            out = [o + (scores_host[i, :c].copy(),) for i, (o, c) in enumerate(zip(out, counts))]
        if return_polygons:
            polys, points = state["polys"].cpu().numpy(), state["points"].cpu().numpy()
            out = [o + ([polys[i, k, :points[i, k]].copy() for k in range(c)],) for i, (o, c) in enumerate(zip(out, counts))]
        return out
