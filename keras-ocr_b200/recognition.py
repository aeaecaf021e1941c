"""Recognizer: drop-in for ``keras_ocr.recognition.Recognizer`` (reference recognition.py:353-537)."""
import string
import typing

import numpy as np
import torch

from . import _lib, tools, weights as weights_mod

DEFAULT_ALPHABET = string.digits + string.ascii_lowercase      # reference recognition.py:25
TARGET_HEIGHT, TARGET_WIDTH, STEPS = 31, 200, 48                # DEFAULT_BUILD_PARAMS, recognition.py:13-23
DEFAULT_BUILD_PARAMS = {"height": 31, "width": 200, "color": False, "filters": (64, 128, 256, 256, 512, 512, 512),
                        "rnn_units": (128, 128), "dropout": 0.25, "rnn_steps_to_discard": 2, "pool_size": 2}


def labels_to_text(rows, alphabet=DEFAULT_ALPHABET):
    """reference recognition.py:527-534: drop blank / -1, map indices to characters.

    Vectorised: the kept labels of all rows are gathered into ONE byte string with a newline after every row, decoded
    once and split (no per-character and no per-row Python work besides the split); alphabets that are not ASCII or
    contain a newline, and tables with out-of-range indices, take the reference's element-wise filter."""
    blank = len(alphabet)
    rows = np.asarray(rows)
    if rows.ndim == 2 and rows.size and alphabet.isascii() and "\n" not in alphabet:
        keep = (rows != blank) & (rows != -1)
        flat = rows[keep]
        if flat.size == 0 or (int(flat.min()) >= 0 and int(flat.max()) < blank):
            out = np.full(flat.size + rows.shape[0], 10, dtype=np.uint8)          # 10 = "\n"
            ends = np.cumsum(keep.sum(1) + 1) - 1
            chars = np.ones(out.size, dtype=bool)
            chars[ends] = False
            out[chars] = np.frombuffer(alphabet.encode("ascii"), dtype=np.uint8)[flat]
            return out.tobytes().decode("ascii").split("\n")[:-1]
    return ["".join(alphabet[idx] for idx in row if idx not in (blank, -1)) for row in rows]


def confidences(logp):
    """Word confidences exp(S) in (0, 1] (float32) from the greedy-path log-probabilities
    S = sum_t log(max_c p[t,c] + 1e-7) that ``b2o_crnn_forward_scored`` writes.  The 1e-7 floor lets S of a
    certain word reach 48 * log(1 + 1e-7) ~ 5e-6 > 0, hence the clip at 1."""
    return np.minimum(np.exp(np.asarray(logp, dtype=np.float32)), np.float32(1.0))


def check_beam(beam_width=None, top_paths=1):
    """Validates a decoder choice before anything is launched (``ValueError`` otherwise): ``beam_width=None`` is greedy
    CTC (the default, and then ``top_paths`` must be 1); an int 1 <= ``beam_width`` <= 128 is CTC prefix beam search
    (``b2o_crnn_forward_beam``) returning the ``top_paths`` best readings, 1 <= ``top_paths`` <= ``beam_width``."""
    def is_int(v):
        return isinstance(v, (int, np.integer)) and not isinstance(v, (bool, np.bool_))
    if not is_int(top_paths) or top_paths < 1:
        raise ValueError(f"top_paths must be an int >= 1, got {top_paths!r}")
    if beam_width is None:
        if top_paths != 1:
            raise ValueError("top_paths > 1 needs beam search: pass beam_width")
        return
    if not is_int(beam_width) or not 1 <= beam_width <= _lib.MAX_BEAM_WIDTH:
        raise ValueError(f"beam_width must be None or an int in [1, {_lib.MAX_BEAM_WIDTH}], got {beam_width!r}")
    if top_paths > beam_width:
        raise ValueError(f"top_paths ({top_paths}) must not exceed beam_width ({beam_width})")


def decode_paths(labels, alphabet=DEFAULT_ALPHABET, logp=None):
    """Host labels -> texts, and logp -> confidences (None without logp).  (B,48) labels / (B,) logp give B strings and
    a float32 array, as the greedy decoder returns them; (B,P,48) / (B,P) -- ``top_paths = P > 1`` -- give B lists of P
    strings and B lists of P confidences, best first."""
    labels = np.asarray(labels)
    if labels.ndim == 2:
        return labels_to_text(labels, alphabet), (None if logp is None else confidences(logp))
    b, p = labels.shape[:2]
    flat = labels_to_text(labels.reshape(b * p, STEPS), alphabet)
    texts = [flat[i * p:(i + 1) * p] for i in range(b)]
    return texts, (None if logp is None else [list(row) for row in confidences(logp)])


class Recognizer:
    """A text recognizer using the CRNN architecture, running as sm_90a CUDA kernels.

    Args:
        alphabet: the characters the model recognises (default ``0-9a-z``; up to 1023 characters).  The
            checkpoint's ``fc_12`` must have ``len(alphabet) + 1`` classes; if it does not, the reference's
            "backbone weights only" behaviour applies (recognition.py:399-411): the top layer is
            re-initialised (Glorot uniform, zero bias) and has to be trained before it is useful.
        weights: ``None`` builds an untrained model for ``alphabet`` (as the reference does); ``"kurapan"`` looks for ``crnn_kurapan.npz`` (exported) or the reference's ``crnn_kurapan.h5``
            (read with h5py where installed) in the cache dir; otherwise a ``.npz`` / ``.h5`` path or a dict
            keyed like ``weights.py``.
        build_params: ``None`` / the defaults (reference recognition.py:13-23), optionally with ``"stn": False`` (the
            recognizer without the spatial transformer, recognition.py:243) and / or ``"color": True`` (RGB crops into a
            3-channel ``conv_1``, recognition.py:214); other architectures raise NotImplementedError.
    """

    def __init__(self, alphabet=None, weights="kurapan", build_params=None, device=None):
        assert alphabet or weights, "At least one of alphabet or weights must be provided."
        # build_params (recognition.py:13-23, 365-368): the CUDA recognizer implements the default architecture; of the
        # build options only ``stn`` (with / without the spatial transformer, recognition.py:243) and ``color`` (RGB instead
        # of gray crops, recognition.py:214) may differ
        params = dict(DEFAULT_BUILD_PARAMS, **(build_params or {}))
        self.stn = bool(params.pop("stn", True))
        self.color = bool(params["color"])                        # RGB crops, no gray conversion (recognition.py:214, 508-510)
        params["color"] = False
        if params != DEFAULT_BUILD_PARAMS:
            changed = sorted(k for k in params if params[k] != DEFAULT_BUILD_PARAMS.get(k))
            raise NotImplementedError(f"build_params other than the defaults are not supported by the CUDA recognizer: {changed}")
        if not torch.cuda.is_available():
            raise _lib.B2OError("keras-ocr_b200 needs a CUDA device (sm_90a); there is no CPU fallback")
        self.alphabet = alphabet or DEFAULT_ALPHABET              # recognition.py:369-375
        if len(self.alphabet) + 1 > _lib.MAX_CLASSES:
            raise ValueError(f"alphabet too long: at most {_lib.MAX_CLASSES - 1} characters")
        self.blank_label_idx = len(self.alphabet)
        self.device_index = torch.cuda.current_device() if device is None else int(device)
        self.device = torch.device("cuda", self.device_index)
        if isinstance(weights, dict):
            tensors = weights
        elif weights is None:
            # reference recognition.py:382-383: no weights -> the freshly built (untrained) model for this alphabet
            tensors = weights_mod.synthetic_crnn_weights(seed=0, alphabet=self.alphabet, stn=self.stn, color=self.color)
        elif isinstance(weights, str) and weights.endswith(".npz"):
            tensors = weights_mod.load_npz(weights)
        elif isinstance(weights, str) and weights.endswith(".h5"):
            tensors = weights_mod.load_keras_h5(weights)
        elif weights == "kurapan":                                # recognition.py:27-44: cache file, sha256-verified
            import os
            cache = tools.get_default_cache_dir()
            if os.path.isfile(os.path.join(cache, "crnn_kurapan.npz")):
                tensors = weights_mod.load_npz(os.path.join(cache, "crnn_kurapan.npz"))
            else:
                tensors = weights_mod.load_keras_h5(tools.find_cached(
                    "crnn_kurapan.h5", sha256="a7d8086ac8f5c3d6a0a828f7d6fbabcaf815415dd125c32533013f85603be46d"))
        else:
            raise NotImplementedError(f"Cannot load weights from {weights}")
        has_stn = "stn.conv_a.kernel" in tensors
        if has_stn and not self.stn:                              # stn=False with a checkpoint that has one: drop it
            tensors = {k: v for k, v in tensors.items() if not k.startswith("stn.")}
        elif self.stn and not has_stn:
            raise ValueError("the checkpoint has no spatial-transformer tensors: pass build_params={'stn': False}")
        in_ch = int(np.shape(tensors["conv_1.kernel"])[2]) if "conv_1.kernel" in tensors else 1
        if in_ch != (3 if self.color else 1):
            raise ValueError(f"conv_1.kernel takes {in_ch} input channel(s): pass build_params={{'color': {in_ch == 3}}}")
        n_classes = len(self.alphabet) + 1
        top = tensors.get("fc_12.kernel")
        if top is None or tuple(np.shape(top)) != (256, n_classes):
            print("Provided alphabet does not match pretrained alphabet. Using backbone weights only.")
            tensors = dict(tensors)
            limit = float(np.sqrt(6.0 / (256 + n_classes)))           # keras Dense default: glorot_uniform, zeros
            tensors["fc_12.kernel"] = np.random.default_rng(0).uniform(-limit, limit, (256, n_classes)).astype(np.float32)
            tensors["fc_12.bias"] = np.zeros(n_classes, np.float32)
        self.ctx = _lib.Context(self.device_index)
        self.ctx.load_crnn(tensors)
        self._keep_workspace = False     # tests set keep_workspace to read intermediate taps
        self._last_ws = None
        self._ws = None                  # reusable CRNN workspace (grown on demand)

    @property
    def keep_workspace(self):
        return self._keep_workspace

    @keep_workspace.setter
    def keep_workspace(self, on):
        """Debug: keep the last forward pass's workspace for ``tap`` and make the CRNN write its fp32 logits
        (off on the product path: the fused Dense + CTC kernel then stores labels only)."""
        self._keep_workspace = bool(on)
        self.ctx.set_debug_taps(self._keep_workspace)

    # ------------------------------------------------------------------ device-resident API
    def gray_device(self, images_t):
        n, h, w, _ = images_t.shape
        gray = torch.empty((n, h, w), dtype=torch.uint8, device=self.device)
        self.ctx.rgb_to_gray(images_t.data_ptr(), n, h, w, gray.data_ptr(), torch.cuda.current_stream(self.device).cuda_stream)
        return gray

    def warp_device(self, gray, boxes_flat, image_index, want_crops=False):
        """tools.warpBox for every box.  ``gray``: (N,H,W) u8 -- or the RGB batch (N,H,W,3) for a color recognizer.
        Returns (crnn_in (B,200,31[,3]) fp16, crops (B,31,200[,3]) u8 or None)."""
        n, h, w = gray.shape[:3]
        color = gray.dim() == 4
        assert color == self.color, "a color recognizer warps the RGB batch, a gray one the gray batch"
        tail = (3,) if color else ()
        b = boxes_flat.shape[0]
        crnn_in = torch.empty((b, TARGET_WIDTH, TARGET_HEIGHT) + tail, dtype=torch.float16, device=self.device)
        crops = torch.empty((b, TARGET_HEIGHT, TARGET_WIDTH) + tail, dtype=torch.uint8, device=self.device) if want_crops else None
        self.ctx.warp_boxes(gray.data_ptr(), n, h, w, boxes_flat.data_ptr(), image_index.data_ptr(), b,
                            crops.data_ptr() if want_crops else None, crnn_in.data_ptr(),
                            torch.cuda.current_stream(self.device).cuda_stream, color=color)
        return crnn_in, crops

    def predict_device(self, crnn_in, with_scores=False, beam_width=None, top_paths=1):
        """CRNN + greedy CTC.  crnn_in: (B,200,31) fp16 -> labels (B,48) int32 (-1 padded).  ``with_scores``: returns
        (labels, logp) with logp (B,) float32 the greedy path's log-probability (``b2o_crnn_forward_scored``).
        ``beam_width``: CTC prefix beam search instead (``b2o_crnn_forward_beam``, see ``check_beam``), logp = the beam
        scores; ``top_paths > 1`` gives labels (B,P,48) and logp (B,P), best first."""
        check_beam(beam_width, top_paths)
        b = crnn_in.shape[0]
        labels = torch.empty((b, STEPS), dtype=torch.int32, device=self.device)
        nbytes = self.ctx.crnn_workspace_bytes(b)
        if self._ws is None or self._ws.numel() < nbytes:
            self._ws = None
            self._ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        ws = self._ws
        stream = torch.cuda.current_stream(self.device).cuda_stream
        logp = None
        if beam_width is not None:
            lead = (b,) if top_paths == 1 else (b, top_paths)
            labels = torch.empty(lead + (STEPS,), dtype=torch.int32, device=self.device)
            logp = torch.empty(lead, dtype=torch.float32, device=self.device) if with_scores else None
            self.ctx.crnn_forward_beam(crnn_in.data_ptr(), b, int(beam_width), int(top_paths), labels.data_ptr(),
                                       logp.data_ptr() if with_scores else None, ws.data_ptr(), nbytes, stream)
        elif with_scores:
            logp = torch.empty((b,), dtype=torch.float32, device=self.device)
            self.ctx.crnn_forward_scored(crnn_in.data_ptr(), b, labels.data_ptr(), logp.data_ptr(), ws.data_ptr(), nbytes,
                                         stream)
        else:
            self.ctx.crnn_forward(crnn_in.data_ptr(), b, labels.data_ptr(), ws.data_ptr(), nbytes, stream)
        self._last_ws = (ws, b) if self.keep_workspace else None
        return (labels, logp) if with_scores else labels

    def tap(self, name, shape, dtype):
        """Debug: copy an intermediate of the last predict_device call (needs keep_workspace=True)."""
        ws, b = self._last_ws
        out = torch.empty(shape, dtype=dtype, device=self.device)
        self.ctx.crnn_tap(name, ws.data_ptr(), b, out.data_ptr(), out.numel() * out.element_size(),
                          torch.cuda.current_stream(self.device).cuda_stream)
        return out

    def recognize_crops(self, crops, return_scores=False, beam_width=None, top_paths=1):
        """crops: (B,31,200) uint8 -- (B,31,200,3) for a color recognizer -- i.e. what tools.warpBox returns -> list[str].
        ``return_scores=True``: a list of (text, confidence) instead, see ``confidences``.  ``beam_width``: beam search
        decoding (``check_beam``); with ``top_paths = P > 1`` each text is a list of P strings and each confidence a
        list of P floats, best first (``decode_paths``)."""
        check_beam(beam_width, top_paths)
        t = crops if isinstance(crops, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(crops))
        t = t.to(self.device).contiguous()
        b = t.shape[0]
        if b == 0:
            return []
        assert t.shape[1:] == (TARGET_HEIGHT, TARGET_WIDTH) + ((3,) if self.color else ()), "crops must be (B,31,200[,3])"
        crnn_in = torch.empty((b, TARGET_WIDTH, TARGET_HEIGHT) + ((3,) if self.color else ()), dtype=torch.float16, device=self.device)
        self.ctx.crops_to_input(t.data_ptr(), b, crnn_in.data_ptr(), torch.cuda.current_stream(self.device).cuda_stream,
                                color=self.color)
        beam = {"beam_width": beam_width, "top_paths": top_paths}
        if not return_scores:
            return decode_paths(self.predict_device(crnn_in, **beam).cpu().numpy(), self.alphabet)[0]
        labels, logp = self.predict_device(crnn_in, with_scores=True, **beam)
        return list(zip(*decode_paths(labels.cpu().numpy(), self.alphabet, logp.cpu().numpy())))

    def recognize(self, image, beam_width=None, top_paths=1):
        """Recognize text from a single pre-cropped image (reference recognition.py:467-489): fit to
        200x31 with zero fill (host, as upstream), gray conversion, then the CUDA CRNN.  ``beam_width`` / ``top_paths``:
        as ``recognize_crops``."""
        import cv2

        check_beam(beam_width, top_paths)
        image = tools.read_and_fit(filepath_or_array=image, width=TARGET_WIDTH, height=TARGET_HEIGHT, cval=0)
        if not self.color and image.ndim == 3 and image.shape[-1] == 3:      # recognition.py:481-483
            image = cv2.cvtColor(image, code=cv2.COLOR_RGB2GRAY)
        return self.recognize_crops(np.ascontiguousarray(image.reshape((1, TARGET_HEIGHT, TARGET_WIDTH) + ((3,) if self.color else ()))),
                                    beam_width=beam_width, top_paths=top_paths)[0]

    def recognize_from_boxes_device(self, images_t, boxes, counts, gray=None, flat=None, image_index=None,
                                    with_scores=False, beam_width=None, top_paths=1):
        """images_t (N,H,W,3) u8 CUDA; boxes (N,M,4,2) f32 CUDA; counts host ndarray -> labels (B,48) i32 CUDA
        (``with_scores``: (labels, logp (B,) f32 CUDA); ``beam_width`` / ``top_paths``: see ``predict_device``).

        Optional device-side by-products of the earlier stages, so that nothing but the kernel launches is
        left to do once the host knows the counts: ``gray`` (N,H,W) u8 from ``b2o_resize_pad_batch``;
        ``flat`` (>=B,4,2) / ``image_index`` (>=B,) from ``b2o_compact_boxes``."""
        check_beam(beam_width, top_paths)
        counts = np.asarray(counts)
        m = boxes.shape[1]
        total = int(np.minimum(counts, m).sum())
        if total == 0:
            return (None, None) if with_scores else None
        if self.color:
            gray = images_t                                       # color recognizer: crops come straight from the RGB batch
        elif gray is None:
            gray = self.gray_device(images_t)
        if flat is None or image_index is None:
            n = len(counts)
            flat = torch.empty((n * m, 4, 2), dtype=torch.float32, device=self.device)
            image_index = torch.empty((n * m,), dtype=torch.int32, device=self.device)
            counts_dev = torch.from_numpy(counts.astype(np.int32)).to(self.device)
            self.ctx.compact_boxes(boxes.data_ptr(), counts_dev.data_ptr(), n, m, flat.data_ptr(),
                                   image_index.data_ptr(), torch.cuda.current_stream(self.device).cuda_stream)
        crnn_in, _ = self.warp_device(gray, flat[:total], image_index[:total])
        return self.predict_device(crnn_in, with_scores=with_scores, beam_width=beam_width, top_paths=top_paths)

    # ------------------------------------------------------------------ reference API
    def recognize_from_boxes(self, images, box_groups, return_scores=False, beam_width=None, top_paths=1,
                             **kwargs) -> typing.List[typing.List[str]]:
        """Same contract as reference recognition.py:491-537.  ``return_scores=True``: every word is a
        (text, confidence) pair instead, see ``confidences``.  ``beam_width`` / ``top_paths``: as ``recognize_crops``."""
        check_beam(beam_width, top_paths)
        assert len(box_groups) == len(images), "You must provide the same number of box groups as images."
        from .detection import _as_device_images

        images_t = _as_device_images(images, self.device)
        counts = np.array([len(b) for b in box_groups], dtype=np.int64)
        if counts.sum() == 0:
            return [[]] * len(images)
        flat = np.concatenate([np.asarray(b, dtype=np.float32).reshape(-1, 4, 2) for b in box_groups if len(b)])
        # caller-supplied quads: tools.warpBox first replaces each by its minimum rotated rectangle and divides by its
        # truncated width / height (tools.py:88-95; ZeroDivisionError for a degenerate box).  Rectangles -- everything
        # a Detector returns -- pass through bit for bit.
        flat = tools.rectify_boxes(flat)
        flat_t = torch.from_numpy(np.ascontiguousarray(flat)).to(self.device)
        idx = torch.from_numpy(np.repeat(np.arange(len(counts), dtype=np.int32), counts)).to(self.device)
        crnn_in, _ = self.warp_device(images_t if self.color else self.gray_device(images_t), flat_t, idx)
        beam = {"beam_width": beam_width, "top_paths": top_paths}
        if return_scores:
            labels, logp = self.predict_device(crnn_in, with_scores=True, **beam)
            predictions = list(zip(*decode_paths(labels.cpu().numpy(), self.alphabet, logp.cpu().numpy())))
        else:
            predictions = decode_paths(self.predict_device(crnn_in, **beam).cpu().numpy(), self.alphabet)[0]
        ends = np.cumsum(counts)
        return [predictions[int(e - c):int(e)] for c, e in zip(counts, ends)]
