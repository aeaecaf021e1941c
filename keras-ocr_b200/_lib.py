"""ctypes binding of ``libb2ocr.so`` (C-ABI in include/b2ocr.h).

There is deliberately no fallback: if the shared library is missing or the device is not an
H100-class (sm_90) GPU, importing/creating fails loudly.  PyTorch is used by the callers only to own
device memory and streams; only raw pointers cross this boundary.
"""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B2O_LIB") or os.path.join(_HERE, "libb2ocr.so")      # B2O_LIB: development builds only

CONV_AUTO, CONV_SIMT, CONV_TC_GENERIC = 0, 1, 2
MAX_CLASSES = 1024            # B2O_MAX_CLASSES in include/b2ocr.h
MAX_BEAM_WIDTH = 128          # B2O_MAX_BEAM_WIDTH in include/b2ocr.h
MAX_LEXICON_WORDS = 1 << 20   # B2O_MAX_LEXICON_WORDS
MAX_LEXICON_LABELS = 1 << 24  # B2O_MAX_LEXICON_LABELS
MAX_LEXICON_TOP_PATHS = 128   # B2O_MAX_LEXICON_TOP_PATHS
MAX_LM_ORDER = 8              # B2O_MAX_LM_ORDER
MAX_LM_HISTORIES = 1 << 20    # B2O_MAX_LM_HISTORIES
MAX_LM_CLASSES = 127          # B2O_MAX_LM_CLASSES
MAX_HOTWORD_NODES = (1 << 24) + 1   # B2O_MAX_HOTWORD_NODES
MAX_PATTERN_STATES = 4096     # B2O_MAX_PATTERN_STATES
MAX_PATTERN_CLASSES = 127     # B2O_MAX_PATTERN_CLASSES
ROTATION_VOTE_WORD, ROTATION_VOTE_PAGE = 0, 1   # B2O_ROTATION_VOTE_WORD / _PAGE
MAX_ALIGN_PATHS = 128         # B2O_MAX_ALIGN_PATHS
MAX_CHAR_ALTERNATIVES = 8     # B2O_MAX_CHAR_ALTERNATIVES
CRAFT_LAST_STEP = 30          # B2O_CRAFT_LAST_STEP
MAX_POLY_SEGMENTS = 8         # B2O_MAX_POLY_SEGMENTS
POLY_POINTS = 2 * (MAX_POLY_SEGMENTS + 1)   # points per entry of a dense polygon table
MAX_WINDOWS = 16              # B2O_MAX_WINDOWS
WINDOW_STRIDE = 136           # B2O_WINDOW_STRIDE
WINDOW_SHRINK = 8             # B2O_WINDOW_SHRINK
CRAFT_MAX_PIXELS = 1 << 25    # B2O_CRAFT_MAX_PIXELS


class B2OError(RuntimeError):
    pass


class _Tensor(ctypes.Structure):
    _fields_ = [("name", ctypes.c_char_p), ("data", ctypes.POINTER(ctypes.c_float)),
                ("ndim", ctypes.c_int32), ("shape", ctypes.c_int64 * 4)]


_c = ctypes
_vp, _i, _f, _sz = _c.c_void_p, _c.c_int, _c.c_float, _c.c_size_t
_fp = _c.POINTER(_c.c_float)


class _ConvTestDesc(ctypes.Structure):
    """b2o_conv_test_desc (include/b2ocr.h), field for field."""
    _fields_ = [("x_dev", _vp), ("n", _i), ("h", _i), ("w", _i), ("cin", _i), ("x_ld", _i),
                ("wgt_host", _fp), ("cout", _i), ("ksize", _i), ("dilation", _i),
                ("s1_host", _fp), ("t1_host", _fp), ("relu", _i), ("s2_host", _fp), ("t2_host", _fp),
                ("out_dev", _vp), ("out_ld", _i), ("out_f32", _i), ("write_full", _i),
                ("pool_dev", _vp), ("pool_ld", _i), ("up_dev", _vp), ("up_ld", _i),
                ("w6_host", _fp), ("b6_host", _fp), ("w8_host", _fp), ("b8_host", _fp), ("scores_dev", _vp),
                ("engine", _i)]


class _ConvPlanDesc(ctypes.Structure):
    """b2o_conv_plan_desc (include/b2ocr.h), field for field."""
    _fields_ = [(name, _i) for name in ("n", "h", "w", "cin", "cout", "ksize", "dilation", "out_f32", "pool", "tail",
                                        "up_add", "engine", "swap", "sm_count")]


class _ConvPlan(ctypes.Structure):
    """b2o_conv_plan (include/b2ocr.h), field for field."""
    _fields_ = [(name, _c.c_int32) for name in ("block_n", "kch", "mode", "pair", "upadd", "body", "tile_w", "tile_h",
                                                "tile_n", "tiles", "stages", "stage_bytes", "stage_tx", "resident_bytes",
                                                "smem_bytes", "grid", "coop_n")]

class CharLMDesc(ctypes.Structure):
    """b2o_char_lm (include/b2ocr.h), field for field."""
    _fields_ = [("order", _i), ("n_histories", _i), ("keys_dev", _vp), ("rows_dev", _vp), ("alpha", _f), ("beta", _f)]


_lmp = _c.POINTER(CharLMDesc)


class HotwordsDesc(ctypes.Structure):
    """b2o_hotwords (include/b2ocr.h), field for field."""
    _fields_ = [("n_nodes", _i), ("n_edges", _i), ("keys_dev", _vp), ("child_dev", _vp), ("final_dev", _vp),
                ("weight", _f)]


_hwp = _c.POINTER(HotwordsDesc)


class PatternDesc(ctypes.Structure):
    """b2o_pattern (include/b2ocr.h), field for field."""
    _fields_ = [("n_states", _i), ("start", _i), ("trans_dev", _vp), ("dist_dev", _vp)]


_patp = _c.POINTER(PatternDesc)


class TilePlan(ctypes.Structure):
    """b2o_tiles (include/b2ocr.h), field for field."""
    _fields_ = [(name, _i) for name in ("hp", "wp", "tile_size", "margin", "t_h", "t_w", "s_h", "s_w", "n_h", "n_w")]


_tilep = _c.POINTER(TilePlan)

# name -> (restype, argtypes); mirrors include/b2ocr.h one to one
SIGNATURES = {
    "b2o_version": (_i, []),
    "b2o_create": (_i, [_i, _c.POINTER(_vp)]),
    "b2o_destroy": (None, [_vp]),
    "b2o_last_error": (_c.c_char_p, [_vp]),
    "b2o_set_conv_engine": (_i, [_vp, _i]),
    "b2o_launch_count": (_c.c_int64, [_vp]),
    "b2o_tc_tile256_launches": (_c.c_int64, [_vp]),
    "b2o_tc_coop_n_launches": (_c.c_int64, [_vp]),
    "b2o_profile_enable": (_i, [_vp, _i]),
    "b2o_profile_read": (_i, [_vp, _c.POINTER(_c.c_double), _c.POINTER(_c.c_double), _c.POINTER(_c.c_int64)]),
    "b2o_load_craft": (_i, [_vp, _c.POINTER(_Tensor), _i]),
    "b2o_load_crnn": (_i, [_vp, _c.POINTER(_Tensor), _i]),
    "b2o_resize_pad": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _i, _i, _i, _vp]),
    "b2o_resize_pad_batch": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp, _i, _i, _vp, _vp]),
    "b2o_jpeg_info": (_i, [_vp, _vp, _sz, _c.POINTER(_i), _c.POINTER(_i), _c.POINTER(_i)]),
    "b2o_decode_jpeg": (_i, [_vp, _vp, _sz, _vp, _i, _i, _vp]),
    "b2o_rgb_to_gray": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp]),
    "b2o_craft_workspace_bytes": (_sz, [_i, _i, _i]),
    "b2o_craft_forward": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _sz, _vp]),
    "b2o_craft_forward_until": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _sz, _i, _vp]),
    "b2o_craft_tap": (_i, [_vp, _c.c_char_p, _vp, _i, _i, _i, _vp, _sz, _vp]),
    "b2o_tile_plan": (_i, [_i, _i, _i, _i, _tilep]),
    "b2o_cut_tiles": (_i, [_vp, _vp, _i, _tilep, _i, _i, _vp, _vp]),
    "b2o_stitch_tiles": (_i, [_vp, _vp, _i, _tilep, _i, _i, _vp, _vp]),
    "b2o_boxes_workspace_bytes": (_sz, [_i, _i, _i, _i]),
    "b2o_get_boxes": (_i, [_vp, _vp, _i, _i, _i, _f, _f, _f, _i, _vp, _vp, _i, _vp, _sz, _vp]),
    "b2o_get_boxes_scored": (_i, [_vp, _vp, _i, _i, _i, _f, _f, _f, _i, _vp, _vp, _vp, _i, _vp, _sz, _vp]),
    "b2o_compact_boxes": (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    "b2o_get_boxes_poly": (_i, [_vp, _vp, _i, _i, _i, _f, _f, _f, _i, _vp, _vp, _vp, _vp, _vp, _i, _vp, _sz, _vp]),
    "b2o_compact_polys": (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp]),
    "b2o_warp_polys": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _i, _vp, _vp, _vp]),
    "b2o_lines_workspace_bytes": (_sz, [_i, _i]),
    "b2o_group_lines": (_i, [_vp, _vp, _vp, _i, _i, _c.c_double, _c.c_double, _c.c_double, _c.c_double, _vp, _vp, _vp,
                             _vp, _vp, _sz, _vp]),
    "b2o_blocks_workspace_bytes": (_sz, [_i, _i]),
    "b2o_group_blocks": (_i, [_vp, _vp, _vp, _vp, _i, _i, _c.c_double, _c.c_double, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "b2o_window_counts": (_i, [_vp, _vp, _vp, _i, _i, _i, _vp, _vp]),
    "b2o_warp_windows": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp]),
    "b2o_stitch_windows": (_i, [_vp, _vp, _i, _vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    "b2o_window_plan_test": (_i, [_vp, _vp, _i, _i, _vp, _vp]),
    "b2o_record_floats": (_sz, [_i]),
    "b2o_record_floats_scored": (_sz, [_i]),
    "b2o_pack_records": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    "b2o_pack_records_scored": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp, _vp]),
    "b2o_warp_boxes": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _i, _vp, _vp, _vp]),
    "b2o_warp_boxes_color": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _i, _vp, _vp, _vp]),
    "b2o_warp_boxes_turned": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _i, _i, _vp, _vp, _vp]),
    "b2o_select_rotation": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _c.POINTER(_c.c_int32), _i, _i, _vp, _vp, _vp, _vp,
                                 _vp, _i, _vp]),
    "b2o_crops_to_input_color": (_i, [_vp, _vp, _i, _vp, _vp]),
    "b2o_crnn_workspace_bytes": (_sz, [_i]),
    "b2o_crops_to_input": (_i, [_vp, _vp, _i, _vp, _vp]),
    "b2o_crnn_forward": (_i, [_vp, _vp, _i, _vp, _vp, _sz, _vp]),
    "b2o_crnn_forward_scored": (_i, [_vp, _vp, _i, _vp, _vp, _vp, _sz, _vp]),
    "b2o_ctc_beam_decode": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _vp, _vp]),
    "b2o_crnn_forward_beam": (_i, [_vp, _vp, _i, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "b2o_ctc_beam_lm_decode": (_i, [_vp, _vp, _i, _i, _i, _i, _lmp, _vp, _vp, _vp, _vp]),
    "b2o_crnn_forward_beam_lm": (_i, [_vp, _vp, _i, _i, _i, _lmp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "b2o_ctc_beam_hotword_decode": (_i, [_vp, _vp, _i, _i, _i, _i, _lmp, _hwp, _vp, _vp, _vp, _vp]),
    "b2o_crnn_forward_beam_hotword": (_i, [_vp, _vp, _i, _i, _i, _lmp, _hwp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "b2o_ctc_beam_pattern_decode": (_i, [_vp, _vp, _i, _i, _i, _i, _patp, _vp, _vp, _vp]),
    "b2o_crnn_forward_beam_pattern": (_i, [_vp, _vp, _i, _i, _i, _patp, _vp, _vp, _vp, _sz, _vp]),
    "b2o_lexicon_workspace_bytes": (_sz, [_i, _i, _i]),
    "b2o_ctc_lexicon_decode": (_i, [_vp, _vp, _i, _i, _vp, _vp, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "b2o_crnn_forward_lexicon": (_i, [_vp, _vp, _i, _vp, _vp, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "b2o_ctc_align": (_i, [_vp, _vp, _i, _i, _vp, _i, _vp, _vp, _vp]),
    "b2o_char_cells": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "b2o_crnn_forward_logits": (_i, [_vp, _vp, _i, _vp, _vp, _vp, _sz, _vp]),
    "b2o_crnn_align": (_i, [_vp, _i, _vp, _i, _vp, _vp, _vp, _vp, _sz, _vp]),
    "b2o_ctc_char_scores": (_i, [_vp, _vp, _i, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp]),
    "b2o_crnn_char_scores": (_i, [_vp, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "b2o_crnn_features": (_i, [_vp, _vp, _i, _vp, _vp, _sz, _vp]),
    "b2o_ctc_train_workspace_bytes": (_sz, [_i, _i]),
    "b2o_ctc_loss_grad": (_i, [_vp, _vp, _i, _vp, _i, _i, _vp, _vp, _vp, _vp, _f, _c.c_uint64, _c.c_uint64, _vp, _vp,
                               _vp, _vp, _vp, _sz, _vp]),
    "b2o_rmsprop_step": (_i, [_vp, _vp, _vp, _vp, _c.c_int64, _f, _f, _f, _vp]),
    "b2o_crnn_set_top": (_i, [_vp, _vp, _vp, _i, _vp]),
    "b2o_crnn_sequence_features": (_i, [_vp, _vp, _i, _vp, _vp, _sz, _vp]),
    "b2o_rnn_train_workspace_bytes": (_sz, [_i, _i]),
    "b2o_rnn_loss_grad": (_i, [_vp, _vp, _i, _vp, _i, _i, _vp, _vp, _vp, _f, _c.c_uint64, _c.c_uint64, _vp, _vp, _vp,
                               _sz, _vp]),
    "b2o_set_debug_taps": (_i, [_vp, _i]),
    "b2o_crnn_tap": (_i, [_vp, _c.c_char_p, _vp, _i, _vp, _sz, _vp]),
    "b2o_conv2d_test": (_i, [_vp, _vp, _i, _i, _i, _i, _c.POINTER(_c.c_float), _i, _i, _i,
                             _c.POINTER(_c.c_float), _c.POINTER(_c.c_float), _i,
                             _c.POINTER(_c.c_float), _c.POINTER(_c.c_float), _vp, _i, _vp]),
    "b2o_conv_test": (_i, [_vp, _c.POINTER(_ConvTestDesc), _vp]),
    "b2o_conv_plan_test": (_i, [_c.POINTER(_ConvPlanDesc), _c.POINTER(_ConvPlan)]),
    "b2o_warp_plan_test": (_i, [_vp, _vp, _i, _vp, _vp]),
    "b2o_get_boxes_test": (_i, [_vp, _vp, _i, _i, _i, _f, _f, _f, _i, _vp, _vp, _vp, _i, _vp, _sz, _vp, _vp, _vp]),
}

# b2o_warp_plan (include/b2ocr.h), field for field: 9 float64, 3 int32, padded to 88 bytes
WARP_PLAN_DTYPE = np.dtype([("m", "<f8", (9,)), ("dw", "<i4"), ("dh", "<i4"), ("valid", "<i4")], align=True)

# b2o_window_plan (include/b2ocr.h), field for field: 12 float64, 4 int32 (112 bytes)
WINDOW_PLAN_DTYPE = np.dtype([("m", "<f8", (9,)), ("a", "<f8"), ("wc", "<f8"), ("sh", "<f8"), ("k", "<i4"),
                              ("dw", "<i4"), ("dh", "<i4"), ("valid", "<i4")], align=True)

_lib = None


def load_library():
    """dlopen libb2ocr.so and type every export of include/b2ocr.h (no GPU needed for this)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise B2OError(f"{LIB_PATH} not found: build it with `python keras-ocr_b200/build.py` "
                       "(there is no CPU fallback)")
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the .so does not export the symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def conv_plan(n, h, w, cin, cout, ksize, dilation=1, out_f32=False, pool=False, tail=False, up_add=False,
              engine=CONV_AUTO, swap=True, sm_count=132):
    """b2o_conv_plan_test (no GPU needed): the plan of one tensor-core convolution as a dict of b2o_conv_plan's fields,
    or None where the library refuses the launch."""
    desc = _ConvPlanDesc(n, h, w, cin, cout, ksize, dilation, int(out_f32), int(pool), int(tail), int(up_add), engine,
                         int(swap), sm_count)
    plan = _ConvPlan()
    if load_library().b2o_conv_plan_test(ctypes.byref(desc), ctypes.byref(plan)) != 0:
        return None
    return {name: getattr(plan, name) for name, _ in _ConvPlan._fields_}


def tile_plan(hp, wp, tile_size, margin):
    """b2o_tile_plan (no GPU needed): the tile grid of a padded (hp, wp) batch as a ``TilePlan``, or None where the
    library refuses the parameters."""
    plan = TilePlan()
    if load_library().b2o_tile_plan(int(hp), int(wp), int(tile_size), int(margin), ctypes.byref(plan)) != 0:
        return None
    return plan


def _tensor_array(weights):
    keep = []
    arr = (_Tensor * len(weights))()
    for k, (name, value) in enumerate(weights.items()):
        a = np.ascontiguousarray(np.asarray(value), dtype=np.float32)
        keep.append(a)
        arr[k].name = name.encode()
        arr[k].data = a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))
        arr[k].ndim = a.ndim
        for d in range(a.ndim):
            arr[k].shape[d] = a.shape[d]
    return arr, keep


def _fptr(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_float)) if a is not None else None


class Context:
    """One b2o_ctx per device.  All methods take raw device pointers (ints) and a stream (int)."""

    def __init__(self, device=0):
        self.lib = load_library()
        handle = _vp()
        rc = self.lib.b2o_create(int(device), ctypes.byref(handle))
        if rc != 0 or not handle:
            raise B2OError(f"b2o_create(device={device}) failed with status {rc}: an sm_90 (H100) GPU is "
                           "required and there is no CPU fallback")
        self.handle = handle
        self.device = device

    def close(self):
        if getattr(self, "handle", None):
            self.lib.b2o_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # pragma: no cover - interpreter shutdown
            pass

    def _check(self, rc, what):
        if rc != 0:
            msg = self.lib.b2o_last_error(self.handle)
            raise B2OError(f"{what} failed ({rc}): {msg.decode() if msg else ''}")

    def set_conv_engine(self, engine):
        self._check(self.lib.b2o_set_conv_engine(self.handle, engine), "b2o_set_conv_engine")

    def launch_count(self):
        return int(self.lib.b2o_launch_count(self.handle))

    def tile256_launches(self):
        """Tensor-core conv launches so far that ran channels by pixels on 16 x 16-pixel tiles."""
        return int(self.lib.b2o_tc_tile256_launches(self.handle))

    def coop_n_launches(self):
        """Tensor-core conv launches so far that ran paired n-tiles (both warpgroups sharing every activation box)."""
        return int(self.lib.b2o_tc_coop_n_launches(self.handle))

    def profile_enable(self, on):
        self._check(self.lib.b2o_profile_enable(self.handle, int(on)), "b2o_profile_enable")

    def profile_read(self):
        ms, flop, n = ctypes.c_double(), ctypes.c_double(), ctypes.c_int64()
        self._check(self.lib.b2o_profile_read(self.handle, ctypes.byref(ms), ctypes.byref(flop), ctypes.byref(n)),
                    "b2o_profile_read")
        return ms.value, flop.value, n.value

    def load_craft(self, weights):
        arr, keep = _tensor_array(weights)
        self._check(self.lib.b2o_load_craft(self.handle, arr, len(weights)), "b2o_load_craft")

    def load_crnn(self, weights):
        arr, keep = _tensor_array(weights)
        self._check(self.lib.b2o_load_crnn(self.handle, arr, len(weights)), "b2o_load_crnn")

    def resize_pad(self, src, hs, ws, hr, wr, dst, index, hp, wp, stream):
        self._check(self.lib.b2o_resize_pad(self.handle, src, hs, ws, hr, wr, dst, index, hp, wp, stream), "b2o_resize_pad")

    def resize_pad_batch(self, src, n, hs, ws, hr, wr, dst, hp, wp, gray, stream):
        self._check(self.lib.b2o_resize_pad_batch(self.handle, src, n, hs, ws, hr, wr, dst, hp, wp, gray, stream),
                    "b2o_resize_pad_batch")

    def jpeg_info(self, data):
        """(height, width, components) of a JPEG byte string, or None if nvJPEG is missing / refuses the stream."""
        buf = (ctypes.c_ubyte * len(data)).from_buffer_copy(data)
        h, w, c = _i(), _i(), _i()
        rc = self.lib.b2o_jpeg_info(self.handle, buf, len(data), ctypes.byref(h), ctypes.byref(w), ctypes.byref(c))
        return (h.value, w.value, c.value) if rc == 0 else None

    def decode_jpeg(self, data, rgb, h, w, stream):
        buf = (ctypes.c_ubyte * len(data)).from_buffer_copy(data)
        return self.lib.b2o_decode_jpeg(self.handle, buf, len(data), rgb, h, w, stream) == 0

    def rgb_to_gray(self, img, n, h, w, gray, stream):
        self._check(self.lib.b2o_rgb_to_gray(self.handle, img, n, h, w, gray, stream), "b2o_rgb_to_gray")

    def craft_workspace_bytes(self, n, h, w):
        return int(self.lib.b2o_craft_workspace_bytes(n, h, w))

    def craft_forward(self, img, n, h, w, scores, ws, ws_bytes, stream):
        self._check(self.lib.b2o_craft_forward(self.handle, img, n, h, w, scores, ws, ws_bytes, stream), "b2o_craft_forward")

    def craft_forward_until(self, img, n, h, w, scores, ws, ws_bytes, last_step, stream):
        self._check(self.lib.b2o_craft_forward_until(self.handle, img, n, h, w, scores, ws, ws_bytes, last_step, stream),
                    "b2o_craft_forward_until")

    def craft_tap(self, name, ws, n, h, w, out, out_bytes, stream):
        """b2o_craft_tap: raises B2OError; its status (B2O_ERR_STATE = -5 for a buffer that is not live) is in the
        message."""
        self._check(self.lib.b2o_craft_tap(self.handle, name.encode(), ws, n, h, w, out, out_bytes, stream),
                    "b2o_craft_tap")

    def cut_tiles(self, img, n, plan, first_tile, n_tiles, tiles, stream):
        self._check(self.lib.b2o_cut_tiles(self.handle, img, n, ctypes.byref(plan), first_tile, n_tiles, tiles, stream),
                    "b2o_cut_tiles")

    def stitch_tiles(self, tile_scores, n, plan, first_tile, n_tiles, scores, stream):
        self._check(self.lib.b2o_stitch_tiles(self.handle, tile_scores, n, ctypes.byref(plan), first_tile, n_tiles,
                                              scores, stream), "b2o_stitch_tiles")

    def boxes_workspace_bytes(self, n, hs, ws, max_boxes):
        return int(self.lib.b2o_boxes_workspace_bytes(n, hs, ws, max_boxes))

    def get_boxes(self, scores, n, hs, ws, det, text, link, size, boxes, counts, max_boxes, wsp, ws_bytes, stream):
        self._check(self.lib.b2o_get_boxes(self.handle, scores, n, hs, ws, det, text, link, size, boxes, counts,
                                           max_boxes, wsp, ws_bytes, stream), "b2o_get_boxes")

    def get_boxes_scored(self, scores, n, hs, ws, det, text, link, size, boxes, counts, box_scores, max_boxes, wsp,
                         ws_bytes, stream):
        self._check(self.lib.b2o_get_boxes_scored(self.handle, scores, n, hs, ws, det, text, link, size, boxes, counts,
                                                  box_scores, max_boxes, wsp, ws_bytes, stream), "b2o_get_boxes_scored")

    def compact_boxes(self, boxes, counts, n, max_boxes, flat, image_index, stream):
        self._check(self.lib.b2o_compact_boxes(self.handle, boxes, counts, n, max_boxes, flat, image_index, stream),
                    "b2o_compact_boxes")

    def get_boxes_poly(self, scores, n, hs, ws, det, text, link, size, boxes, counts, box_scores, polys, points,
                       max_boxes, wsp, ws_bytes, stream):
        self._check(self.lib.b2o_get_boxes_poly(self.handle, scores, n, hs, ws, det, text, link, size, boxes, counts,
                                                box_scores, polys, points, max_boxes, wsp, ws_bytes, stream),
                    "b2o_get_boxes_poly")

    def compact_polys(self, polys, points, counts, n, max_boxes, flat_polys, flat_points, image_index, stream):
        self._check(self.lib.b2o_compact_polys(self.handle, polys, points, counts, n, max_boxes, flat_polys, flat_points,
                                               image_index, stream), "b2o_compact_polys")

    def warp_polys(self, img, channels, n, h, w, polys, points, image_index, n_polys, crops, crnn_in, stream):
        self._check(self.lib.b2o_warp_polys(self.handle, img, channels, n, h, w, polys, points, image_index, n_polys,
                                            crops, crnn_in, stream), "b2o_warp_polys")

    def lines_workspace_bytes(self, n, max_boxes):
        return int(self.lib.b2o_lines_workspace_bytes(n, max_boxes))

    def group_lines(self, boxes, counts, n, max_boxes, cos_tol, height_ratio, offset_ratio, gap_ratio, line_counts,
                    word_order, line_start, line_boxes, ws, ws_bytes, stream):
        self._check(self.lib.b2o_group_lines(self.handle, boxes, counts, n, max_boxes, float(cos_tol),
                                             float(height_ratio), float(offset_ratio), float(gap_ratio), line_counts,
                                             word_order, line_start, line_boxes, ws, ws_bytes, stream),
                    "b2o_group_lines")

    def blocks_workspace_bytes(self, n, max_boxes):
        return int(self.lib.b2o_blocks_workspace_bytes(n, max_boxes))

    def group_blocks(self, line_counts, line_start, line_boxes, n, max_boxes, row_gap, col_gap, block_counts,
                     line_order, block_start, block_boxes, ws, ws_bytes, stream):
        self._check(self.lib.b2o_group_blocks(self.handle, line_counts, line_start, line_boxes, n, max_boxes,
                                              float(row_gap), float(col_gap), block_counts, line_order, block_start,
                                              block_boxes, ws, ws_bytes, stream), "b2o_group_blocks")

    def window_counts(self, boxes, counts, n, max_boxes, max_windows, windows, stream):
        self._check(self.lib.b2o_window_counts(self.handle, boxes, counts, n, max_boxes, max_windows, windows, stream),
                    "b2o_window_counts")

    def warp_windows(self, img, channels, n, h, w, boxes, image_index, words, win_start, n_words, max_windows, first,
                     count, crops, crnn_in, stream):
        self._check(self.lib.b2o_warp_windows(self.handle, img, channels, n, h, w, boxes, image_index, words, win_start,
                                              n_words, max_windows, first, count, crops, crnn_in, stream),
                    "b2o_warp_windows")

    def stitch_windows(self, logits, k, theta, boxes, words, win_start, n_words, max_windows, labels, logp, stream):
        self._check(self.lib.b2o_stitch_windows(self.handle, logits, k, theta, boxes, words, win_start, n_words,
                                                max_windows, labels, logp, stream), "b2o_stitch_windows")

    def window_plan_test(self, boxes, n, max_windows, plans, stream):
        """b2o_window_plan_test: ``plans`` addresses n * max_windows records of WINDOW_PLAN_DTYPE on the device."""
        self._check(self.lib.b2o_window_plan_test(self.handle, boxes, n, max_windows, plans, stream),
                    "b2o_window_plan_test")

    def record_floats(self, rec_boxes):
        return int(self.lib.b2o_record_floats(rec_boxes))

    def pack_records(self, boxes, counts, labels, inv_scale, n, max_boxes, rows, rec_boxes, records, stream):
        self._check(self.lib.b2o_pack_records(self.handle, boxes, counts, labels, inv_scale, n, max_boxes, rows,
                                              rec_boxes, records, stream), "b2o_pack_records")

    def record_floats_scored(self, rec_boxes):
        return int(self.lib.b2o_record_floats_scored(rec_boxes))

    def pack_records_scored(self, boxes, counts, labels, box_scores, logp, inv_scale, n, max_boxes, rows, rec_boxes,
                            records, stream):
        self._check(self.lib.b2o_pack_records_scored(self.handle, boxes, counts, labels, box_scores, logp, inv_scale, n,
                                                     max_boxes, rows, rec_boxes, records, stream),
                    "b2o_pack_records_scored")

    def warp_boxes(self, gray, n, h, w, boxes, image_index, n_boxes, crops, crnn_in, stream, color=False):
        fn = self.lib.b2o_warp_boxes_color if color else self.lib.b2o_warp_boxes
        self._check(fn(self.handle, gray, n, h, w, boxes, image_index, n_boxes, crops, crnn_in, stream), "b2o_warp_boxes")

    def warp_boxes_turned(self, img, channels, n, h, w, boxes, image_index, n_boxes, turn, crops, crnn_in, stream):
        self._check(self.lib.b2o_warp_boxes_turned(self.handle, img, channels, n, h, w, boxes, image_index, n_boxes,
                                                   turn, crops, crnn_in, stream), "b2o_warp_boxes_turned")

    def select_rotation(self, labels, logp, image_index, n_images, b, top_paths, turns, vote, labels_out, logp_out,
                        turn_out, boxes, table, max_boxes, stream):
        """b2o_select_rotation: ``turns`` a host sequence of ints, ``vote`` ROTATION_VOTE_WORD / ROTATION_VOTE_PAGE."""
        t = (ctypes.c_int32 * len(turns))(*[int(r) for r in turns])
        self._check(self.lib.b2o_select_rotation(self.handle, labels, logp, image_index, n_images, b, top_paths, t,
                                                 len(turns), vote, labels_out, logp_out, turn_out, boxes, table,
                                                 max_boxes, stream), "b2o_select_rotation")

    def crnn_workspace_bytes(self, b):
        return int(self.lib.b2o_crnn_workspace_bytes(b))

    def crops_to_input(self, crops, b, crnn_in, stream, color=False):
        fn = self.lib.b2o_crops_to_input_color if color else self.lib.b2o_crops_to_input
        self._check(fn(self.handle, crops, b, crnn_in, stream), "b2o_crops_to_input")

    def crnn_forward(self, crnn_in, b, labels, ws, ws_bytes, stream):
        self._check(self.lib.b2o_crnn_forward(self.handle, crnn_in, b, labels, ws, ws_bytes, stream), "b2o_crnn_forward")

    def crnn_forward_scored(self, crnn_in, b, labels, logp, ws, ws_bytes, stream):
        self._check(self.lib.b2o_crnn_forward_scored(self.handle, crnn_in, b, labels, logp, ws, ws_bytes, stream),
                    "b2o_crnn_forward_scored")

    def ctc_beam_decode(self, logits, b, k, beam_width, top_paths, labels, logp, stream):
        self._check(self.lib.b2o_ctc_beam_decode(self.handle, logits, b, k, beam_width, top_paths, labels, logp, stream),
                    "b2o_ctc_beam_decode")

    def crnn_forward_beam(self, crnn_in, b, beam_width, top_paths, labels, logp, ws, ws_bytes, stream):
        self._check(self.lib.b2o_crnn_forward_beam(self.handle, crnn_in, b, beam_width, top_paths, labels, logp, ws,
                                                   ws_bytes, stream), "b2o_crnn_forward_beam")

    def ctc_beam_lm_decode(self, logits, b, k, beam_width, top_paths, lm, labels, logp, fused, stream):
        """``lm``: a ``CharLMDesc``."""
        self._check(self.lib.b2o_ctc_beam_lm_decode(self.handle, logits, b, k, beam_width, top_paths, ctypes.byref(lm),
                                                    labels, logp, fused, stream), "b2o_ctc_beam_lm_decode")

    def crnn_forward_beam_lm(self, crnn_in, b, beam_width, top_paths, lm, labels, logp, fused, ws, ws_bytes, stream):
        self._check(self.lib.b2o_crnn_forward_beam_lm(self.handle, crnn_in, b, beam_width, top_paths, ctypes.byref(lm),
                                                      labels, logp, fused, ws, ws_bytes, stream),
                    "b2o_crnn_forward_beam_lm")

    def ctc_beam_hotword_decode(self, logits, b, k, beam_width, top_paths, lm, hw, labels, logp, fused, stream):
        """``lm``: a ``CharLMDesc`` or None (no model); ``hw``: a ``HotwordsDesc``."""
        self._check(self.lib.b2o_ctc_beam_hotword_decode(self.handle, logits, b, k, beam_width, top_paths,
                                                         None if lm is None else ctypes.byref(lm), ctypes.byref(hw),
                                                         labels, logp, fused, stream), "b2o_ctc_beam_hotword_decode")

    def crnn_forward_beam_hotword(self, crnn_in, b, beam_width, top_paths, lm, hw, labels, logp, fused, ws, ws_bytes,
                                  stream):
        self._check(self.lib.b2o_crnn_forward_beam_hotword(self.handle, crnn_in, b, beam_width, top_paths,
                                                           None if lm is None else ctypes.byref(lm), ctypes.byref(hw),
                                                           labels, logp, fused, ws, ws_bytes, stream),
                    "b2o_crnn_forward_beam_hotword")

    def ctc_beam_pattern_decode(self, logits, b, k, beam_width, top_paths, pattern, labels, logp, stream):
        """``pattern``: a ``PatternDesc``."""
        self._check(self.lib.b2o_ctc_beam_pattern_decode(self.handle, logits, b, k, beam_width, top_paths,
                                                         ctypes.byref(pattern), labels, logp, stream),
                    "b2o_ctc_beam_pattern_decode")

    def crnn_forward_beam_pattern(self, crnn_in, b, beam_width, top_paths, pattern, labels, logp, ws, ws_bytes, stream):
        self._check(self.lib.b2o_crnn_forward_beam_pattern(self.handle, crnn_in, b, beam_width, top_paths,
                                                           ctypes.byref(pattern), labels, logp, ws, ws_bytes, stream),
                    "b2o_crnn_forward_beam_pattern")

    def lexicon_workspace_bytes(self, b, n_words, top_paths):
        return int(self.lib.b2o_lexicon_workspace_bytes(b, n_words, top_paths))

    def ctc_lexicon_decode(self, logits, b, k, offsets, labels, n_words, top_paths, labels_out, logp, ws, ws_bytes,
                           stream):
        self._check(self.lib.b2o_ctc_lexicon_decode(self.handle, logits, b, k, offsets, labels, n_words, top_paths,
                                                    labels_out, logp, ws, ws_bytes, stream), "b2o_ctc_lexicon_decode")

    def crnn_forward_lexicon(self, crnn_in, b, offsets, labels, n_words, top_paths, labels_out, logp, ws, ws_bytes,
                             stream):
        self._check(self.lib.b2o_crnn_forward_lexicon(self.handle, crnn_in, b, offsets, labels, n_words, top_paths,
                                                      labels_out, logp, ws, ws_bytes, stream), "b2o_crnn_forward_lexicon")

    def ctc_align(self, logits, b, k, labels, top_paths, spans, logp, stream):
        self._check(self.lib.b2o_ctc_align(self.handle, logits, b, k, labels, top_paths, spans, logp, stream),
                    "b2o_ctc_align")

    def char_cells(self, spans, b, top_paths, theta, boxes, turns, cells, stream):
        self._check(self.lib.b2o_char_cells(self.handle, spans, b, top_paths, theta, boxes, turns, cells, stream),
                    "b2o_char_cells")

    def crnn_forward_logits(self, crnn_in, b, labels, logp, ws, ws_bytes, stream):
        self._check(self.lib.b2o_crnn_forward_logits(self.handle, crnn_in, b, labels, logp, ws, ws_bytes, stream),
                    "b2o_crnn_forward_logits")

    def crnn_align(self, b, labels, top_paths, spans, logp, theta, ws, ws_bytes, stream):
        self._check(self.lib.b2o_crnn_align(self.handle, b, labels, top_paths, spans, logp, theta, ws, ws_bytes, stream),
                    "b2o_crnn_align")

    def ctc_char_scores(self, logits, b, k, labels, top_paths, alternatives, conf, alt_labels, alt_post, logp, stream):
        self._check(self.lib.b2o_ctc_char_scores(self.handle, logits, b, k, labels, top_paths, alternatives, conf,
                                                 alt_labels, alt_post, logp, stream), "b2o_ctc_char_scores")

    def crnn_char_scores(self, b, labels, top_paths, alternatives, conf, alt_labels, alt_post, logp, ws, ws_bytes,
                         stream):
        self._check(self.lib.b2o_crnn_char_scores(self.handle, b, labels, top_paths, alternatives, conf, alt_labels,
                                                  alt_post, logp, ws, ws_bytes, stream), "b2o_crnn_char_scores")

    def crnn_features(self, crnn_in, b, features, ws, ws_bytes, stream):
        self._check(self.lib.b2o_crnn_features(self.handle, crnn_in, b, features, ws, ws_bytes, stream),
                    "b2o_crnn_features")

    def ctc_train_workspace_bytes(self, b, k):
        return int(self.lib.b2o_ctc_train_workspace_bytes(b, k))

    def ctc_loss_grad(self, features, n_rows, index, b, k, w, bias, offsets, labels, dropout, seed, step, loss, grad_w,
                      grad_b, logits, ws, ws_bytes, stream):
        self._check(self.lib.b2o_ctc_loss_grad(self.handle, features, n_rows, index, b, k, w, bias, offsets, labels,
                                               float(dropout), int(seed), int(step), loss, grad_w, grad_b, logits, ws,
                                               ws_bytes, stream), "b2o_ctc_loss_grad")

    def rmsprop_step(self, param, grad, acc, n, lr, rho, eps, stream):
        self._check(self.lib.b2o_rmsprop_step(self.handle, param, grad, acc, n, lr, rho, eps, stream), "b2o_rmsprop_step")

    def crnn_set_top(self, w, bias, k, stream):
        self._check(self.lib.b2o_crnn_set_top(self.handle, w, bias, k, stream), "b2o_crnn_set_top")

    def crnn_sequence_features(self, crnn_in, b, out, ws, ws_bytes, stream):
        self._check(self.lib.b2o_crnn_sequence_features(self.handle, crnn_in, b, out, ws, ws_bytes, stream),
                    "b2o_crnn_sequence_features")

    def rnn_train_workspace_bytes(self, b, k):
        return int(self.lib.b2o_rnn_train_workspace_bytes(b, k))

    def rnn_loss_grad(self, x, n_rows, index, b, k, params, offsets, labels, dropout, seed, step, loss, grad, ws,
                      ws_bytes, stream):
        self._check(self.lib.b2o_rnn_loss_grad(self.handle, x, n_rows, index, b, k, params, offsets, labels,
                                               float(dropout), int(seed), int(step), loss, grad, ws, ws_bytes, stream),
                    "b2o_rnn_loss_grad")

    def set_debug_taps(self, on):
        self._check(self.lib.b2o_set_debug_taps(self.handle, int(on)), "b2o_set_debug_taps")

    def crnn_tap(self, name, ws, b, out, out_bytes, stream):
        self._check(self.lib.b2o_crnn_tap(self.handle, name.encode(), ws, b, out, out_bytes, stream), "b2o_crnn_tap")

    def conv2d_test(self, x, n, h, w, cin, wgt, cout, ksize, dilation, s1, t1, relu, s2, t2, out, engine, stream):
        wgt = np.ascontiguousarray(wgt, np.float32)
        s1 = np.ascontiguousarray(s1, np.float32)
        t1 = np.ascontiguousarray(t1, np.float32)
        s2 = None if s2 is None else np.ascontiguousarray(s2, np.float32)
        t2 = None if t2 is None else np.ascontiguousarray(t2, np.float32)
        self._check(self.lib.b2o_conv2d_test(self.handle, x, n, h, w, cin, _fptr(wgt), cout, ksize, dilation, _fptr(s1),
                                             _fptr(t1), int(relu), _fptr(s2), _fptr(t2), out, engine, stream),
                    "b2o_conv2d_test")

    def conv_test(self, x, n, h, w, cin, x_ld, wgt, cout, ksize, dilation, s1, t1, relu, s2, t2, out, out_ld, engine,
                  stream, out_f32=False, write_full=True, pool=None, pool_ld=0, up=None, up_ld=0, tail=None, scores=None):
        """b2o_conv_test: device pointers are ints (channel 0 of their slice); ``tail`` = (w6 (16,16), b6, w8 (16,2), b8)
        host arrays, ``scores`` the device pointer of the (n,h,w,2) fp32 output."""
        keep = [np.ascontiguousarray(a, np.float32) if a is not None else None for a in (wgt, s1, t1, s2, t2)]
        tail = [np.ascontiguousarray(a, np.float32) for a in tail] if tail is not None else [None] * 4
        d = _ConvTestDesc(x, n, h, w, cin, x_ld, _fptr(keep[0]), cout, ksize, dilation, _fptr(keep[1]), _fptr(keep[2]),
                          int(relu), _fptr(keep[3]), _fptr(keep[4]), out, out_ld, int(out_f32), int(write_full),
                          pool, pool_ld, up, up_ld, *[_fptr(a) for a in tail], scores, engine)
        self._check(self.lib.b2o_conv_test(self.handle, ctypes.byref(d), stream), "b2o_conv_test")

    def warp_plan_test(self, boxes, n, plans, stream):
        """b2o_warp_plan_test: ``plans`` addresses n records of WARP_PLAN_DTYPE on the device."""
        self._check(self.lib.b2o_warp_plan_test(self.handle, boxes, n, plans, stream), "b2o_warp_plan_test")

    def get_boxes_test(self, scores, n, hs, ws, det, text, link, size, boxes, counts, box_scores, max_boxes, wsp,
                       ws_bytes, labels, comps, stream):
        """b2o_get_boxes_test: b2o_get_boxes_scored plus the label plane (n,hs,ws) int32 and the kept components
        (n,max_boxes,7) int32 (root, left, top, width, height, area, maxtext key)."""
        self._check(self.lib.b2o_get_boxes_test(self.handle, scores, n, hs, ws, det, text, link, size, boxes, counts,
                                                box_scores, max_boxes, wsp, ws_bytes, labels, comps, stream),
                    "b2o_get_boxes_test")


_contexts = {}


def get_context(device=0):
    """Process-wide context cache (weights are loaded per owner object, see Detector/Recognizer)."""
    if device not in _contexts:
        _contexts[device] = Context(device)
    return _contexts[device]
