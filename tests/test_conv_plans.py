"""The plans of the tensor-core convolutions (``plan_conv_tc`` in keras-ocr_b200/csrc/conv_tc.cu, through
``b2o_conv_plan_test``) against the restatement here.  CPU only.

Every tensor-core convolution the CRAFT and CRNN forwards launch -- at the views they launch it on, with the fused pool,
fused tail and (commuted decoder) upsample-add each one uses -- on both tensor-core engines, at the sizes of
tests/test_gpu_craft_stages.py, the bench's detector input and the recognizer's maps, in batches of 1 to 300; and every
distinct such layer over a sweep of small and odd maps.  Each must have a plan whose instance is compiled, whose shared
memory fits a CTA, whose barriers' transaction counts fit an mbarrier and whose ring holds 2 to 8 stages; the choices
that change the order in which an output's products are added (halo or generic tiles, the body, MODE and the halo tile)
must not change with the batch, since a crop's result may not change with the batch it travels in; and the plan must
equal ``restate``: the K chunk and N tile, ``pick_box``, the halo cover rule, the resident filter bank and the
channels-by-pixels rules (``swap`` off turns both channels-by-pixels bodies off).
"""
import collections
import functools

import pytest

from keras_ocr_b200 import _lib
from keras_ocr_b200 import weights as W
from tests import stage_refs as R
from tests.test_gpu_craft_stages import SIZES

AUTO, GENERIC = _lib.CONV_AUTO, _lib.CONV_TC_GENERIC
PIXELS, CHANNELS, TILE256 = 0, 1, 2          # b2o_conv_plan.body
SMEM = 227 * 1024                            # a CTA's dynamic shared memory on sm_90
TX_MAX = (1 << 20) - 1                       # an mbarrier's transaction count
TAIL_BYTES = (256 + 16 + 32 + 2) * 4         # the fused tail's constants, staged in shared memory
BATCHES = [1, 2, 3, 7, 33, 132, 133, 300]
BENCH = (1536, 1536)                         # bench.py's detector input
CRNN_MAPS = {"in": (200, 31), "x1": (200, 31), "x2": (200, 31), "p3": (100, 15), "x4": (100, 15), "p5": (50, 7),
             "x6": (50, 7)}
# the compiled conv_tc_kernel<BLOCK_N, KCH, MODE, PAIR, UPADD> instances
COMBOS = [(16, 64), (32, 64), (64, 64), (128, 64), (16, 32), (32, 32), (32, 16), (64, 16)]
COMPILED = ({(bn, kch, mode, 0, 0) for bn, kch in COMBOS for mode in (0, 1, 2)} |
            {(bn, 64, mode, 1, 0) for bn in (64, 128) for mode in (0, 1, 2)} | {(64, 64, 0, 0, 1), (128, 64, 0, 0, 1)})

Launch = collections.namedtuple("Launch", "layer n h w cin cout k dil out_f32 pool tail up_add")


# ------------------------------------------------------------------------------------------------ the restatement
def tiling(cin, cout):
    """(K chunk, N tile) of a layer; N tile 0: the layer runs on the SIMT engine."""
    kch = 64 if cin % 64 == 0 else 32 if cin % 32 == 0 else 16 if cin % 16 == 0 else 0
    if kch == 0 or cout % 16:
        return kch, 0
    bn = 128
    while bn > 16 and cout % bn:
        bn //= 2
    if cout % bn or (kch == 32 and bn > 32) or (kch == 16 and bn not in (32, 64)):
        return kch, 0
    return kch, bn


@functools.lru_cache(maxsize=None)
def pick_box(n, h, w):
    """The (bw, bh, bn) power-of-two 128-pixel box of the generic tiles that wastes the fewest pixels, wide rows first on
    ties, and the pixels it covers: ((bw, bh, bn), cover)."""
    best, box, best_cover = 1e30, (128, 1, 1), 0.0
    for lw in range(8):
        for lh in range(8 - lw):
            ln = 7 - lw - lh
            bw, bh, bn = 1 << lw, 1 << lh, 1 << ln
            if ln > 0 and bn > 2 * n:
                continue
            cover = float(-(-w // bw) * bw) * float(-(-h // bh) * bh) * float(-(-n // bn) * bn)
            score = cover * (1.0 + 0.001 * (7 - lw)) * (1.05 if (bw < 8 and w >= 8) else 1.0)
            if score < best:
                best, box, best_cover = score, (bw, bh, bn), cover
    return box, best_cover


def halo_tiles(h, w, k, dil, pool, engine):
    """3x3 layers of dilation 1 take the 8 x 16 halo tile on the AUTO engine when a fused pool needs it, or when it
    covers at most 15 % more pixels of an image than the best generic box: both per image (as if the batch were
    unbounded), so the choice never depends on the batch."""
    if k != 3 or dil != 1 or engine == GENERIC:
        return False
    big = 1 << 20
    return pool or float((w + 7) // 8 * 8) * float((h + 15) // 16 * 16) <= 1.15 * (pick_box(big, h, w)[1] / big)


def restate(n, h, w, cin, cout, k, dil=1, out_f32=False, pool=False, tail=False, up_add=False, engine=AUTO, swap=True):
    """The plan's fields that follow from the rules, or None where the launch is refused."""
    kch, bn = tiling(cin, cout)
    if up_add and (k != 1 or kch != 64 or bn < 64 or out_f32 or pool or tail or h % 2 or w % 2):
        return None
    if (tail and (bn != 16 or cout != 16 or pool)) or bn == 0:
        return None
    halo = halo_tiles(h, w, k, dil, pool, engine)
    if pool and (not halo or out_f32):
        return None
    pooled_pixels = not pool or (h >= 2 and w >= 2)
    # channels by pixels: the 64-channel fp16 layers
    ct = swap and cout == 64 and bn == 64 and not out_f32 and not up_add and not tail and pooled_pixels
    b_bytes = bn * kch * 2
    out_tiles = 2 * 128 * 64 * 2 + (2 * 32 * 64 * 2 if pool else 0)
    budget = SMEM - 1024 - 512 - (TAIL_BYTES if tail else 0) - (out_tiles if ct else 0)
    a_bytes = (18 * 8 if halo else 128) * kch * 2
    a_stride = -(-a_bytes // 1024) * 1024
    bank = k * k * cin * bn * 2
    # the whole filter bank in shared memory: halo tiles, one N tile, two stages beside it, one barrier's transaction
    resident = halo and cout == bn and bank + 2 * a_stride <= budget and bank <= TX_MAX
    # channels by pixels on 16 x 16 tiles: the streamed 128-channel fp16 halo layers, where a 16-wide tile covers the
    # same columns as an 8-wide one
    t256 = (swap and halo and not resident and kch == 64 and bn == 128 and not out_f32 and not up_add and not tail and
            (w + 15) // 16 * 16 == (w + 7) // 8 * 8 and pooled_pixels)
    if t256:
        a_bytes = a_stride = 18 * 16 * kch * 2
    box = (16, 16, 1) if t256 else (8, 16, 1) if halo else pick_box(n, h, w)[0]
    filter_taps = 0 if resident else 3 if halo else 1
    return dict(block_n=bn, kch=kch, mode=2 if resident else 1 if halo else 0, pair=0, upadd=int(up_add),
                body=TILE256 if t256 else CHANNELS if ct else PIXELS, tile_w=box[0], tile_h=box[1], tile_n=box[2],
                tiles=-(-w // box[0]) * -(-h // box[1]) * -(-n // box[2]) * (cout // bn),
                stage_bytes=a_stride + filter_taps * b_bytes, stage_tx=a_bytes + filter_taps * b_bytes,
                resident_bytes=bank if resident else 0)


# ------------------------------------------------------------------------------------------------ the forwards' launches
def craft_launches(n, h, w, engine):
    """Every tensor-core launch of b2o_craft_forward on (n, h, w, 3) images.  On AUTO the pool and the tail are fused,
    and the commuted halves of upconvN.conv.0 (B2O_UPCONV_COMMUTE=1) run where the skip tensor is exactly twice the
    decoder tensor: ".y" on the decoder tensor, ".s" on the skip tensor with the upsample-add."""
    dims = R.craft_dims(h, w)
    auto = engine == AUTO
    level = lambda s: dims[R.CRAFT_BUFS[s[0]][0]]            # noqa: E731
    out = []
    for i, st in enumerate(R.CRAFT_STEPS):
        kind = st["kind"]
        if kind == "stem":                                   # slice1.0 over the 16-channel input
            out.append(Launch("stem16", n, *dims[1], 16, 64, 3, 1, False, False, False, False))
        if kind in ("conv", "upconv"):
            cin, cout, k, dil, _, _ = R.CRAFT_LAYERS[st["layer"]]
            tail = auto and R.CRAFT_STEPS[i + 1]["kind"] == "tail"
            out.append(Launch(st["layer"], n, *level(st["src"]), cin, cout, k, dil, False, auto and "pool" in st, tail,
                              False))
        if kind == "upconv" and auto:
            (yh, yw), (sh, sw) = level(st["y"]), level(st["skip"])
            if (sh, sw) == (2 * yh, 2 * yw):
                cin, cout = R.CRAFT_LAYERS[st["layer"]][:2]
                cy = st["skip"][1]                           # the decoder tensor's channels come first in the concat
                out.append(Launch(st["layer"] + ".y", n, yh, yw, cy, cout, 1, 1, False, False, False, False))
                out.append(Launch(st["layer"] + ".s", n, sh, sw, cin - cy, cout, 1, 1, False, False, False, True))
    return out


def crnn_launches(b, engine):
    """Every tensor-core launch of b2o_crnn_forward on b crops: conv_2 .. conv_7 (conv_1 runs on the CUDA cores), the
    STN (conv_a as a 1x1 GEMM on AUTO) and the dense layers, at the views crnn_forward gives them."""
    auto = engine == AUTO
    convs = {name: (cin, cout, k) for name, cin, cout, k, _ in W.CRNN_CONVS}
    out = [Launch(layer, b, *CRNN_MAPS[src], *convs[layer], 1, False, auto and pool is not None, False, False)
           for layer, src, _, pool in R.CRNN_STEPS if layer != "conv_1"]
    stn_a = ("stn.conv_a_gemm", 512, 512, 1) if auto else ("stn.conv_a", 512, 16, 5)
    flat = lambda name, rows, cin, cout, f32=False: Launch(name, 1, 1, rows, cin, cout, 1, 1, f32, False, False, False)  # noqa: E731
    return out + [
        Launch(stn_a[0], b, 50, 7, *stn_a[1:], 1, False, False, False, False),
        Launch("stn.conv_b", b, 50, 7, 16, 32, 5, 1, False, False, False, False),
        flat("stn.dense_a", b, 11200, 64), flat("fc_9", 50 * b, 3584, 128),
        flat("lstm_in_1", 50 * b, 128, 1024, True), flat("lstm_in_2", 50 * b, 128, 1024, True),
    ]


# ------------------------------------------------------------------------------------------------ checks
def _plan(lc, engine, swap):
    return _lib.conv_plan(lc.n, lc.h, lc.w, lc.cin, lc.cout, lc.k, lc.dil, lc.out_f32, lc.pool, lc.tail, lc.up_add,
                          engine, swap)


def _restated(lc, engine, swap):
    return restate(lc.n, lc.h, lc.w, lc.cin, lc.cout, lc.k, lc.dil, lc.out_f32, lc.pool, lc.tail, lc.up_add, engine, swap)


def _check(lc, engine, swap, must_exist=True):
    """The plan of one launch against the invariants and the restatement; returns the fields that may not depend on
    the batch (None where the launch is refused)."""
    got, want = _plan(lc, engine, swap), _restated(lc, engine, swap)
    if must_exist:
        assert got is not None, (lc, engine, swap, "no plan")
    if got is None or want is None:
        assert got == want, (lc, engine, swap, got, want)
        return None
    assert {key: got[key] for key in want} == want, (lc, engine, swap, got, want)
    assert (got["block_n"], got["kch"], got["mode"], got["pair"], got["upadd"]) in COMPILED, (lc, got)
    assert got["smem_bytes"] <= SMEM, (lc, got)
    assert got["stages"] * got["stage_bytes"] + got["resident_bytes"] <= got["smem_bytes"], (lc, got)
    assert got["stage_tx"] <= TX_MAX and got["resident_bytes"] <= TX_MAX, (lc, got)
    assert 2 <= got["stages"] <= 8, (lc, got)
    assert got["grid"] == min(got["tiles"], 132), (lc, got)
    if not swap:
        assert got["body"] == PIXELS, (lc, got)
    return got["mode"], got["body"], (got["tile_w"], got["tile_h"]) if got["mode"] else None


def _check_batches(launches_of, engine, swap, must_exist=True):
    """launches_of(b): the launches for batch b, the same layers in the same order for every b."""
    seen = {}
    for b in BATCHES:
        for i, lc in enumerate(launches_of(b)):
            key = _check(lc, engine, swap, must_exist)
            assert seen.setdefault(i, key) == key, (lc, engine, swap, "changes with the batch", seen[i], key)


FORWARD_SHAPES = sorted({(h, w) for _, h, w in SIZES} | {BENCH})


@pytest.mark.parametrize("swap", [1, 0])
@pytest.mark.parametrize("engine", [AUTO, GENERIC], ids=["auto", "tc_generic"])
@pytest.mark.parametrize("shape", FORWARD_SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
def test_craft_forward_plans(shape, engine, swap):
    _check_batches(lambda b: craft_launches(b, *shape, engine), engine, swap)


@pytest.mark.parametrize("swap", [1, 0])
@pytest.mark.parametrize("engine", [AUTO, GENERIC], ids=["auto", "tc_generic"])
def test_crnn_forward_plans(engine, swap):
    _check_batches(lambda b: crnn_launches(b, engine), engine, swap)


def _distinct_layers():
    """Every distinct (layer shape, epilogue) the forwards launch on either engine."""
    found = {}
    for engine in (AUTO, GENERIC):
        for lc in craft_launches(1, 64, 64, engine) + crnn_launches(1, engine):
            found.setdefault(lc._replace(layer=None, n=0, h=0, w=0), lc.layer + ("" if engine == AUTO else "/generic"))
    return found


LAYERS = _distinct_layers()
# every height 1..70 against a few widths and every width against a few heights, and very long thin maps
SWEEP = sorted({(h, w) for h in range(1, 71) for w in (1, 2, 7, 8, 9, 16, 17, 31, 33, 70)} |
               {(h, w) for w in range(1, 71) for h in (1, 2, 15, 16, 17, 31, 70)} |
               {(2048, 40), (32, 2048), (40, 2048), (2048, 32)})


@pytest.mark.parametrize("layer", list(LAYERS), ids=list(LAYERS.values()))
def test_small_and_odd_maps(layer):
    """A plan wherever the library takes the launch; refused only where the restatement refuses it (an upsample-add
    over an odd map)."""
    engine = GENERIC if LAYERS[layer].endswith("/generic") else AUTO
    for h, w in SWEEP:
        _check_batches(lambda b: [layer._replace(n=b, h=h, w=w)], engine, 1, must_exist=not layer.up_add)


def test_every_layer_of_the_forwards_is_swept():
    """The forwards' tensor-core layers at both engines: what the sweep covers."""
    names = set(LAYERS.values())
    assert {"stem16", "basenet.slice1.3", "conv_cls.4", "upconv4.conv.0.s", "stn.conv_a_gemm", "lstm_in_1",
            "stn.conv_a/generic"} <= names, names
    assert any(lc.tail for lc in LAYERS) and any(lc.pool for lc in LAYERS) and any(lc.up_add for lc in LAYERS)


def test_refusals():
    """Launches the library has no plan for."""
    assert _lib.conv_plan(1, 32, 32, 64, 64, 3, 2, pool=True) is None                    # pool on generic tiles
    assert _lib.conv_plan(1, 32, 32, 64, 64, 3, pool=True, engine=GENERIC) is None       # the same
    assert _lib.conv_plan(1, 32, 32, 64, 64, 3, up_add=True) is None                     # upsample-add on a 3x3 layer
    assert _lib.conv_plan(1, 32, 32, 32, 64, 1, up_add=True) is None                     # ... with 32-channel chunks
    assert _lib.conv_plan(1, 32, 32, 64, 32, 1, up_add=True) is None                     # ... with a 32-column N tile
    assert _lib.conv_plan(1, 32, 32, 64, 64, 1, out_f32=True, up_add=True) is None       # ... with fp32 output
    assert _lib.conv_plan(1, 32, 32, 32, 32, 3, tail=True) is None                       # tail on a 32-channel layer
    assert _lib.conv_plan(1, 32, 32, 64, 64, 3, out_f32=True, pool=True) is None         # fp32 output with a pool
    assert _lib.conv_plan(1, 32, 32, 3, 64, 3) is None                                   # 3 input channels: SIMT
    assert _lib.conv_plan(1, 32, 32, 64, 2, 1) is None                                   # 2 output channels: SIMT
    assert _lib.conv_plan(1, 32, 32, 64, 64, 3, engine=_lib.CONV_SIMT) is None           # not a tensor-core engine
    assert _lib.conv_plan(0, 32, 32, 64, 64, 3) is None                                  # empty batch


def test_compiled_instances():
    assert len(COMPILED) == 32
