"""conv_tc_kernel's ping-pong schedule: a tile's result may not depend on which consumer warpgroup runs it, nor on where
it sits in its CTA's sequence of tiles.

The kernel's grid is min(total tiles, SM count) persistent CTAs; CTA c runs tiles c, c + G, c + 2G, ... (G = the grid
size), and the CTA's j-th tile (its "position") goes to consumer warpgroup 1 for even j and to warpgroup 2 for odd j.
Every image here is 16 x 24 pixels and every layer has one n-tile, so an image is 3 tiles, consecutive in that order:
8 x 16 halo tiles, or the 8 x 16 x 1 generic box, which ``pick_box`` takes whenever the batch has an odd number of
images (every other box wastes pixels then).  The checked image is run alone, behind one or two leading images (odd and
even shifts), and inside batches larger than the GPU whose leading images put its tiles at CTA positions 0, 1 and 2:
warpgroup 1 on a CTA's first tile, warpgroup 2 on its second (after the first warpgroup's turn), and warpgroup 1
again on its third (after stepping over the other warpgroup's stages in the ring).  ``_positions`` computes those
positions from the device's SM count and the test asserts the layouts reach all three.  For every instantiated
(BLOCK_N, KCH, MODE, UPADD) combination -- the instance that ran is read from the profiler's kernel name -- and with a
fused pool, the fused CRAFT tail, fp32 output and channel slices, the image's outputs must be the same bits in every
layout and within the fp64 bound of tests/stage_refs.py.  A grid sweep then runs batches of 1, SM - 1, SM, SM + 1 and
2 SM + 1 one-tile images: grids smaller than the GPU, CTAs with one tile and with an odd or even number of tiles.
"""
import re

import numpy as np
import pytest
import torch

from keras_ocr_b200 import _lib
from tests import test_gpu_conv_epilogues as E

pytestmark = pytest.mark.gpu

H, W = 16, 24                    # 3 tiles (8 x 16) per image per n-tile
TILES_PER_IMAGE = 3
SMEM = 227 * 1024                # a CTA's shared memory


def _streamed_cin(bn, kch):
    """Smallest cin that keeps kch as the layer's K chunk and whose 3x3 filter bank alone exceeds shared memory, so B
    is streamed through the ring (MODE 1)."""
    cin = kch
    while not ((kch == 64 or cin % (2 * kch)) and 9 * cin * bn * 2 > SMEM):
        cin += kch
    return cin


def _inst(bn, kch, mode, upadd=False):
    return f"{bn},{kch},{mode},false,{'true' if upadd else 'false'}"


# (BLOCK_N, KCH) pairs conv_tc_run instantiates; cout = BLOCK_N gives one n-tile.  inst: the conv_tc_kernel template
# arguments (BLOCK_N, KCH, MODE, PAIR, UPADD) each engine must launch.
COMBOS = [(16, 64), (32, 64), (64, 64), (128, 64), (16, 32), (32, 32), (32, 16), (64, 16)]
CASES = []
for bn, kch in COMBOS:
    # resident bank (MODE 2) on the product route, generic tiles (MODE 0) on TC_GENERIC
    CASES.append(dict(E._case(f"bn{bn}_kch{kch}_resident", 1, H, W, kch, bn, engines=("auto", "tc_generic")),
                      inst={"auto": _inst(bn, kch, 2), "tc_generic": _inst(bn, kch, 0)}))
    # streamed bank (MODE 1)
    CASES.append(dict(E._case(f"bn{bn}_kch{kch}_streamed", 1, H, W, _streamed_cin(bn, kch), bn, engines=("auto",)),
                      inst={"auto": _inst(bn, kch, 1)}))
CASES += [
    dict(E._case("pool_resident", 1, H, W, 64, 64, pool=True, write_full=1, engines=("auto",)),
         inst={"auto": _inst(64, 64, 2)}),
    dict(E._case("pool_streamed_aff2", 1, H, W, 128, 128, aff2=True, pool=True, write_full=0, engines=("auto",)),
         inst={"auto": _inst(128, 64, 1)}),
    dict(E._case("tail", 1, H, W, 32, 16, tail=True, engines=("auto",)), inst={"auto": _inst(16, 32, 2)}),
    dict(E._case("f32_slice", 1, H, W, 64, 64, out=(4, 8), out_f32=True, aff2=True, engines=("auto", "tc_generic")),
         inst={"auto": _inst(64, 64, 2), "tc_generic": _inst(64, 64, 0)}),
    dict(E._case("slice_in_and_out", 1, H, W, 128, 128, x=(64, 0), out=(64, 64), engines=("auto", "tc_generic")),
         inst={"auto": _inst(128, 64, 1), "tc_generic": _inst(128, 64, 0)}),
    dict(E._case("upadd_64", 1, H, W, 128, 64, k=1, up=(0, 0), engines=("auto",)),
         inst={"auto": _inst(64, 64, 0, upadd=True)}),
    dict(E._case("upadd_128_slice", 1, H, W, 256, 128, k=1, x=(128, 0), up=(8, 16), engines=("auto",)),
         inst={"auto": _inst(128, 64, 0, upadd=True)}),
]


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _layouts(sm):
    """(leading, trailing) images around the checked one; each batch has an odd number of images."""
    k1 = -(-sm // TILES_PER_IMAGE)            # first image whose tiles start at or after tile sm: CTA position 1
    k2 = -(-2 * sm // TILES_PER_IMAGE)        # ... at or after tile 2 sm: CTA position 2
    t0 = k1 + (k1 % 2)                        # trailing images that fill the GPU behind an image at position 0
    return [(0, 0), (1, 1), (2, 0), (0, t0), (k1, k1 % 2), (k2, k2 % 2)]


def _positions(lead, trail, sm):
    """CTA-sequence positions of the checked image's tiles in the batch (lead, trail)."""
    total = TILES_PER_IMAGE * (lead + 1 + trail)
    grid = min(total, sm)
    return {t // grid for t in range(TILES_PER_IMAGE * lead, TILES_PER_IMAGE * (lead + 1))}


def test_layouts_reach_both_warpgroups_and_later_positions():
    """By construction (no device needed beyond the SM count): positions 0, 1 and 2 are all reached."""
    for sm in (1, 2, 7, 16, 78, 114, 132, 144):
        reached = set().union(*(_positions(lead, trail, sm) for lead, trail in _layouts(sm)))
        assert {0, 1, 2} <= reached or sm < 3, (sm, reached)
        assert all((lead + 1 + trail) % 2 == 1 for lead, trail in _layouts(sm))


@pytest.fixture(scope="module")
def ctx(cuda_device):
    c = _lib.Context(0)
    yield c
    c.close()


def _batch(case, d, first, n):
    """Images first .. first + n - 1 of the pool as a case of its own."""
    sub = dict(d, x=d["x"][first:first + n], up=None if d["up"] is None else d["up"][first:first + n])
    return dict(case, n=n), sub


def _image(slabs, key, index, off, c):
    return slabs[key].body()[index:index + 1, ..., off:off + c].contiguous().cpu().numpy()


def _instances(prof):
    found = set()
    for e in prof.key_averages():
        m = re.search(r"conv_tc_kernel<([^>]*)>", e.key)
        if m:
            found.add(m.group(1).replace(" ", ""))
    return found


_POOLS = {}


def _pool(case, n):
    if case["name"] not in _POOLS:
        _POOLS.clear()                                       # one case's images at a time
        _POOLS[case["name"]] = E._inputs(dict(case, n=n))
    return _POOLS[case["name"]]


@pytest.mark.parametrize("engine", ["auto", "tc_generic"])
@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_tile_position_does_not_matter(ctx, case, engine):
    """The checked image's outputs: the expected kernel instance, within the fp64 bound, and the same bits at CTA
    positions 0, 1 and 2 (both warpgroups) and behind odd and even shifts."""
    if engine not in case["engines"]:
        pytest.skip(f"{case['name']} is not run by the {engine} engine")
    from torch.profiler import ProfilerActivity, profile

    sm = _sm_count()
    layouts = _layouts(sm)
    assert {0, 1, 2} <= set().union(*(_positions(lead, trail, sm) for lead, trail in layouts))
    target = max(lead for lead, _ in layouts)                # the checked image's index in the pool
    d = _pool(case, target + 1 + max(trail for _, trail in layouts))
    ref = E._reference(dict(case, name=f"{case['name']}@{target}"), _batch(case, d, target, 1)[1])
    cout, oo = case["cout"], case["out"][0]
    tag = f"{case['name']}[{engine}]"
    first = None
    for lead, trail in layouts:
        c, sub = _batch(case, d, target - lead, lead + 1 + trail)
        if first is None:
            with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
                s = E._run(ctx, c, sub, E.ENGINES[engine])
            assert _instances(prof) == {case["inst"][engine]}, (tag, _instances(prof))
        else:
            s = E._run(ctx, c, sub, E.ENGINES[engine])
        got = {}
        if E._out_is_written(case, engine):
            got["out"] = _image(s, "out", lead, oo, cout)
        if case["pool"]:
            got["pool"] = _image(s, "pool", lead, case["pool_view"][0], cout)
        if case["tail"]:
            got["scores"] = _image(s, "scores", lead, 0, 2)
        if first is None:
            first = got
            for key, v in got.items():
                E._check_values(f"{tag} {key}", v.astype(np.float64), ref[key])
            continue
        for key, v in got.items():
            assert np.array_equal(first[key].view(np.uint8), v.view(np.uint8)), \
                (tag, key, f"{lead} leading, {trail} trailing images: CTA positions {_positions(lead, trail, sm)}")


SWEEP = [E._case("sweep_resident", 1, 16, 8, 64, 128), E._case("sweep_streamed", 1, 16, 8, 128, 128)]


@pytest.mark.parametrize("engine", ["auto", "tc_generic"])
@pytest.mark.parametrize("case", SWEEP, ids=[c["name"] for c in SWEEP])
def test_grid_sizes(ctx, case, engine):
    """One-tile images: the last one's output is the same bits in batches of 1, SM - 1, SM, SM + 1 and 2 SM + 1."""
    sm = _sm_count()
    sizes = [1, sm - 1, sm, sm + 1, 2 * sm + 1]
    d = E._inputs(dict(case, n=sizes[-1]))
    ref = E._reference(dict(case, name=case["name"] + "_last", n=1), dict(d, x=d["x"][-1:]))
    first = None
    for k in sizes:
        c, sub = _batch(dict(case, n=sizes[-1]), d, sizes[-1] - k, k)
        got = _image(E._run(ctx, c, sub, E.ENGINES[engine]), "out", k - 1, case["out"][0], case["cout"])
        if first is None:
            first = got
            E._check_values(f"{case['name']}[{engine}]", got.astype(np.float64), ref["out"])
        assert np.array_equal(first.view(np.uint8), got.view(np.uint8)), (case["name"], engine, k)
