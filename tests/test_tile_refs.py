"""The tile grid of ``b2o_tile_plan`` (through ``_lib.tile_plan``) against its statement in tests/tile_refs.py and the
properties DESIGN.md section 1 ("Tiles") promises; the NumPy cut and stitch; ``detection.check_tiles`` and the default
rule.  CPU only."""
import itertools

import numpy as np
import pytest

from keras_ocr_b200 import _lib, detection
from tests import tile_refs as TR

LENGTHS = [32, 33, 100, 511, 512, 513, 767, 768, 1024, 1675, 2047, 2048, 2049, 2080, 2304, 3072, 4095, 4096, 6144, 8192]
TILES = [512, 640, 1024, 2048]
MARGINS = [0, 64, 128]


def _plan(hp, wp, t, m):
    p = _lib.tile_plan(hp, wp, t, m)
    return None if p is None else {f: getattr(p, f) for f, _ in _lib.TilePlan._fields_}


@pytest.mark.parametrize("tile_size,margin", [(t, m) for t in TILES for m in MARGINS] + [(2048, 256), (1024, 256)])
def test_plan_matches_statement_and_properties(tile_size, margin):
    for hp, wp in itertools.product(LENGTHS, LENGTHS[::3]):
        got = _plan(hp, wp, tile_size, margin)
        assert got == TR.plan(hp, wp, tile_size, margin), (hp, wp)
        for length, t, s, k in ((hp, got["t_h"], got["s_h"], got["n_h"]), (wp, got["t_w"], got["s_w"], got["n_w"])):
            assert t == min(tile_size, length) and s == t - 2 * margin
            if length <= tile_size:
                assert k == 1                                   # a page that fits is one tile
            else:
                assert (k - 1) * s + t >= length > (k - 2) * s + t   # the fewest tiles that cover it
            origins = [i * s for i in range(k)]
            assert all(o % 32 == 0 for o in origins)            # the VGG pooling grids of every tile align with the page's
            core = TR.cores(length, t, s, k, margin)
            covered = np.zeros(length, np.int32)
            for (lo, hi), o in zip(core, origins):
                assert o <= lo < hi <= min(o + t, length)
                covered[lo:hi] += 1
                # every core pixel is margin px from its tile's edge, except at the page's edge
                assert lo == 0 or lo - o >= margin
                assert hi == length or o + t - hi >= margin
            assert (covered == 1).all()                         # the cores partition [0, length)
            half = np.zeros(length // 2, np.int32)
            for lo, hi in TR.score_cores(length, t, s, k, margin):
                half[lo:hi] += 1
            assert (half == 1).all()                            # and so do their score-map halves


@pytest.mark.parametrize("args", [(31, 512, 512, 0), (512, 31, 512, 0), (512, 512, 500, 0), (512, 512, 2080, 0),
                                  (512, 512, 0, 0), (512, 512, 512, 136), (512, 512, 512, 8), (512, 512, 512, -16),
                                  (512, 512, 256, 128)])
def test_plan_rejects(args):
    assert _lib.tile_plan(*args) is None
    assert TR.plan(*args) is None


def test_tile_counts():
    assert _plan(3072, 3072, 2048, 128)["n_h"] == 2                  # 2048 + 1792 >= 3072
    assert _plan(6144, 6144, 2048, 128)["n_w"] == 4                  # 2048 + 3 * 1792 >= 6144 > 2048 + 2 * 1792
    assert _plan(2048, 2048, 2048, 128)["n_h"] == 1
    p = _plan(1536, 3000, 512, 128)
    assert (p["n_h"], p["n_w"]) == (5, 11) and (p["t_h"], p["t_w"]) == (512, 512)
    p = _plan(2304, 1675, 2048, 128)
    assert (p["n_h"], p["n_w"], p["t_w"]) == (2, 1, 1675)


def test_numpy_cut_and_stitch_round_trip():
    rng = np.random.default_rng(0)
    n, hp, wp = 2, 1100, 700
    p = TR.plan(hp, wp, 512, 128)
    img = rng.integers(0, 255, (n, hp, wp, 3), dtype=np.uint8)
    tiles = TR.cut(img, p)
    assert tiles.shape == (n * p["n_h"] * p["n_w"], 512, 512, 3)
    assert (tiles[-1, :, wp - (p["n_w"] - 1) * p["s_w"]:] == 255).all()   # the overhang past the page
    # a "score" that is each tile's own pixel, halved: the stitch then rebuilds the page's halved pixels exactly
    ts = tiles[:, ::2, ::2, :2].astype(np.float32)
    whole = TR.stitch(ts, p, n)
    assert np.array_equal(whole, img[:, ::2, ::2, :2].astype(np.float32)[:, :hp // 2, :wp // 2])
    # chunked: the same map
    out = None
    for first in range(0, ts.shape[0], 3):
        out = TR.stitch(ts[first:first + 3], p, n, first=first, out=out)
    assert np.array_equal(out, whole)


@pytest.mark.parametrize("bad", [True, False, 512.0, "512", 500, 0, -512, 4 * detection.TILE_MARGIN - 32, 2080, 4096])
def test_check_tiles_rejects(bad):
    with pytest.raises(ValueError):
        detection.check_tiles(bad)


def test_check_tiles_and_default_rule():
    assert detection.check_tiles() is None and detection.check_tiles(None) is None
    assert detection.check_tiles(np.int64(1024)) == 1024 and detection.check_tiles(2048) == 2048
    rule = detection.tile_size_for
    assert rule(2048, 8192) is None                    # wide but not tall: the whole-page forward, as before
    assert rule(2049, 100) == 2048 and rule(6144, 6144) == 2048
    assert rule(768, 768, 512) == 512 and rule(512, 512, 512) is None and rule(512, 513, 512) == 512
