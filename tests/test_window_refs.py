"""CPU: the wide-word reference (tests/window_refs.py) on hand cases with written-out answers, and its window crops
bit for bit against cv2.getPerspectiveTransform + cv2.warpPerspective."""
import cv2
import numpy as np
import pytest

from tests import image_refs as I
from tests import window_refs as R

BLANK, C = 36, 37


def axis(x0, y0, x1, y1):
    return np.array([[x0, y0], [x1, y0], [x1, y1], [x0, y1]], np.float32)


def below(v):
    return float(np.nextafter(np.float32(v), np.float32(-np.inf)))


def above(v):
    return float(np.nextafter(np.float32(v), np.float32(np.inf)))


def window_cases(seed=0, n=60, H=180, W=900):
    """Wide and narrow rotated rectangles, corners in any cyclic order, on a random page."""
    rng = np.random.default_rng(seed)
    quads = [I._rect(rng.uniform(0, W), rng.uniform(0, H), rng.uniform(100, 1600), rng.uniform(6, 45),
                     rng.uniform(-90, 90), int(rng.integers(4)), bool(rng.integers(2))) for _ in range(n)]
    quads += [axis(3, 3, 203, 34), axis(3, 3, 613, 34), axis(-40, 20, 1400, 44), axis(10, 10, 11, 12)]
    return rng.integers(0, 256, (H, W), dtype=np.uint8), np.stack(quads).astype(np.float32)


# ----------------------------------------------------------------------------------------------- count and plans
@pytest.mark.parametrize("quad, k", [
    (axis(10, 0, 210, 31), 1),                      # w 31 = 200 h exactly: wc = 200 fits
    (axis(10, 0, below(210), 31), 1),               # one ulp narrower: w = 199
    (axis(10, 0, above(210), 31), 1),               # one ulp wider: w stays 200
    (axis(10, 0, 210, below(31)), 2),               # one ulp lower: h = 30, wc = 206.67
    (axis(10, 0, 211, 31), 2),                      # w = 201
    (axis(0, 0, 400, 31), 3),                       # wc = 400: starts 0, 136, 200
    (axis(0, 0, 550, 31), 4),                       # starts 0, 136, 272, 350
    (axis(0, 0, 608, 31), 4),                       # wc = T = 608: K = M
    (axis(0, 0, 1000, 31), 4),                      # past the cap: scale 0.608 shrinks the word, K stays M
    (axis(0, 0, 0, 31), 1),                         # w = 0: warpBox raises, read as today
])
def test_window_count(quad, k):
    assert R.extent(quad, 4)[3] == k
    assert R.extent(quad, 1)[3] == 1


def test_starts_and_shrink_past_the_cap():
    _, wc, sh, k, _ = R.extent(axis(0, 0, 550, 31), 4)
    assert (wc, sh, k) == (550.0, 31.0, 4)
    assert R.starts(k, wc).tolist() == [0.0, 136.0, 272.0, 350.0]
    _, wc, sh, k, _ = R.extent(axis(0, 0, 1000, 31), 4)
    assert k == 4 and abs(wc - 608) < 1e-9 and abs(sh - 18.848) < 1e-9
    p = R.plan(axis(0, 0, 1000, 31), 4, 3)
    assert p["dw"] == 200 and p["dh"] == 18 and abs(p["a"] - 408) < 1e-9


def test_windows_tile_the_word_with_overlaps_of_64():
    _, quads = window_cases()
    wide = 0
    for q in quads:
        for m in (2, 4, 16):
            _, wc, _, k, ok = R.extent(q, m)
            if not ok or k == 1:
                continue
            wide += 1
            a = R.starts(k, wc)
            assert a[0] == 0 and a[-1] + 200 == wc and k <= m
            assert np.all(np.diff(a) > 0) and np.all(np.diff(a) <= 136 + 1e-9)    # every overlap >= 64
    assert wide > 50


def test_a_word_that_fits_has_warpbox_plan():
    _, quads = window_cases()
    for q in quads:
        for m in (1, 4):
            p = R.plan(q, m, 0)
            if R.extent(q, m)[3] != 1 or not p["valid"]:
                continue
            m_ref, dw, dh = I.warp_plan(q)
            assert p["m"].tobytes() == m_ref.tobytes() and (p["dw"], p["dh"]) == (dw, dh)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_window_crops_equal_cv2(seed):
    """Every window crop, gray and colour, equals cv2.getPerspectiveTransform + cv2.warpPerspective of step 3.  The
    crops follow the fp64 LU model of getPerspectiveTransform the kernels use (tests/cvmodels.py), whose matrix can
    differ from cv2's own solve in the last bits (as it does for plain warpBox boxes): such a crop may differ from cv2's
    in a sample whose 1/32-pixel coordinate rounds the other way -- one sample in 5 million on seed 0, none on 1 and 2."""
    from tests import cvmodels as M

    img, quads = window_cases(seed)
    rgb = np.stack([img, img[::-1], 255 - img], -1)
    compared = off = 0
    for q in quads:
        box, wc, sh, k, ok = R.extent(q, 4)
        if not ok or k == 1:
            continue
        for j, a in enumerate(R.starts(k, wc)):
            dst = np.array([[0.0 - a, 0], [wc - a, 0], [wc - a, sh], [0.0 - a, sh]]).astype(np.float32)
            mat = cv2.getPerspectiveTransform(src=box, dst=dst)
            for src in (img, rgb):
                want = np.zeros((31, 200) + src.shape[2:], np.uint8)
                want[:min(31, int(sh))] = cv2.warpPerspective(src, mat, dsize=(200, int(sh)))[:31]
                got = R.crop(src, q, 4, j)
                if not np.array_equal(got, want):
                    assert not np.array_equal(mat, M.get_persp(box, dst)), (q.tolist(), j)
                    off += int((got != want).sum())
                compared += 1
    assert compared > 400 and off <= 1


# ----------------------------------------------------------------------------------------------- step positions
def test_positions_without_stn():
    assert R.positions(0.0).tolist() == [4.0 * (t + 2) + 1.5 for t in range(48)]   # 9.5 .. 197.5
    assert R.positions(136.0)[0] == 145.5


def test_positions_identity_and_shifted_theta():
    ident = np.array([1, 0, 0, 0, 1, 0], np.float32)
    p = R.positions(0.0, ident)
    assert p[0] == 4.0 * ((0.5 * ((-1.0 + 4.0 / 49.0) + 1.0)) * 50.0) + 1.5     # u = 50 r / 49 at r = 2
    assert p[-1] == 200.0                                                       # u = 50, x = 201.5, clamped
    shifted = R.positions(0.0, np.array([1, 0, 0, 0, 1, 0.1], np.float32))
    assert np.allclose((shifted - p)[:40], 4 * 0.5 * np.float64(np.float32(0.1)) * 50)
    flipped = R.positions(10.0, np.array([1, 0, 0, 0, -1, 0], np.float32))   # time runs backwards: held flat
    assert np.all(flipped == flipped[0]) and abs(flipped[0] - (10 + 4 * (50 - 100 / 49) + 1.5)) < 1e-12


# ----------------------------------------------------------------------------------------------- the stitch
def emitting(steps_to_class):
    """(48, 37) logits: blank everywhere except {step: class}."""
    lg = np.zeros((48, C), np.float32)
    lg[:, BLANK] = 5.0
    for t, c in steps_to_class.items():
        lg[t, c], lg[t, BLANK] = 5.0, 0.0
        lg[t, c] = 6.0
    return lg


def test_a_character_at_the_overlap_is_read_once():
    # windows at 0 and 136: window 0's step t lies at 4t + 9.5, window 1's at 145.5 + 4t; overlap [136, 200], mid 168
    a = np.array([0.0, 136.0])
    # 'x' (23) at 169.5, just past mid: window 0 step 40, window 1 step 6
    row, _, kept, cuts = R.stitch([emitting({40: 23}), emitting({6: 23})], None, a, 2)
    assert cuts == [165.5]                          # step 6 (169.5) emits; step 5 (165.5) and window 0's 39 are blank
    assert row[:2].tolist() == [23, -1]
    assert (1, 6) in kept and (0, 40) not in kept
    # 'x' at 161.5, just before mid: window 0 step 38, window 1 step 4
    row, _, kept, cuts = R.stitch([emitting({38: 23}), emitting({4: 23})], None, a, 2)
    assert cuts == [169.5] and row[:2].tolist() == [23, -1] and (0, 38) in kept and (1, 4) not in kept
    # one character on each side of mid, each read once, in order
    row, _, _, _ = R.stitch([emitting({2: 0, 37: 1, 42: 2}), emitting({3: 1, 8: 2, 20: 3})], None, a, 2)
    assert row[:5].tolist() == [0, 1, 2, 3, -1]


def test_no_blank_pair_cuts_at_mid():
    a = np.array([0.0, 136.0])
    busy = emitting({t: 25 for t in range(48)})     # window 1 never emits a blank
    row, _, kept, cuts = R.stitch([emitting({}), busy], None, a, 2)
    assert cuts == [168.0]
    assert [t for k, t in kept if k == 0] == list(range(40))     # 4t + 9.5 < 168
    assert [t for k, t in kept if k == 1] == list(range(6, 48))  # 145.5 + 4t >= 168
    assert row[:2].tolist() == [25, -1]


def test_kept_steps_cover_every_position_once():
    rng = np.random.default_rng(3)
    for _ in range(20):
        k = int(rng.integers(2, 6))
        wc = 200 + (k - 1) * 136 - rng.uniform(0, 135)
        a = R.starts(k, wc)
        lg = rng.normal(size=(k, 48, C)).astype(np.float32)
        lg[..., BLANK] += 1.0
        th = np.tile(np.array([1, 0, 0, 0, 1, 0], np.float32), (k, 1))
        th[:, 5] = rng.uniform(-0.05, 0.05, k)
        row, s, kept, cuts = R.stitch(lg, th, a, k)
        pos = np.concatenate([R.positions(a[j], th[j]) for j in range(k)])
        got = [pos[j * 48 + t] for j, t in kept]
        assert np.all(np.diff(got) >= 0)                          # in order along the word
        assert all(cuts[j] >= a[j + 1] and cuts[j] <= a[j] + 200 for j in range(k - 1))
        assert np.isfinite(s) and row.shape == (48 * k,)


def test_one_window_is_plain_greedy():
    rng = np.random.default_rng(5)
    lg = rng.normal(size=(48, C)).astype(np.float32)
    row, s, kept, _ = R.stitch(lg[None], None, np.zeros(1), 4)
    labels, s_ref = R.greedy(lg)
    assert row[:len(labels)].tolist() == labels and np.all(row[len(labels):] == -1)
    assert s == s_ref and len(kept) == 48


def test_a_cut_never_falls_below_the_previous_one():
    # three windows, the last just past the second: a = 0, 136, 137, steps at 9.5 + 4t, 145.5 + 4t and 146.5 + 4t
    a = np.array([0.0, 136.0, 137.0])
    w0 = emitting({})
    w1 = emitting({t: 25 for t in range(10, 48)})   # blank only at steps 0..9 (145.5 .. 181.5)
    w2 = emitting({t: 25 for t in range(2, 48)})    # blank only at steps 0, 1 (146.5, 150.5)
    _, _, kept, cuts = R.stitch([w0, w1, w2], None, a, 3)
    # cut 0: window 1's 169.5 is nearest mid 168 and blank in both.  Cut 1 (overlap [137, 336], mid 236.5): the only
    # blank pair is at 150.5, below cut 0, so it is raised to 169.5 and window 1 keeps nothing
    assert cuts == [169.5, 169.5]
    assert [k for k, _ in kept if k == 1] == []
    pos = [R.positions(a[k])[t] for k, t in kept]
    assert np.all(np.diff(pos) > 0)                 # in order along the word, no position kept twice
