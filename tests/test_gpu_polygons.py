"""Polygons for curved words on the GPU: b2o_get_boxes_poly, b2o_compact_polys and b2o_warp_polys against the CPU
references of tests/polygon_refs.py, their memory contracts, and the pipeline with return_polygons=True on straight
bench pages and on rendered curved pages."""
import cv2
import numpy as np
import pytest
import torch

from keras_ocr_b200 import _lib, recognition, weights as W
from oracle import synth
from tests import box_refs, image_refs, polygon_refs as P

pytestmark = pytest.mark.gpu

THR = (box_refs.DET, box_refs.TEXT, box_refs.LINK, 10)
DEV = torch.device("cuda", 0)


@pytest.fixture(scope="module")
def ctx(cuda_device):
    c = _lib.Context(0)
    yield c
    c.close()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def run_poly(ctx, scores, max_boxes=256, scored=True):
    n, hs, ws, _ = scores.shape
    t = torch.from_numpy(np.ascontiguousarray(scores)).to(DEV)
    nbytes = ctx.boxes_workspace_bytes(n, hs, ws, max_boxes)
    wsp = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    boxes = torch.full((n, max_boxes, 4, 2), float("nan"), device=DEV)
    counts = torch.full((n,), -7, dtype=torch.int32, device=DEV)
    bsc = torch.full((n, max_boxes), float("nan"), device=DEV) if scored else None
    polys = torch.full((n, max_boxes, P.POLY_POINTS, 2), -5.0, device=DEV)
    points = torch.full((n, max_boxes), -3, dtype=torch.int32, device=DEV)
    ctx.get_boxes_poly(t.data_ptr(), n, hs, ws, *THR, boxes.data_ptr(), counts.data_ptr(),
                       bsc.data_ptr() if scored else None, polys.data_ptr(), points.data_ptr(), max_boxes,
                       wsp.data_ptr(), nbytes, _stream())
    torch.cuda.synchronize()
    return dict(boxes=boxes.cpu().numpy(), counts=counts.cpu().numpy(), scores=bsc.cpu().numpy() if scored else None,
                polys=polys.cpu().numpy(), points=points.cpu().numpy())


def run_plain(ctx, scores, max_boxes=256):
    n, hs, ws, _ = scores.shape
    t = torch.from_numpy(np.ascontiguousarray(scores)).to(DEV)
    nbytes = ctx.boxes_workspace_bytes(n, hs, ws, max_boxes)
    wsp = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    boxes = torch.full((n, max_boxes, 4, 2), float("nan"), device=DEV)
    counts = torch.full((n,), -7, dtype=torch.int32, device=DEV)
    bsc = torch.full((n, max_boxes), float("nan"), device=DEV)
    labels = torch.full((n, hs, ws), -9, dtype=torch.int32, device=DEV)
    comps = torch.full((n, max_boxes, 7), -9, dtype=torch.int32, device=DEV)
    ctx.get_boxes_test(t.data_ptr(), n, hs, ws, *THR, boxes.data_ptr(), counts.data_ptr(), bsc.data_ptr(), max_boxes,
                       wsp.data_ptr(), nbytes, labels.data_ptr(), comps.data_ptr(), _stream())
    torch.cuda.synchronize()
    return dict(boxes=boxes.cpu().numpy(), counts=counts.cpu().numpy(), scores=bsc.cpu().numpy(),
                labels=labels.cpu().numpy(), comps=comps.cpu().numpy())


def _same(a, b):
    """Bit for bit, except that any NaN equals any NaN (unused polygon points)."""
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype.kind == "f":
        assert a.shape == b.shape and (np.isnan(a) == np.isnan(b)).all()
        a, b = np.where(np.isnan(a), 0, a).astype(a.dtype), np.where(np.isnan(b), 0, b).astype(b.dtype)
    np.testing.assert_array_equal(a.view(np.uint8), b.view(np.uint8))


# ------------------------------------------------------------------------------------------------ 1. boxes unchanged
@pytest.mark.parametrize("name, scores, max_boxes", box_refs.cases(), ids=[c[0] for c in box_refs.cases()])
def test_boxes_are_those_of_get_boxes(ctx, name, scores, max_boxes):
    got, ref = run_poly(ctx, scores, max_boxes), run_plain(ctx, scores, max_boxes)
    _same(got["counts"], ref["counts"])
    _same(got["boxes"], ref["boxes"])
    _same(got["scores"], ref["scores"])
    plain = run_poly(ctx, scores, max_boxes, scored=False)
    _same(plain["boxes"], ref["boxes"])
    _same(plain["polys"], got["polys"])


@pytest.mark.parametrize("seed", [0, 1])
def test_boxes_unchanged_on_seeded_score_maps(ctx, seed):
    scores = synth.score_maps(seed, 4, 256, 320, 24)
    got, ref = run_poly(ctx, scores), run_plain(ctx, scores)
    _same(got["counts"], ref["counts"])
    _same(got["boxes"], ref["boxes"])
    _same(got["scores"], ref["scores"])


# ------------------------------------------------------------------------------------------------ 2. polygons exact
def _paint(h, w, masks):
    s = np.zeros((h, w, 2), np.float32)
    rng = np.random.default_rng(7)
    for m in masks:
        s[..., 0][m > 0] = rng.uniform(0.75, 0.99, int((m > 0).sum())).astype(np.float32)
    return s


def _place(canvas, m, y, x):
    h, w = m.shape
    y0, x0 = max(y, 0), max(x, 0)
    y1, x1 = min(y + h, canvas.shape[0]), min(x + w, canvas.shape[1])
    out = np.zeros(canvas.shape, np.uint8)
    out[y0:y1, x0:x1] = m[y0 - y:y1 - y, x0 - x:x1 - x]
    return out


def polygon_maps():
    """(name, scores (h,w,2)): arcs, S-curves, straight, short, gapped and border-touching components."""
    H, W = 260, 420
    cases = []
    arcs = [P.arc_band(s, radius=r, thickness=t, rotate_deg=a)[0] for s, r, t, a in
            [(60, 70, 9, 0), (120, 60, 8, 20), (180, 50, 10, -15), (90, 90, 12, 40)]]
    cases.append(("arcs", _paint(H, W, [_place(np.zeros((H, W)), arcs[0], 0, 0), _place(np.zeros((H, W)), arcs[1], 0, 200),
                                         _place(np.zeros((H, W)), arcs[3], 100, 150)])))
    cases.append(("arc180", _paint(H, W, [_place(np.zeros((H, W)), arcs[2], 40, 100)])))
    sines = [P.sine_band(a, length=l)[0] for a, l in [(8, 140), (12, 180)]]
    cases.append(("s_curves", _paint(H, W, [_place(np.zeros((H, W)), sines[0], 10, 10),
                                             _place(np.zeros((H, W)), sines[1], 130, 200)])))
    cases.append(("straight", _paint(H, W, [_place(np.zeros((H, W)), P.straight_band(a, 70, 9), 20 + 110 * (k // 3),
                                                   10 + 130 * (k % 3)) for k, a in enumerate([0, 15, 30, 60, 100, 165])])))
    short = [P.straight_band(20, 14, 9), P.arc_band(90, radius=12, thickness=6)[0], P.straight_band(0, 30, 12)]
    cases.append(("short", _paint(H, W, [_place(np.zeros((H, W)), m, 30 + 70 * k, 40 + 90 * k) for k, m in enumerate(short)])))
    # one component whose segmap has a gap: text & link pixels across the arc leave the segmap (detection.py:246), and
    # the dilation closes the gap again
    gapped = _paint(H, W, [_place(np.zeros((H, W)), P.arc_band(120, radius=70, thickness=9)[0], 20, 60)])
    mid = 60 + P.arc_band(120, radius=70, thickness=9)[0].shape[1] // 2
    gapped[:, mid - 1:mid + 1, 1] = np.where(gapped[:, mid - 1:mid + 1, 0] > 0, 0.9, 0)
    cases.append(("gapped", gapped))
    border = [_place(np.zeros((H, W)), arcs[1], -30, -20), _place(np.zeros((H, W)), arcs[0], H - 70, W - 150),
              _place(np.zeros((H, W)), sines[1], 100, -60)]
    cases.append(("border", _paint(H, W, border)))
    return cases


POLY_CASES = polygon_maps()


def _check_polys(out, scores, labels, comps, i):
    c = int(out["counts"][i])
    blobs = P.component_blobs(scores, labels, comps, c)
    for k in range(c):
        want, npts = P.polygon(blobs[k], out["boxes"][i, k] / 2)
        assert int(out["points"][i, k]) == npts, (i, k)
        _same(out["polys"][i, k], want)


@pytest.mark.parametrize("name, scores", POLY_CASES, ids=[c[0] for c in POLY_CASES])
def test_polygons_equal_the_reference(ctx, name, scores):
    ref = run_plain(ctx, scores[None])
    alone = run_poly(ctx, scores[None])
    _check_polys(alone, scores, ref["labels"][0], ref["comps"][0], 0)
    if name in ("arcs", "arc180", "s_curves"):
        assert (alone["points"][0, :alone["counts"][0]] > 4).any()
    if name == "straight":
        assert (alone["points"][0, :alone["counts"][0]] == 4).all()
    others = [s for n, s in POLY_CASES if n != name]
    batch = np.stack(others[:3] + [scores] + others[3:7])[:8]
    at = 3
    got = run_poly(ctx, batch)
    again = run_poly(ctx, batch)
    for key in ("polys", "points", "boxes"):
        _same(got[key], again[key])
    c = int(alone["counts"][0])
    _same(got["polys"][at, :c], alone["polys"][0, :c])
    _same(got["points"][at, :c], alone["points"][0, :c])


# ------------------------------------------------------------------------------------------------ 3. warp exact
def _seeded_polys(rng, H, W):
    out = []
    for k in range(23):
        s = int(rng.integers(2, P.S_MAX + 1))
        cx, cy = rng.uniform(-20, W + 20), rng.uniform(-20, H + 20)
        length, thick = rng.uniform(20, 600 if k % 5 == 0 else 160), rng.uniform(4, 60 if k % 7 == 0 else 25)
        bend, ang = rng.uniform(-1.5, 1.5), rng.uniform(-np.pi, np.pi)
        tt = np.linspace(-0.5, 0.5, s + 1)
        a = ang + bend * tt
        centre = np.stack([cx + length * np.cumsum(np.cos(a)) / (s + 1), cy + length * np.cumsum(np.sin(a)) / (s + 1)], -1)
        normal = np.stack([-np.sin(a), np.cos(a)], -1) * thick / 2
        top, bot = centre - normal, centre + normal
        out.append(np.concatenate([top, bot[::-1]]).astype(np.float32))
    return out


def _warp_dev(ctx, img, channels, polys, points, idx):
    b = len(points)
    img_t = torch.from_numpy(np.ascontiguousarray(img)).to(DEV)
    n, h, w = img.shape[:3]
    tail = (3,) if channels == 3 else ()
    crops = torch.full((b, 31, 200) + tail, 77, dtype=torch.uint8, device=DEV)
    x = torch.empty((b, 200, 31) + tail, dtype=torch.float16, device=DEV)
    pol, pts, ix = (torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in (polys, points, idx))
    ctx.warp_polys(img_t.data_ptr(), channels, n, h, w, pol.data_ptr(), pts.data_ptr(), ix.data_ptr(), b,
                   crops.data_ptr(), x.data_ptr(), _stream())
    torch.cuda.synchronize()
    return crops.cpu().numpy(), x.cpu().numpy()


@pytest.mark.parametrize("channels", [1, 3])
def test_warp_polys_equals_the_piecewise_reference(ctx, channels):
    rng = np.random.default_rng(11)
    n, H, W = 3, 157, 211
    img = rng.integers(0, 256, (n, H, W) + ((3,) if channels == 3 else ()), dtype=np.uint8)
    entries = _seeded_polys(rng, H, W)
    polys = np.full((len(entries), P.POLY_POINTS, 2), np.nan, np.float32)
    points = np.array([len(e) for e in entries], np.int32)
    for k, e in enumerate(entries):
        polys[k, :len(e)] = e
    idx = rng.integers(0, n, len(entries)).astype(np.int32)
    crops, x = _warp_dev(ctx, img, channels, polys, points, idx)
    differ = 0
    for k in range(len(entries)):
        want = P.warp_poly(img[idx[k]], polys[k], int(points[k]), model=True)
        np.testing.assert_array_equal(crops[k], want, err_msg=f"entry {k}")
        # real cv2 per segment: its warpPerspective rounds a few pixels of a non-affine segment differently from the
        # pinned model (measured: 1 pixel in 1 of 23 gray crops, 6 pixels in 2 of 23 colour crops, by up to 6 levels)
        cv = P.warp_poly(img[idx[k]], polys[k], int(points[k]))
        diff = crops[k] != cv
        assert diff.sum() <= 3 * channels and np.abs(crops[k].astype(int) - cv).max() <= 8, k
        differ += int(diff.any())
    assert differ <= 2
    np.testing.assert_array_equal(x, image_refs.crops_to_input(crops))
    lay = [P.warp_layout(polys[k], int(points[k])) for k in range(len(entries))]
    assert any(l is not None and l[1] == 200 for l in lay) and any(l is not None and l[2] == 31 for l in lay)


@pytest.mark.parametrize("channels", [1, 3])
def test_four_point_entries_equal_warp_boxes(ctx, channels):
    g = image_refs.warp_cases()[0]
    img = g["rgb"] if channels == 3 else g["gray"]
    quads, idx = g["quads"], g["image_index"]
    polys = np.full((len(quads), P.POLY_POINTS, 2), np.nan, np.float32)
    polys[:, :4] = quads
    crops, x = _warp_dev(ctx, img, channels, polys, np.full(len(quads), 4, np.int32), idx)
    n, h, w = img.shape[:3]
    ref_c = torch.full(crops.shape, 77, dtype=torch.uint8, device=DEV)
    ref_x = torch.empty(x.shape, dtype=torch.float16, device=DEV)
    img_t, q_t, ix_t = (torch.from_numpy(np.ascontiguousarray(a)).to(DEV) for a in (img, quads, idx))
    ctx.warp_boxes(img_t.data_ptr(), n, h, w, q_t.data_ptr(), ix_t.data_ptr(), len(quads), ref_c.data_ptr(),
                   ref_x.data_ptr(), _stream(), color=channels == 3)
    torch.cuda.synchronize()
    _same(crops, ref_c.cpu().numpy())
    _same(x, ref_x.cpu().numpy())


# ------------------------------------------------------------------------------------------------ 4. memory contracts
GUARD = 4096


def _guarded(nbytes, fill):
    buf = torch.full((nbytes + 2 * GUARD,), fill, dtype=torch.uint8, device=DEV)
    return buf, buf[GUARD:GUARD + nbytes]


def _contract_get_boxes_poly(ctx, fill, wfill):
    scores = POLY_CASES[0][1][None].repeat(2, 0)
    n, hs, ws, _ = scores.shape
    m = 16
    sc = torch.from_numpy(scores).to(DEV)
    sc_before = sc.clone()
    nb = ctx.boxes_workspace_bytes(n, hs, ws, m)
    bufs = {k: _guarded(sz, fill) for k, sz in [("boxes", n * m * 32), ("counts", n * 4), ("scores", n * m * 4),
                                                 ("polys", n * m * P.POLY_POINTS * 8), ("points", n * m * 4)]}
    wbuf, wsp = _guarded(nb, wfill)
    p = {k: v[1].data_ptr() for k, v in bufs.items()}
    ctx.get_boxes_poly(sc.data_ptr(), n, hs, ws, *THR, p["boxes"], p["counts"], p["scores"], p["polys"], p["points"],
                       m, wsp.data_ptr(), nb, _stream())
    torch.cuda.synchronize()
    assert torch.equal(sc, sc_before)
    return {k: v[0].cpu().numpy() for k, v in bufs.items()}, wbuf.cpu().numpy()


def test_get_boxes_poly_memory_contract(ctx):
    runs = [_contract_get_boxes_poly(ctx, f, w) for f, w in ((0x00, 0xFF), (0xFF, 0x00))]
    counts = runs[0][0]["counts"][GUARD:GUARD + 8].view(np.int32)
    m, per = 16, {"boxes": 32, "scores": 4, "polys": P.POLY_POINTS * 8, "points": 4}
    for (out, wb), fill, wfill in zip(runs, (0x00, 0xFF), (0xFF, 0x00)):
        for k, buf in out.items():
            assert (buf[:GUARD] == fill).all() and (buf[-GUARD:] == fill).all(), k
        assert (wb[:GUARD] == wfill).all() and (wb[-GUARD:] == wfill).all()
        for k, size in per.items():                              # unwritten slots keep the prefill
            body = out[k][GUARD:-GUARD].reshape(2, m, size)
            for i in range(2):
                assert (body[i, min(int(counts[i]), m):] == fill).all(), k
    for k in runs[0][0]:                                         # written bytes do not depend on the prefill
        if k == "counts":
            assert (runs[0][0][k][GUARD:-GUARD] == runs[1][0][k][GUARD:-GUARD]).all()
            continue
        size = per[k]
        a, b = (r[0][k][GUARD:-GUARD].reshape(2, m, size) for r in runs)
        for i in range(2):
            c = min(int(counts[i]), m)
            assert (a[i, :c] == b[i, :c]).all(), k


def test_compact_polys_memory_contract(ctx):
    n, m = 3, 8
    rng = np.random.default_rng(3)
    polys = torch.from_numpy(rng.normal(size=(n, m, P.POLY_POINTS, 2)).astype(np.float32)).to(DEV)
    points = torch.from_numpy(rng.integers(4, 19, (n, m)).astype(np.int32)).to(DEV)
    counts = torch.tensor([3, 0, 11], dtype=torch.int32, device=DEV)                 # 11 > m: capped
    before = [t.clone() for t in (polys, points, counts)]
    outs = []
    for fill in (0x00, 0xFF):
        fp, fpv = _guarded(n * m * P.POLY_POINTS * 8, fill)
        pt, ptv = _guarded(n * m * 4, fill)
        ix, ixv = _guarded(n * m * 4, fill)
        ctx.compact_polys(polys.data_ptr(), points.data_ptr(), counts.data_ptr(), n, m, fpv.data_ptr(), ptv.data_ptr(),
                          ixv.data_ptr(), _stream())
        torch.cuda.synchronize()
        outs.append([b.cpu().numpy() for b in (fp, pt, ix)])
        for b in outs[-1]:
            assert (b[:GUARD] == fill).all() and (b[-GUARD:] == fill).all()
    total = 3 + 0 + 8
    for a, b, per in zip(outs[0], outs[1], (P.POLY_POINTS * 8, 4, 4)):
        assert (a[GUARD:GUARD + total * per] == b[GUARD:GUARD + total * per]).all()
        assert (a[GUARD + total * per:-GUARD] == 0x00).all() and (b[GUARD + total * per:-GUARD] == 0xFF).all()
    flat = outs[0][0][GUARD:GUARD + total * P.POLY_POINTS * 8].view(np.float32).reshape(total, P.POLY_POINTS, 2)
    src = polys.cpu().numpy()
    np.testing.assert_array_equal(flat, np.concatenate([src[0, :3], src[2, :8]]))
    np.testing.assert_array_equal(outs[0][2][GUARD:GUARD + total * 4].view(np.int32), [0] * 3 + [2] * 8)
    for t, b in zip((polys, points, counts), before):
        assert torch.equal(t, b)


def test_warp_polys_memory_contract(ctx):
    rng = np.random.default_rng(5)
    img = torch.from_numpy(rng.integers(0, 256, (2, 60, 90), dtype=np.uint8)).to(DEV)
    entries = _seeded_polys(rng, 60, 90)[:5]
    polys = np.full((5, P.POLY_POINTS, 2), np.nan, np.float32)
    for k, e in enumerate(entries):
        polys[k, :len(e)] = e
    pts = torch.tensor([len(e) for e in entries], dtype=torch.int32, device=DEV)
    pol, idx = torch.from_numpy(polys).to(DEV), torch.tensor([0, 1, 1, 0, 1], dtype=torch.int32, device=DEV)
    before = [t.clone() for t in (img, pol, pts, idx)]
    outs = []
    for fill in (0x00, 0xFF):
        cb, cv = _guarded(5 * 31 * 200, fill)
        xb, xv = _guarded(5 * 200 * 31 * 2, fill)
        ctx.warp_polys(img.data_ptr(), 1, 2, 60, 90, pol.data_ptr(), pts.data_ptr(), idx.data_ptr(), 5, cv.data_ptr(),
                       xv.data_ptr(), _stream())
        torch.cuda.synchronize()
        outs.append([cb.cpu().numpy(), xb.cpu().numpy()])
        for b in outs[-1]:
            assert (b[:GUARD] == fill).all() and (b[-GUARD:] == fill).all()
    for a, b in zip(*outs):                                  # every crop byte is written, whatever the prefill
        assert (a[GUARD:-GUARD] == b[GUARD:-GUARD]).all()
    for t, b in zip((img, pol, pts, idx), before):
        _same(t.cpu().numpy(), b.cpu().numpy())


def test_invalid_calls_launch_nothing(ctx):
    d = torch.empty(1 << 16, dtype=torch.uint8, device=DEV)
    p = d.data_ptr()
    n0 = ctx.launch_count()
    bad = [
        lambda: ctx.get_boxes_poly(p, 1, 8, 8, *THR, p, p, None, None, p, 4, p, 1 << 16, _stream()),    # polys NULL
        lambda: ctx.get_boxes_poly(p, 1, 8, 8, *THR, p, p, None, p, p, 4, p, 1, _stream()),             # workspace short
        lambda: ctx.compact_polys(p, p, p, 0, 4, p, p, p, _stream()),
        lambda: ctx.warp_polys(p, 2, 1, 8, 8, p, p, p, 1, p, None, _stream()),                          # channels 2
        lambda: ctx.warp_polys(p, 1, 1, 8, 8, p, p, p, 1, None, None, _stream()),                       # no output
    ]
    for call in bad:
        with pytest.raises(_lib.B2OError):
            call()
    ctx.warp_polys(p, 1, 1, 8, 8, p, p, p, 0, p, None, _stream())                                      # empty: no-op
    assert ctx.launch_count() == n0


# ------------------------------------------------------------------------------------------------ 5.-7. pipeline
@pytest.fixture(scope="module")
def pipe(cuda_device):
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    from keras_ocr_b200.recognition import Recognizer
    return Pipeline(detector=Detector(weights=W.synthetic_craft_weights(3, textlike=True), device=0),
                    recognizer=Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True), device=0), scale=2)


def test_straight_pages_keep_their_boxes(pipe):
    images, _ = synth.text_images(seed=1000, n=8, h=768, w=768, n_words=32)
    ref = pipe.recognize(images)
    got = pipe.recognize(images, return_polygons=True)
    assert [len(g) for g in got] == [len(r) for r in ref]
    for g, r in zip(got, ref):
        for (t, box, poly), (t0, box0) in zip(g, r):
            assert t == t0
            _same(box, box0)
            _same(poly, box)


def render_curved(rng, bend_deg, h=768, w=768, n_words=6):
    """Hershey words, each glyph rotated onto an arc that turns by ``bend_deg`` over the word; (page, words)."""
    page = np.full((h, w, 3), 255, np.uint8)
    words = []
    rows = 3
    for k in range(n_words):
        word = synth.random_word(rng, 4, 8)
        scale, thick = 1.6, 3
        widths = [cv2.getTextSize(ch, cv2.FONT_HERSHEY_SIMPLEX, scale, thick)[0][0] for ch in word]
        total = sum(widths) + 2 * len(word)
        th = cv2.getTextSize(word, cv2.FONT_HERSHEY_SIMPLEX, scale, thick)[0][1]
        sweep = np.radians(bend_deg)
        radius = total / max(sweep, 1e-6)
        cx = (k % 2 + 0.5) * w / 2 + rng.uniform(-20, 20)
        cy = (k // 2 + 0.5) * h / rows + rng.uniform(-10, 10)
        colour = tuple(int(c) for c in rng.integers(0, 90, 3))
        s = -total / 2
        for ch, cw in zip(word, widths):
            theta = (s + cw / 2) / radius if bend_deg else 0.0
            px = cx + (radius * np.sin(theta) if bend_deg else s + cw / 2)
            py = cy + (radius * (1 - np.cos(theta)) if bend_deg else 0.0) - (radius * (1 - np.cos(sweep / 2)) / 2 if bend_deg else 0)
            tile = np.full((2 * th + 20, cw + 20, 3), 255, np.uint8)
            cv2.putText(tile, ch, (10, th + 10), cv2.FONT_HERSHEY_SIMPLEX, scale, colour, thick, cv2.LINE_AA)
            rot = cv2.getRotationMatrix2D((tile.shape[1] / 2, th / 2 + 10), -np.degrees(theta), 1.0)
            rot[0, 2] += px - tile.shape[1] / 2
            rot[1, 2] += py - (th / 2 + 10)
            warped = cv2.warpAffine(tile, rot, (w, h), flags=cv2.INTER_LINEAR, borderValue=(255, 255, 255))
            page = np.minimum(page, warped)
            s += cw + 2
        words.append(word)
    return page, words


BENDS = (30, 60, 90, 120)
# words read per bend (of 24: 4 pages x 6 words) by the first H100 run, without and with polygons
EXPECTED = {30: (24, 24), 60: (2, 2), 90: (0, 1), 120: (0, 0)}


def _read(results, words):
    got = 0
    for res, ws in zip(results, words):
        texts = [w[0] for w in res]
        for word in ws:
            if word in texts:
                texts.remove(word)
                got += 1
    return got


def curved_pages(bend, n=4):
    rng = np.random.default_rng(100 + bend)
    pages = [render_curved(rng, bend) for _ in range(n)]
    return np.stack([p[0] for p in pages]), [p[1] for p in pages]


def test_curved_pages(pipe):
    table = {}
    for bend in BENDS:
        images, words = curved_pages(bend)
        plain = _read(pipe.recognize(images), words)
        poly = _read(pipe.recognize(images, return_polygons=True), words)
        table[bend] = (plain, poly)
    print("curved words read (default, polygons) of 24 per bend:", table)
    for bend, (plain, poly) in table.items():
        assert poly >= plain, (bend, plain, poly)
    if EXPECTED is not None:
        assert table == EXPECTED


def test_composition(pipe):
    images, _ = curved_pages(90, n=2)
    base = pipe.recognize(images, return_polygons=True)
    scored = pipe.recognize(images, return_polygons=True, return_scores=True)
    for b, s in zip(base, scored):
        for (t, box, poly), (t2, box2, score, conf, poly2) in zip(b, s):
            assert t == t2 and 0 < conf <= 1 and score >= 0.7
            _same(poly, poly2)
    beam = pipe.recognize(images, return_polygons=True, recognition_kwargs={"beam_width": 8, "top_paths": 2})
    assert all(isinstance(w[0], list) and len(w[0]) == 2 for page in beam for w in page)
    words = sorted({w[0] for page in base for w in page if w[0]})
    lex = pipe.recognize(images, return_polygons=True, recognition_kwargs={"lexicon": words})
    assert [[w[0] for w in p] for p in lex] == [[w[0] for w in p] for p in base]
    pipe.inflight = 2
    try:
        split = pipe.recognize(np.concatenate([images] * 4), return_polygons=True)
    finally:
        pipe.inflight = 1
    for g, r in zip(split[:2], base):
        assert [w[0] for w in g] == [w[0] for w in r]
    n0 = pipe.detector.ctx.launch_count() + pipe.recognizer.ctx.launch_count()
    with pytest.raises(ValueError):
        pipe.recognize(images, return_polygons=True, recognition_kwargs={"rotations": (0, 2)})
    with pytest.raises(ValueError):
        pipe.recognize(images, return_polygons=True, return_char_boxes=True)
    assert pipe.detector.ctx.launch_count() + pipe.recognizer.ctx.launch_count() == n0


def test_detect_and_recognize_from_boxes_with_polygons(pipe):
    images, _ = curved_pages(30, n=2)
    padded, _ = pipe.prepare_device(images)
    batch = padded.cpu().numpy()
    boxes, polys = zip(*pipe.detector.detect(batch, return_polygons=True))
    assert [len(b) for b in boxes] == [len(b) for b in pipe.detector.detect(batch)]
    for g, b in zip(polys, boxes):
        for p, q in zip(g, b):
            if len(p) == 4:
                _same(p, q)
    # every box as a straight 3-segment polygon (the top and bottom edges cut in thirds) next to the boxes themselves
    cut = [[np.concatenate([q[0] + (q[1] - q[0]) * np.arange(4)[:, None] / 3,
                            q[3] + (q[2] - q[3]) * np.arange(3, -1, -1)[:, None] / 3]).astype(np.float32) for q in b]
           for b in boxes]
    mixed = [[p if k % 2 else q for k, (p, q) in enumerate(zip(c, b))] for c, b in zip(cut, boxes)]
    texts = pipe.recognizer.recognize_from_boxes(batch, mixed)
    plain = pipe.recognizer.recognize_from_boxes(batch, list(boxes))
    assert [len(t) for t in texts] == [len(t) for t in plain]
    for t, r in zip(texts, plain):                                       # the 4-point entries read exactly as boxes
        assert t[::2] == r[::2]
    assert sum(a == b for t, r in zip(texts, plain) for a, b in zip(t[1::2], r[1::2])) >= 0.9 * sum(len(t[1::2]) for t in texts)
    assert plain == [[w[0] for w in page] for page in pipe.recognize(images)]
    with pytest.raises(ValueError):
        recognition.check_polygons([np.zeros((7, 2))])
