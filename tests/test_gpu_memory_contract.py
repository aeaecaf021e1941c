"""Where every C entry point writes and what it reads: its memory contract, checked byte by byte.

Each output and each workspace lives inside a guarded buffer (``Guarded``): GUARD bytes before and after it in the same
allocation, its own start 256-byte aligned, every byte prefilled with one pattern.  Workspaces are exactly
``b2o_*_workspace_bytes`` long, so the trailing guard starts at the last legal byte + 1.  Every case runs once per
prefill pattern -- 0x00, 0xFF and, for buffers holding only fp16 / fp32 data, 0x7B (0x7B7B is a large finite fp16,
0x7B7B7B7B a large finite fp32; it survives max and ReLU, which absorb a NaN or a zero).  Buffers of indices or labels
never get 0x7B (they take 0x00 in that run): a stale index must show as a wrong value, never as an address.  A workspace
takes the next run's pattern, so bytes copied from untouched scratch into an output differ from the output's prefill.

For every case (``run``):
  (a) every guard byte is unchanged;
  (b) the bytes the header says are written are bit-identical under every prefill, i.e. do not depend on prior content;
  (c) the bytes the header says are not written still hold the prefill;
  (d) every const input is bit-unchanged (only the documented in-place arguments may change);
  (e) a rejected call returns its documented status, writes no output or workspace byte and launches nothing;
  (f) an empty call (b = 0, n_boxes = 0) writes nothing and launches nothing.

The written extents, one row per entry point (c = min(counts[i], max_boxes) per image; "ws" = scratch, guards only):

  resize_pad             dst slot `index` (hp*wp*3), every other slot untouched
  resize_pad_batch       dst (n,hp,wp,3) all; gray (n,hp,wp) all when given
  rgb_to_gray            gray (n,h,w) all
  warp_boxes[_color|_turned]  crops (n_boxes,31,200[,3]) all; crnn_in (n_boxes,200,31[,3]) fp16 all when given
  crops_to_input[_color] crnn_in (b,200,31[,3]) all
  craft_forward          scores (n,h/2,w/2,2) all; ws
  get_boxes[_scored]     counts (n) all; boxes[i][:c] and box_scores[i][:c]; slots past c untouched; ws
  get_boxes_test         as _scored, labels (n,hs,ws) all, comps[i][:c] (slots past c untouched); labels / comps NULL
                         is rejected before anything runs
  compact_boxes          flat[:sum c] and image_index[:sum c]; the rest untouched
  pack_records[_scored]  records (rows, record_floats[_scored]) all, padding rows included
  select_rotation        labels_out, logp_out, turn_out all; boxes (b,4,2) and the table slots of the b words in
                         place, every other table slot untouched
  crnn_forward[_scored|_logits]  labels (b,48) all; logp (b) all when given; ws
  crnn_forward_beam / _lexicon   labels (b,P,48) all; logp (b,P) all; ws (the CRNN's, then the lexicon scratch)
  crnn_features          features (b,48,256) fp16 all; ws
  ctc_beam_decode        labels (b,P,48) all; logp (b,P) all
  ctc_lexicon_decode     labels (b,P,48) all; logp (b,P) all; ws
  ctc_align              spans (b,P,48,2) all; logp (b,P) all when given
  char_cells             cells (b,P,48,4,2) all
  ctc_loss_grad          loss (b) all; logits (b,48,K) all -- the rows of a bad crop are NaN; grad_w, grad_b all; ws
  rmsprop_step           param, acc: the n elements in place; grad unchanged
  crnn_set_top           reads w, bias only
  decode_jpeg            rgb (h,w,3) all
  crnn_align             spans (b,P,48,2), logp (b,P), theta (b,6) all, and only after a forward that kept its logits
                         in the same ws with the same b (B2O_ERR_STATE otherwise, nothing written)
  crnn_tap               out: the tap's bytes, and only for a buffer the last forward wrote in that ws with that b
"""
import ctypes

import numpy as np
import pytest
import torch

from keras_ocr_b200 import _lib, weights as W

pytestmark = pytest.mark.gpu

GUARD = 4096
FLOAT_RUNS = (0x00, 0xFF, 0x7B)       # prefill of fp16 / fp32 buffers, one run each
INDEX_RUNS = (0x00, 0xFF, 0x00)       # the same runs for buffers holding indices or labels
OK, ERR_ARG, ERR_WORKSPACE, ERR_STATE = 0, -2, -4, -5
T = 48


def _stream():
    return torch.cuda.current_stream().cuda_stream


class Guarded:
    """``nbytes`` at a 256-byte aligned address inside one allocation, GUARD bytes of guard on each side, all prefilled
    with ``fill``."""

    def __init__(self, nbytes, fill):
        self.nbytes, self.fill = int(nbytes), int(fill)
        self.raw = torch.full((GUARD + self.nbytes + GUARD,), self.fill, dtype=torch.uint8, device="cuda")
        assert self.ptr % 256 == 0

    @property
    def ptr(self):
        return self.raw.data_ptr() + GUARD

    def view(self, dtype):
        return self.raw[GUARD:GUARD + self.nbytes].view(dtype)

    def guards_changed(self):
        return int((self.raw[:GUARD] != self.fill).sum() + (self.raw[GUARD + self.nbytes:] != self.fill).sum())

    def interior_changed(self):
        return int((self.raw[GUARD:GUARD + self.nbytes] != self.fill).sum())

    def interior(self):
        return self.raw[GUARD:GUARD + self.nbytes].cpu().numpy()


def _bytes(a):
    return np.ascontiguousarray(a).view(np.uint8).reshape(-1)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def rows(n_rows, row_bytes, keep):
    """Byte mask of a (n_rows, row_bytes) buffer: row r written iff keep[r]."""
    return np.repeat(np.asarray(keep, bool), row_bytes)


def run(ctx, call, bufs, inputs=(), status=OK, launches=None, float_runs=True):
    """Runs ``call(g)`` once per prefill run, g = {name: Guarded}; ``bufs`` = {name: (nbytes, kind, written)}, kind "f"
    (fp16 / fp32 only: 0x7B run too) or "i", written = True (all), False (none), None (scratch: guards only) or a
    callable (interiors of the first run) -> byte mask.  ``inputs``: device tensors that must not change.
    Returns the interiors of the first run."""
    n_runs = 3 if float_runs else 2
    got = []
    for r in range(n_runs):
        # a scratch buffer takes the next run's pattern: a copy of untouched scratch into an output differs from the
        # output's own prefill
        g = {k: Guarded(nb, (FLOAT_RUNS if kind == "f" else INDEX_RUNS)[(r + (w is None)) % 3])
             for k, (nb, kind, w) in bufs.items()}
        before = [t.clone() for t in inputs]
        torch.cuda.synchronize()
        n0 = ctx.launch_count()
        rc = call(g)
        torch.cuda.synchronize()
        assert rc == status, (rc, ctx.lib.b2o_last_error(ctx.handle))
        if launches is not None:
            assert ctx.launch_count() - n0 == launches
        for k, buf in g.items():
            assert buf.guards_changed() == 0, f"{k}: a guard byte changed (prefill {buf.fill:#x})"
            if bufs[k][2] is False:
                assert buf.interior_changed() == 0, f"{k}: a byte of an unwritten buffer changed (prefill {buf.fill:#x})"
        for t, t0 in zip(inputs, before):
            assert torch.equal(t.view(torch.uint8), t0.view(torch.uint8)), "a const input changed"
        got.append({k: (buf.interior(), buf.fill) for k, buf in g.items()
                    if bufs[k][2] is not None and bufs[k][2] is not False})
    first = {k: v[0] for k, v in got[0].items()}
    for k, (nb, kind, written) in bufs.items():
        if written is None or written is False:
            continue
        if callable(written):
            mask = np.asarray(written(first), bool)
        else:
            mask = np.full(nb, written) if isinstance(written, bool) else np.asarray(written, bool)
        assert mask.shape == (nb,)
        for run_bytes in got:
            data, fill = run_bytes[k]
            assert np.array_equal(data[mask], first[k][mask]), f"{k}: written bytes depend on the prefill ({fill:#x})"
            bad = np.flatnonzero(data[~mask] != fill)
            assert bad.size == 0, f"{k}: {bad.size} bytes outside the written extent changed (prefill {fill:#x})"
    return first


def rejected(ctx, call, bufs, status, inputs=()):
    """(e): the call returns ``status``, every output / workspace byte keeps its prefill, no launch."""
    run(ctx, call, {k: (nb, kind, False) for k, (nb, kind) in bufs.items()}, inputs, status=status, launches=0)


# ------------------------------------------------------------------------------------------ contexts
@pytest.fixture(scope="module")
def ctx(cuda_device):
    return _lib.Context(0)


@pytest.fixture(scope="module")
def crnn(cuda_device):
    c = _lib.Context(0)
    c.load_crnn(W.synthetic_crnn_weights(seed=2))
    return c


@pytest.fixture(scope="module")
def crnn_k3(cuda_device):
    alphabet = "ab"
    c = _lib.Context(0)
    c.load_crnn(W.synthetic_crnn_weights(seed=5, alphabet=alphabet))
    return c


def _crnn_input(b, seed, ch=1):
    rng = np.random.default_rng(seed)
    x = (rng.integers(0, 256, (b, 200, 31) + ((ch,) if ch > 1 else ()), dtype=np.uint8) / 255).astype(np.float16)
    x[:, 120:] = 0                                                  # the zero tail of a warpBox crop
    return _dev(x)


# ------------------------------------------------------------------------------------------ images
def test_resize_pad(ctx):
    rng = np.random.default_rng(1)
    hs, ws_, hr, wr, hp, wp, n = 37, 53, 29, 41, 33, 47, 3
    src = _dev(rng.integers(0, 256, (hs, ws_, 3), dtype=np.uint8))
    slot = hp * wp * 3
    L = ctx.lib
    out = run(ctx, lambda g: L.b2o_resize_pad(ctx.handle, src.data_ptr(), hs, ws_, hr, wr, g["dst"].ptr, 1, hp, wp,
                                              _stream()),
              {"dst": (n * slot, "i", rows(n, slot, [False, True, False]))}, [src], float_runs=False)
    assert (out["dst"][slot:2 * slot].reshape(hp, wp, 3)[hr:] == 255).all()
    rejected(ctx, lambda g: L.b2o_resize_pad(ctx.handle, src.data_ptr(), hs, ws_, hp + 1, wr, g["dst"].ptr, 1, hp, wp,
                                             _stream()), {"dst": (n * slot, "i")}, ERR_ARG, [src])


@pytest.mark.parametrize("gray", [False, True], ids=["rgb", "with_gray"])
def test_resize_pad_batch(ctx, gray):
    rng = np.random.default_rng(2)
    n, hs, ws_, hr, wr, hp, wp = 3, 37, 53, 29, 41, 33, 47
    src = _dev(rng.integers(0, 256, (n, hs, ws_, 3), dtype=np.uint8))
    bufs = {"dst": (n * hp * wp * 3, "i", True)}
    if gray:
        bufs["gray"] = (n * hp * wp, "i", True)
    L = ctx.lib

    def call(g, hr=hr):
        return L.b2o_resize_pad_batch(ctx.handle, src.data_ptr(), n, hs, ws_, hr, wr, g["dst"].ptr, hp, wp,
                                      g["gray"].ptr if gray else None, _stream())
    run(ctx, call, bufs, [src], float_runs=False)
    rejected(ctx, lambda g: call(g, hr=hp + 1), {k: v[:2] for k, v in bufs.items()}, ERR_ARG, [src])


def test_rgb_to_gray(ctx):
    n, h, w = 2, 33, 47
    img = _dev(np.random.default_rng(3).integers(0, 256, (n, h, w, 3), dtype=np.uint8))
    L = ctx.lib
    run(ctx, lambda g: L.b2o_rgb_to_gray(ctx.handle, img.data_ptr(), n, h, w, g["gray"].ptr, _stream()),
        {"gray": (n * h * w, "i", True)}, [img], float_runs=False)
    rejected(ctx, lambda g: L.b2o_rgb_to_gray(ctx.handle, img.data_ptr(), 0, h, w, g["gray"].ptr, _stream()),
             {"gray": (n * h * w, "i")}, ERR_ARG, [img])


def _boxes(n_boxes, n, h, w, seed):
    """n_boxes rotated quads inside (h, w) images, the last one degenerate (all four corners equal) when n_boxes > 1."""
    rng = np.random.default_rng(seed)
    out = np.zeros((n_boxes, 4, 2), np.float32)
    for k in range(n_boxes):
        cx, cy = rng.uniform(20, w - 20), rng.uniform(10, h - 10)
        a, bw, bh = rng.uniform(-0.4, 0.4), rng.uniform(8, 30), rng.uniform(4, 12)
        c, s = np.cos(a), np.sin(a)
        for j, (dx, dy) in enumerate(((-bw, -bh), (bw, -bh), (bw, bh), (-bw, bh))):
            out[k, j] = (cx + c * dx - s * dy, cy + s * dx + c * dy)
    if n_boxes > 1:
        out[-1] = out[-1, 0]
    idx = np.sort(rng.integers(0, n, n_boxes)).astype(np.int32)
    return _dev(out), _dev(idx)


@pytest.mark.parametrize("n_boxes", [1, 7])
@pytest.mark.parametrize("variant", ["gray", "color", "turned0", "turned1", "turned2", "turned3", "gray_no_crnn_in"])
def test_warp_boxes(ctx, n_boxes, variant):
    n, h, w = 2, 64, 96
    ch = 3 if variant == "color" else 1
    rng = np.random.default_rng(4)
    img = _dev(rng.integers(0, 256, (n, h, w) + ((3,) if ch == 3 else ()), dtype=np.uint8))
    boxes, idx = _boxes(n_boxes, n, h, w, seed=n_boxes)
    want_in = variant != "gray_no_crnn_in"
    bufs = {"crops": (n_boxes * 31 * 200 * ch, "i", True)}
    if want_in:
        bufs["crnn_in"] = (n_boxes * 200 * 31 * ch * 2, "f", True)
    L = ctx.lib
    turn = int(variant[-1]) if variant.startswith("turned") else None

    def call(g, turn=turn, nb=n_boxes):
        cin = g["crnn_in"].ptr if want_in else None
        args = (img.data_ptr(), n, h, w, boxes.data_ptr(), idx.data_ptr(), nb)
        if turn is not None:
            return L.b2o_warp_boxes_turned(ctx.handle, img.data_ptr(), ch, n, h, w, boxes.data_ptr(), idx.data_ptr(),
                                           nb, turn, g["crops"].ptr, cin, _stream())
        fn = L.b2o_warp_boxes_color if ch == 3 else L.b2o_warp_boxes
        return fn(ctx.handle, *args, g["crops"].ptr, cin, _stream())
    out = run(ctx, call, bufs, [img, boxes, idx])
    if n_boxes > 1:                                                  # the degenerate box: an all-zero crop
        assert not out["crops"].reshape(n_boxes, -1)[-1].any()
    sizes = {k: v[:2] for k, v in bufs.items()}
    rejected(ctx, lambda g: call(g, turn=4), sizes, ERR_ARG, [img, boxes, idx])
    run(ctx, lambda g: call(g, nb=0), {k: (nb, kind, False) for k, (nb, kind) in sizes.items()}, [img, boxes, idx],
        launches=0)


@pytest.mark.parametrize("color", [False, True])
def test_crops_to_input(ctx, color):
    b, ch = 3, 3 if color else 1
    crops = _dev(np.random.default_rng(5).integers(0, 256, (b, 31, 200, ch), dtype=np.uint8))
    fn = ctx.lib.b2o_crops_to_input_color if color else ctx.lib.b2o_crops_to_input
    run(ctx, lambda g: fn(ctx.handle, crops.data_ptr(), b, g["x"].ptr, _stream()), {"x": (b * 200 * 31 * ch * 2, "f", True)},
        [crops])
    rejected(ctx, lambda g: fn(ctx.handle, crops.data_ptr(), -1, g["x"].ptr, _stream()), {"x": (b * 6200 * ch * 2, "f")},
             ERR_ARG, [crops])
    run(ctx, lambda g: fn(ctx.handle, crops.data_ptr(), 0, g["x"].ptr, _stream()), {"x": (64, "f", False)}, [crops],
        launches=0)


# ------------------------------------------------------------------------------------------ detector
@pytest.fixture(scope="module")
def craft(cuda_device):
    c = _lib.Context(0)
    c.load_craft(W.synthetic_craft_weights(3))
    return c


@pytest.mark.parametrize("shape", [(2, 33, 47), (1, 32, 2048)])
def test_craft_forward(craft, shape):
    n, h, w = shape
    img = _dev(np.random.default_rng(6).integers(0, 256, (n, h, w, 3), dtype=np.uint8))
    nbytes = craft.craft_workspace_bytes(n, h, w)
    sbytes = n * (h // 2) * (w // 2) * 2 * 4
    L = craft.lib

    def call(g, ws_bytes=nbytes):
        return L.b2o_craft_forward(craft.handle, img.data_ptr(), n, h, w, g["scores"].ptr, g["ws"].ptr, ws_bytes, _stream())
    run(craft, call, {"scores": (sbytes, "f", True), "ws": (nbytes, "f", None)}, [img])
    rejected(craft, lambda g: call(g, nbytes - 1), {"scores": (sbytes, "f"), "ws": (nbytes, "f")}, ERR_WORKSPACE, [img])


def _score_map(n, hs, ws_):
    """Image 0: 12 separate 4 x 4 text blobs; image 1: nothing above any threshold (no box)."""
    s = np.zeros((n, hs, ws_, 2), np.float32)
    for k in range(12):
        y, x = 3 + 9 * (k // 5), 3 + 10 * (k % 5)
        s[0, y:y + 4, x:x + 4, 0] = 0.9 - 0.01 * k
    return _dev(s)


@pytest.mark.parametrize("max_boxes", [1, 16])
@pytest.mark.parametrize("entry", ["get_boxes", "scored", "scored_null", "test"])
def test_get_boxes(ctx, max_boxes, entry):
    n, hs, ws_ = 2, 40, 56
    scores = _score_map(n, hs, ws_)
    nbytes = ctx.boxes_workspace_bytes(n, hs, ws_, max_boxes)
    L = ctx.lib
    thr = (0.7, 0.4, 0.4, 10)

    def kept(itemsize):                                              # slots k < min(counts[i], max_boxes)
        def mask(first):
            c = np.minimum(first["counts"].view(np.int32), max_boxes)
            return np.concatenate([np.repeat(np.arange(max_boxes) < c[i], itemsize) for i in range(n)])
        return mask
    bufs = {"boxes": (n * max_boxes * 32, "f", kept(32)), "counts": (n * 4, "i", True), "ws": (nbytes, "i", None)}
    if entry in ("scored", "test"):
        bufs["box_scores"] = (n * max_boxes * 4, "f", kept(4))
    if entry == "test":
        bufs["labels"] = (n * hs * ws_ * 4, "i", True)
        bufs["comps"] = (n * max_boxes * 28, "i", kept(28))

    def call(g, ws_bytes=nbytes, labels=True):
        p = lambda k: g[k].ptr if k in g else None                   # noqa: E731
        if entry == "get_boxes":
            return L.b2o_get_boxes(ctx.handle, scores.data_ptr(), n, hs, ws_, *thr, p("boxes"), p("counts"), max_boxes,
                                   p("ws"), ws_bytes, _stream())
        if entry == "test":
            return L.b2o_get_boxes_test(ctx.handle, scores.data_ptr(), n, hs, ws_, *thr, p("boxes"), p("counts"),
                                        p("box_scores"), max_boxes, p("ws"), ws_bytes, p("labels") if labels else None,
                                        p("comps"), _stream())
        return L.b2o_get_boxes_scored(ctx.handle, scores.data_ptr(), n, hs, ws_, *thr, p("boxes"), p("counts"),
                                      p("box_scores"), max_boxes, p("ws"), ws_bytes, _stream())
    out = run(ctx, call, bufs, [scores], float_runs=False)
    assert list(out["counts"].view(np.int32)) == [12, 0]               # max_boxes 1: the overflow path
    sizes = {k: v[:2] for k, v in bufs.items()}
    rejected(ctx, lambda g: call(g, nbytes - 1), sizes, ERR_WORKSPACE, [scores])
    if entry == "test":                                              # refused before getBoxes runs
        rejected(ctx, lambda g: call(g, labels=False), sizes, ERR_ARG, [scores])


def test_compact_boxes(ctx):
    n, mb = 3, 4
    table = _dev(np.random.default_rng(7).normal(size=(n, mb, 4, 2)).astype(np.float32))
    counts = _dev(np.array([2, 0, 9], np.int32))                     # 9 > max_boxes: 4 are stored
    L = ctx.lib
    kept = 2 + 0 + 4
    out = run(ctx, lambda g: L.b2o_compact_boxes(ctx.handle, table.data_ptr(), counts.data_ptr(), n, mb, g["flat"].ptr,
                                                 g["index"].ptr, _stream()),
              {"flat": (n * mb * 32, "f", rows(n * mb, 32, np.arange(n * mb) < kept)),
               "index": (n * mb * 4, "i", rows(n * mb, 4, np.arange(n * mb) < kept))}, [table, counts])
    assert list(out["index"].view(np.int32)[:kept]) == [0, 0, 2, 2, 2, 2]
    rejected(ctx, lambda g: L.b2o_compact_boxes(ctx.handle, table.data_ptr(), counts.data_ptr(), 0, mb, g["flat"].ptr,
                                                g["index"].ptr, _stream()),
             {"flat": (n * mb * 32, "f"), "index": (n * mb * 4, "i")}, ERR_ARG, [table, counts])


@pytest.mark.parametrize("scored", [False, True])
@pytest.mark.parametrize("case", ["short_shard", "empty"])
def test_pack_records(ctx, scored, case):
    n, rows_, mb, rec_boxes = 2, 3, 4, 2                             # rows > n: a short last shard
    rng = np.random.default_rng(8)
    table = _dev(rng.normal(size=(n, mb, 4, 2)).astype(np.float32) * 100)
    cnt = [3, 1] if case == "short_shard" else [0, 0]                # image 0: more boxes than rec_boxes
    counts = _dev(np.array(cnt, np.int32))
    total = sum(min(c, mb) for c in cnt)
    labels = _dev(rng.integers(-1, 36, (max(total, 1), T)).astype(np.int32)) if total else None
    box_scores = _dev(rng.uniform(0, 1, (n, mb)).astype(np.float32))
    logp = _dev(-rng.uniform(0, 9, max(total, 1)).astype(np.float32)) if total else None
    inv = _dev(np.array([0.5, 2.0], np.float32))
    fl = (ctx.record_floats_scored if scored else ctx.record_floats)(rec_boxes)
    L = ctx.lib
    ptr = lambda t: t.data_ptr() if t is not None else None          # noqa: E731
    ins = [t for t in (table, counts, labels, box_scores, logp, inv) if t is not None]

    def call(g, rows_=rows_):
        if scored:
            return L.b2o_pack_records_scored(ctx.handle, table.data_ptr(), counts.data_ptr(), ptr(labels),
                                             box_scores.data_ptr(), ptr(logp), inv.data_ptr(), n, mb, rows_, rec_boxes,
                                             g["rec"].ptr, _stream())
        return L.b2o_pack_records(ctx.handle, table.data_ptr(), counts.data_ptr(), ptr(labels), inv.data_ptr(), n, mb,
                                  rows_, rec_boxes, g["rec"].ptr, _stream())
    out = run(ctx, call, {"rec": (rows_ * fl * 4, "i", True)}, ins, float_runs=False)
    rec = out["rec"].view(np.float32).reshape(rows_, fl)
    assert list(rec[:, 0]) == [min(cnt[0], mb), min(cnt[1], mb), -1]
    rejected(ctx, lambda g: call(g, rows_=n - 1), {"rec": (rows_ * fl * 4, "i")}, ERR_ARG, ins)


@pytest.mark.parametrize("vote", [_lib.ROTATION_VOTE_WORD, _lib.ROTATION_VOTE_PAGE], ids=["word", "page"])
@pytest.mark.parametrize("turns", [(2,), (1, 3, 0, 2)], ids=["one_turn", "four_turns"])
@pytest.mark.parametrize("in_place", [False, True], ids=["no_boxes", "boxes_and_table"])
def test_select_rotation(ctx, vote, turns, in_place):
    rng = np.random.default_rng(9)
    b, n_images, tp, mb, nt = 5, 2, 3, 4, len(turns)
    idx = _dev(np.array([0, 0, 0, 1, 1], np.int32))
    labels = _dev(rng.integers(-1, 36, (nt, b, tp, T)).astype(np.int32))
    logp = _dev(-rng.uniform(0, 20, (nt, b, tp)).astype(np.float32))
    boxes0 = rng.normal(size=(b, 4, 2)).astype(np.float32)
    table0 = rng.normal(size=(n_images, mb, 4, 2)).astype(np.float32)
    table0[0, :3], table0[1, :2] = boxes0[:3], boxes0[3:]
    bufs = {"labels": (b * tp * T * 4, "i", True), "logp": (b * tp * 4, "f", True), "turn": (b * 4, "i", True)}
    L = ctx.lib
    th = (ctypes.c_int32 * nt)(*turns)
    state = {}

    def call(g, n_turns=nt):
        boxes, table = _dev(boxes0), _dev(table0)
        state.update(boxes=boxes, table=table)
        rc = L.b2o_select_rotation(ctx.handle, labels.data_ptr(), logp.data_ptr(), idx.data_ptr(), n_images, b, tp, th,
                                   n_turns, vote, g["labels"].ptr, g["logp"].ptr, g["turn"].ptr,
                                   boxes.data_ptr() if in_place else None, table.data_ptr() if in_place else None, mb,
                                   _stream())
        torch.cuda.synchronize()
        state.update(boxes=boxes.cpu().numpy(), table=table.cpu().numpy())
        return rc
    out = run(ctx, call, bufs, [labels, logp, idx])
    chosen = out["turn"].view(np.int32)
    assert set(chosen) <= set(turns)
    if in_place:             # each box's own corners, reordered; the words' table slots receive them, the rest unchanged
        got = state["boxes"]
        for k in range(b):
            assert np.array_equal(np.unique(got[k], axis=0), np.unique(boxes0[k], axis=0))
        tab = table0.copy()
        tab[0, :3], tab[1, :2] = got[:3], got[3:]
        assert np.array_equal(state["table"], tab)
    else:
        assert np.array_equal(state["boxes"], boxes0) and np.array_equal(state["table"], table0)
    rejected(ctx, lambda g: call(g, n_turns=5), {k: v[:2] for k, v in bufs.items()}, ERR_ARG, [labels, logp, idx])
    assert np.array_equal(state["boxes"], boxes0) and np.array_equal(state["table"], table0)


# ------------------------------------------------------------------------------------------ recognizer
def _lexicon():
    words = [[0, 1, 2], [], [5] * 30, [3], [7, 7], [40], [1, 2, 3, 4]]        # empty, unalignable, out of range
    off = np.zeros(len(words) + 1, np.int32)
    off[1:] = np.cumsum([len(wd) for wd in words])
    return _dev(off), _dev(np.array([c for wd in words for c in wd], np.int16)), len(words)


@pytest.mark.parametrize("b", [1, 9, 17])
@pytest.mark.parametrize("entry", ["forward", "scored", "scored_null", "logits", "lexicon", "features"])
def test_crnn_forward(crnn, b, entry):
    x = _crnn_input(b, seed=b)
    nbytes = crnn.crnn_workspace_bytes(b)
    off, lab, n_words = _lexicon()
    tp = 8 if entry == "lexicon" else 1                              # more than the 4 finite entries
    if entry == "lexicon":
        nbytes += crnn.lexicon_workspace_bytes(b, n_words, tp)
    L = crnn.lib
    if entry == "features":
        bufs = {"features": (b * T * 256 * 2, "f", True)}
    else:
        bufs = {"labels": (b * tp * T * 4, "i", True)}
        if entry != "forward":
            bufs["logp"] = (b * tp * 4, "f", entry != "scored_null")
    bufs["ws"] = (nbytes, "f" if entry != "lexicon" else "i", None)
    p = lambda g, k: g[k].ptr if k in g and not (k == "logp" and entry == "scored_null") else None   # noqa: E731

    def call(g, ws_bytes=nbytes, bb=b):
        s = _stream()
        if entry == "forward":
            return L.b2o_crnn_forward(crnn.handle, x.data_ptr(), bb, p(g, "labels"), p(g, "ws"), ws_bytes, s)
        if entry in ("scored", "scored_null"):
            return L.b2o_crnn_forward_scored(crnn.handle, x.data_ptr(), bb, p(g, "labels"), p(g, "logp"), p(g, "ws"),
                                             ws_bytes, s)
        if entry == "logits":
            return L.b2o_crnn_forward_logits(crnn.handle, x.data_ptr(), bb, p(g, "labels"), p(g, "logp"), p(g, "ws"),
                                             ws_bytes, s)
        if entry == "lexicon":
            return L.b2o_crnn_forward_lexicon(crnn.handle, x.data_ptr(), bb, off.data_ptr(), lab.data_ptr(), n_words, tp,
                                              p(g, "labels"), p(g, "logp"), p(g, "ws"), ws_bytes, s)
        return L.b2o_crnn_features(crnn.handle, x.data_ptr(), bb, p(g, "features"), p(g, "ws"), ws_bytes, s)
    out = run(crnn, call, bufs, [x, off, lab])
    if entry == "lexicon":                                           # slots past the finite entries: -1 and -inf
        assert (out["labels"].view(np.int32).reshape(b, tp, T)[:, 4:] == -1).all()
        assert (out["logp"].view(np.float32).reshape(b, tp)[:, 4:] == -np.inf).all()
    sizes = {k: v[:2] for k, v in bufs.items()}
    rejected(crnn, lambda g: call(g, nbytes - 1), sizes, ERR_WORKSPACE, [x])
    run(crnn, lambda g: call(g, bb=0), {k: (nb, kind, False) for k, (nb, kind) in sizes.items()}, [x], launches=0)


@pytest.mark.parametrize("b", [1, 9, 17])
def test_crnn_forward_beam_more_paths_than_prefixes(crnn_k3, b):
    """K = 3, top_paths = beam_width = 128: the beam starts with fewer distinct prefixes than paths."""
    x = _crnn_input(b, seed=30 + b)
    nbytes, tp = crnn_k3.crnn_workspace_bytes(b), 128
    L = crnn_k3.lib

    def call(g, ws_bytes=nbytes):
        return L.b2o_crnn_forward_beam(crnn_k3.handle, x.data_ptr(), b, 128, tp, g["labels"].ptr, g["logp"].ptr,
                                       g["ws"].ptr, ws_bytes, _stream())
    bufs = {"labels": (b * tp * T * 4, "i", True), "logp": (b * tp * 4, "f", True), "ws": (nbytes, "f", None)}
    run(crnn_k3, call, bufs, [x])
    rejected(crnn_k3, lambda g: call(g, nbytes - 1), {k: v[:2] for k, v in bufs.items()}, ERR_WORKSPACE, [x])


def _logits(b, k, seed):
    return _dev((np.random.default_rng(seed).normal(size=(b, T, k)) * 3).astype(np.float32))


@pytest.mark.parametrize("k", [2, 1024])
def test_ctc_beam_decode(ctx, k):
    b, bw, tp = 3, 128, 128
    lg = _logits(b, k, seed=k)
    L = ctx.lib
    bufs = {"labels": (b * tp * T * 4, "i", True), "logp": (b * tp * 4, "f", True)}

    def call(g, top=tp, bb=b):
        return L.b2o_ctc_beam_decode(ctx.handle, lg.data_ptr(), bb, k, bw, top, g["labels"].ptr, g["logp"].ptr, _stream())
    out = run(ctx, call, bufs, [lg])
    if k == 2:                                                       # blank and one label: fewer prefixes than paths
        assert (out["logp"].view(np.float32) == -np.inf).any()
    sizes = {kk: v[:2] for kk, v in bufs.items()}
    rejected(ctx, lambda g: call(g, top=bw + 1), sizes, ERR_ARG, [lg])
    run(ctx, lambda g: call(g, bb=0), {kk: (nb, kind, False) for kk, (nb, kind) in sizes.items()}, [lg], launches=0)


@pytest.mark.parametrize("k", [2, 1024])
def test_ctc_lexicon_decode(ctx, k):
    b, tp = 3, 8
    lg = _logits(b, k, seed=k + 1)
    off, lab, n_words = _lexicon()
    nbytes = ctx.lexicon_workspace_bytes(b, n_words, tp)
    L = ctx.lib
    bufs = {"labels": (b * tp * T * 4, "i", True), "logp": (b * tp * 4, "f", True), "ws": (nbytes, "i", None)}

    def call(g, ws_bytes=nbytes):
        return L.b2o_ctc_lexicon_decode(ctx.handle, lg.data_ptr(), b, k, off.data_ptr(), lab.data_ptr(), n_words, tp,
                                        g["labels"].ptr, g["logp"].ptr, g["ws"].ptr, ws_bytes, _stream())
    out = run(ctx, call, bufs, [lg, off, lab])
    finite = int(np.isfinite(out["logp"].view(np.float32).reshape(b, tp)[0]).sum())
    assert finite < tp
    rejected(ctx, lambda g: call(g, nbytes - 1), {kk: v[:2] for kk, v in bufs.items()}, ERR_WORKSPACE, [lg, off, lab])


def _readings(b, tp, k, seed):
    """Readings of every kind: ordinary, empty, unalignable (too many doubled letters), a label outside [0, k-2]."""
    rng = np.random.default_rng(seed)
    out = np.full((b, tp, T), -1, np.int32)
    for i in range(b):
        for p in range(tp):
            kind = (i * tp + p) % 4
            if kind == 0:
                n = int(rng.integers(1, 10))
                out[i, p, :n] = rng.integers(0, k - 1, n)
            elif kind == 2:
                out[i, p, :25] = 0
            elif kind == 3:
                out[i, p, :2] = (0, k - 1)
    return _dev(out)


@pytest.mark.parametrize("k", [2, 1024])
@pytest.mark.parametrize("with_logp", [True, False])
def test_ctc_align_and_char_cells(ctx, k, with_logp):
    b, tp = 3, 128
    lg, labels = _logits(b, k, seed=k + 2), _readings(b, tp, k, seed=k)
    L = ctx.lib
    bufs = {"spans": (b * tp * T * 8, "i", True)}
    if with_logp:
        bufs["logp"] = (b * tp * 4, "f", True)
    state = {}

    def call(g, top=tp):
        rc = L.b2o_ctc_align(ctx.handle, lg.data_ptr(), b, k, labels.data_ptr(), top, g["spans"].ptr,
                             g["logp"].ptr if with_logp else None, _stream())
        state["spans"] = g["spans"].view(torch.int32).clone()
        return rc
    run(ctx, call, bufs, [lg, labels])
    rejected(ctx, lambda g: call(g, top=129), {kk: v[:2] for kk, v in bufs.items()}, ERR_ARG, [lg, labels])
    # char_cells on those spans, with and without theta / boxes / turns
    spans = state["spans"]
    rng = np.random.default_rng(k)
    theta = _dev(np.tile(np.array([1, 0.02, 0.01, -0.03, 1.05, 0.1], np.float32), (b, 1)))
    boxes, _ = _boxes(b, 1, 64, 96, seed=3)
    turns = _dev(rng.integers(0, 4, b).astype(np.int32))
    for th, bx, tu in ((None, None, None), (theta, None, None), (theta, boxes, turns), (None, boxes, None)):
        ins = [t for t in (spans, th, bx, tu) if t is not None]
        ptr = lambda t: t.data_ptr() if t is not None else None      # noqa: E731
        run(ctx, lambda g: L.b2o_char_cells(ctx.handle, spans.data_ptr(), b, tp, ptr(th), ptr(bx), ptr(tu), g["cells"].ptr,
                                            _stream()), {"cells": (b * tp * T * 32, "f", True)}, ins)
    rejected(ctx, lambda g: L.b2o_char_cells(ctx.handle, spans.data_ptr(), b, tp, None, None, turns.data_ptr(),
                                             g["cells"].ptr, _stream()), {"cells": (b * tp * T * 32, "f")}, ERR_ARG, [spans])


# ------------------------------------------------------------------------------------------ training
@pytest.mark.parametrize("grads", [True, False], ids=["grads", "loss_only"])
def test_ctc_loss_grad(ctx, grads):
    """b = 17: the last 16-crop split-K chunk holds one crop.  Crops 2 (empty text), 5 (a label outside [0, K-2]) and 11
    (row index outside [0, n_rows)) are bad: loss +inf / NaN, no gradient, and their logits rows all NaN."""
    k, n_rows, b = 37, 20, 17
    rng = np.random.default_rng(10)
    feats = _dev(np.tanh(rng.normal(size=(n_rows, T, 256))).astype(np.float16))
    w = _dev((rng.normal(size=(256, k)) * 0.1).astype(np.float32))
    bias = _dev((rng.normal(size=k) * 0.5).astype(np.float32))
    texts = [[int(c) for c in rng.integers(0, k - 1, int(rng.integers(1, 8)))] for _ in range(b)]
    texts[2], texts[5] = [], [k - 1]
    off = np.zeros(b + 1, np.int32)
    off[1:] = np.cumsum([len(t) for t in texts])
    off, lab = _dev(off), _dev(np.array([c for t in texts for c in t], np.int16))
    index = np.arange(b, dtype=np.int32) % n_rows
    index[11] = n_rows
    index = _dev(index)
    nbytes = ctx.ctc_train_workspace_bytes(b, k)
    L = ctx.lib
    bufs = {"loss": (b * 4, "f", True), "logits": (b * T * k * 4, "f", True)}
    if grads:
        bufs.update(gw=(256 * k * 4, "f", True), gb=(k * 4, "f", True), ws=(nbytes, "f", None))

    def call(g, ws_bytes=nbytes, bb=b):
        p = lambda kk: g[kk].ptr if kk in g else None                # noqa: E731
        return L.b2o_ctc_loss_grad(ctx.handle, feats.data_ptr(), n_rows, index.data_ptr(), bb, k, w.data_ptr(),
                                   bias.data_ptr(), off.data_ptr(), lab.data_ptr(), 0.0, 0, 0, p("loss"), p("gw"), p("gb"),
                                   p("logits"), p("ws"), ws_bytes if grads else 0, _stream())
    ins = [feats, w, bias, off, lab, index]
    out = run(ctx, call, bufs, ins)
    loss = out["loss"].view(np.float32)
    assert loss[2] == np.inf and loss[5] == np.inf and np.isnan(loss[11]) and np.isfinite(np.delete(loss, [2, 5, 11])).all()
    lg = out["logits"].view(np.float32).reshape(b, T, k)
    assert np.isnan(lg[[2, 5, 11]]).all() and np.isfinite(np.delete(lg, [2, 5, 11], 0)).all()
    sizes = {kk: v[:2] for kk, v in bufs.items()}
    if grads:
        rejected(ctx, lambda g: call(g, nbytes - 1), sizes, ERR_WORKSPACE, ins)
    rejected(ctx, lambda g: call(g, bb=-1), sizes, ERR_ARG, ins)
    run(ctx, lambda g: call(g, bb=0), {kk: (nb, kind, False) for kk, (nb, kind) in sizes.items()}, ins, launches=0)


@pytest.mark.parametrize("n", [1, 255, 257])
def test_rmsprop_step(ctx, n):
    rng = np.random.default_rng(n)
    p0 = rng.normal(size=n).astype(np.float32)
    g0 = rng.normal(size=n).astype(np.float32)
    a0 = rng.uniform(0, 1, n).astype(np.float32)
    bufs = {}
    for name, v in (("param", p0), ("grad", g0), ("acc", a0)):
        buf = Guarded(n * 4, 0x7B)
        buf.view(torch.float32).copy_(torch.from_numpy(v))
        bufs[name] = buf
    grad_before = bufs["grad"].view(torch.uint8).clone()
    n0 = ctx.launch_count()
    assert ctx.lib.b2o_rmsprop_step(ctx.handle, bufs["param"].ptr, bufs["grad"].ptr, bufs["acc"].ptr, n, 1e-3, 0.9, 1e-7,
                                    _stream()) == OK
    torch.cuda.synchronize()
    assert ctx.launch_count() - n0 == 1
    assert all(buf.guards_changed() == 0 for buf in bufs.values())
    assert torch.equal(bufs["grad"].view(torch.uint8), grad_before)
    one = np.float32(1)
    acc = np.float32(0.9) * a0 + (one - np.float32(0.9)) * (g0 * g0)
    param = p0 - (np.float32(1e-3) * g0) / (np.sqrt(acc) + np.float32(1e-7))
    assert np.array_equal(bufs["acc"].view(torch.float32).cpu().numpy(), acc)
    assert np.array_equal(bufs["param"].view(torch.float32).cpu().numpy(), param)
    n0 = ctx.launch_count()
    assert ctx.lib.b2o_rmsprop_step(ctx.handle, bufs["param"].ptr, bufs["grad"].ptr, bufs["acc"].ptr, 0, 1e-3, 0.9, 1e-7,
                                    _stream()) == OK
    assert ctx.lib.b2o_rmsprop_step(ctx.handle, bufs["param"].ptr, bufs["grad"].ptr, bufs["acc"].ptr, n, -1.0, 0.9, 1e-7,
                                    _stream()) == ERR_ARG
    torch.cuda.synchronize()
    assert ctx.launch_count() == n0
    assert np.array_equal(bufs["param"].view(torch.float32).cpu().numpy(), param)


def test_crnn_set_top_reads_only(cuda_device):
    c = _lib.Context(0)
    wts = W.synthetic_crnn_weights(seed=2)
    c.load_crnn(wts)
    k = len(W.ALPHABET) + 1
    w, bias = Guarded(256 * k * 4, 0x7B), Guarded(k * 4, 0x7B)
    w.view(torch.float32).copy_(torch.from_numpy(np.asarray(wts["fc_12.kernel"], np.float32).reshape(-1)))
    bias.view(torch.float32).copy_(torch.from_numpy(np.asarray(wts["fc_12.bias"], np.float32)))
    before = (w.raw.clone(), bias.raw.clone())
    n0 = c.launch_count()
    assert c.lib.b2o_crnn_set_top(c.handle, w.ptr, bias.ptr, k, _stream()) == OK
    assert c.lib.b2o_crnn_set_top(c.handle, w.ptr, bias.ptr, k + 1, _stream()) == ERR_ARG
    torch.cuda.synchronize()
    assert c.launch_count() == n0
    assert torch.equal(w.raw, before[0]) and torch.equal(bias.raw, before[1])


@pytest.mark.parametrize("kind", ["color_420", "gray_odd_width"])
def test_decode_jpeg(ctx, kind):
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(11)
    h, w = 45, 67
    if kind == "color_420":
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        ok, enc = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, 90, cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                                             cv2.IMWRITE_JPEG_SAMPLING_FACTOR_420])
    else:
        ok, enc = cv2.imencode(".jpg", rng.integers(0, 256, (h, w), dtype=np.uint8))
    assert ok
    data = enc.tobytes()
    if ctx.jpeg_info(data) is None:
        pytest.skip("nvJPEG is not available")
    assert ctx.jpeg_info(data)[:2] == (h, w)
    buf = (ctypes.c_ubyte * len(data)).from_buffer_copy(data)
    L = ctx.lib
    run(ctx, lambda g: L.b2o_decode_jpeg(ctx.handle, buf, len(data), g["rgb"].ptr, h, w, _stream()),
        {"rgb": (h * w * 3, "i", True)}, float_runs=False)
    rejected(ctx, lambda g: L.b2o_decode_jpeg(ctx.handle, buf, len(data), None, h, w, _stream()), {"rgb": (h * w * 3, "i")},
             ERR_ARG)


# ------------------------------------------------------------------------------------------ CRNN state
TAP_BYTES = {"features": 50 * 7 * 512 * 2, "theta": 24, "warped": 50 * 7 * 512 * 2, "fc_9": 50 * 128 * 2,
             "l1": 50 * 128 * 2, "l2": 50 * 256 * 2, "logits": 48 * 37 * 4, "x1": 200 * 31 * 64 * 2,
             "x2": 200 * 31 * 128 * 2, "x3": 200 * 31 * 256 * 2, "p3": 100 * 15 * 256 * 2, "x4": 100 * 15 * 256 * 2,
             "x5": 100 * 15 * 512 * 2, "p5": 50 * 7 * 512 * 2, "x6": 50 * 7 * 512 * 2}
BACKBONE = ("features", "theta", "warped", "fc_9", "l1", "l2", "x1", "x2", "p3", "x4", "p5", "x6")


class _CrnnRun:
    """A CRNN context, its input and two exact-size workspaces of b = 9 and one of b = 5."""

    def __init__(self, c):
        self.c, self.b = c, 9
        self.x = _crnn_input(9, seed=40)
        self.ws = {bb: torch.zeros(c.crnn_workspace_bytes(bb), dtype=torch.uint8, device="cuda") for bb in (9, 5)}
        self.other = torch.zeros(c.crnn_workspace_bytes(9), dtype=torch.uint8, device="cuda")
        self.labels = torch.empty((9, T), dtype=torch.int32, device="cuda")

    def forward(self, how, b=9, ws=None):
        ws = self.ws[b] if ws is None else ws
        c, L, s = self.c, self.c.lib, _stream()
        args = (c.handle, self.x.data_ptr(), b)
        if how == "forward":
            rc = L.b2o_crnn_forward(*args, self.labels.data_ptr(), ws.data_ptr(), ws.numel(), s)
        elif how == "logits":
            rc = L.b2o_crnn_forward_logits(*args, self.labels.data_ptr(), None, ws.data_ptr(), ws.numel(), s)
        elif how == "beam":
            lab = torch.empty((b, 2, T), dtype=torch.int32, device="cuda")
            rc = L.b2o_crnn_forward_beam(*args, 4, 2, lab.data_ptr(), None, ws.data_ptr(), ws.numel(), s)
        elif how == "lexicon":
            off, lab, nw = _lexicon()
            need = c.crnn_workspace_bytes(b) + c.lexicon_workspace_bytes(b, nw, 1)
            ws = torch.zeros(need, dtype=torch.uint8, device="cuda")
            self.lex_ws = ws
            out = torch.empty((b, T), dtype=torch.int32, device="cuda")
            rc = L.b2o_crnn_forward_lexicon(*args, off.data_ptr(), lab.data_ptr(), nw, 1, out.data_ptr(), None,
                                            ws.data_ptr(), ws.numel(), s)
        else:
            feats = torch.empty((b, T, 256), dtype=torch.float16, device="cuda")
            rc = L.b2o_crnn_features(*args, feats.data_ptr(), ws.data_ptr(), ws.numel(), s)
        assert rc == OK
        return ws

    def tap(self, name, b=9, ws=None):
        ws = self.ws[b] if ws is None else ws
        out = Guarded(b * TAP_BYTES[name], 0x7B)
        rc = self.c.lib.b2o_crnn_tap(self.c.handle, name.encode(), ws.data_ptr(), b, out.ptr, out.nbytes, _stream())
        torch.cuda.synchronize()
        assert out.guards_changed() == 0
        if rc != OK:
            assert (out.interior() == 0x7B).all()
        return rc, out

    def align(self, b=9, ws=None):
        ws = self.ws[b] if ws is None else ws
        labels = torch.full((b, 1, T), -1, dtype=torch.int32, device="cuda")
        spans, logp, theta = Guarded(b * T * 8, 0x00), Guarded(b * 4, 0x7B), Guarded(b * 24, 0x7B)
        n0 = self.c.launch_count()
        rc = self.c.lib.b2o_crnn_align(self.c.handle, b, labels.data_ptr(), 1, spans.ptr, logp.ptr, theta.ptr,
                                       ws.data_ptr(), ws.numel(), _stream())
        torch.cuda.synchronize()
        assert all(g.guards_changed() == 0 for g in (spans, logp, theta))
        if rc != OK:
            assert self.c.launch_count() == n0
            assert (spans.interior() == 0).all() and (logp.interior() == 0x7B).all() and (theta.interior() == 0x7B).all()
        return rc


@pytest.fixture
def crnn_run(cuda_device):
    c = _lib.Context(0)
    c.load_crnn(W.synthetic_crnn_weights(seed=2))
    return _CrnnRun(c)


def test_crnn_tap_and_align_before_any_forward(crnn_run):
    assert crnn_run.tap("l2")[0] == ERR_STATE
    assert crnn_run.align() == ERR_STATE


@pytest.mark.parametrize("how", ["logits", "beam", "lexicon"])
def test_crnn_align_after_a_forward_that_kept_its_logits(crnn_run, how):
    ws = crnn_run.forward(how)
    assert crnn_run.align(ws=ws) == OK
    rc, out = crnn_run.tap("logits", ws=ws)
    assert rc == OK and np.isfinite(out.interior().view(np.float32)).all()
    assert crnn_run.align(b=5, ws=ws) == ERR_STATE                  # another b moves every slot
    assert crnn_run.align(ws=crnn_run.other) == ERR_STATE           # another workspace
    assert crnn_run.tap("logits", ws=crnn_run.other)[0] == ERR_STATE


@pytest.mark.parametrize("how", ["forward", "features"])
def test_crnn_align_refused_without_logits(crnn_run, how):
    """A greedy forward with the debug taps off does not keep its logits, b2o_crnn_features stops after l2: the logits
    slot holds whatever was there before, so align and the tap refuse -- also when the taps are switched on later."""
    crnn_run.forward(how)
    assert crnn_run.align() == ERR_STATE
    assert crnn_run.tap("logits")[0] == ERR_STATE
    crnn_run.c.set_debug_taps(1)
    assert crnn_run.tap("logits")[0] == ERR_STATE
    assert crnn_run.align() == ERR_STATE
    for name in BACKBONE:                                            # what the forward did write stays readable
        assert crnn_run.tap(name)[0] == OK, name
    crnn_run.forward("forward")                                      # now with the taps on: the logits are kept
    assert crnn_run.tap("logits")[0] == OK and crnn_run.align() == OK


def test_crnn_tap_follows_the_last_forward(crnn_run):
    crnn_run.forward("logits", b=5)
    crnn_run.forward("logits")
    assert crnn_run.tap("l2", b=5)[0] == ERR_STATE                 # an earlier forward's b and ws
    assert crnn_run.tap("l2")[0] == OK
    assert crnn_run.tap("x3")[0] == ERR_STATE and crnn_run.tap("x5")[0] == ERR_STATE     # AUTO fuses their pools
    for name in BACKBONE + ("logits",):
        assert crnn_run.tap(name)[0] == OK, name
    crnn_run.c.set_conv_engine(_lib.CONV_SIMT)
    crnn_run.forward("logits")
    assert crnn_run.tap("x3")[0] == OK and crnn_run.tap("x5")[0] == OK
    crnn_run.forward("features")
    assert crnn_run.tap("logits")[0] == ERR_STATE and crnn_run.tap("l2")[0] == OK
    # a rejected forward (workspace one byte short) changes nothing; its slots are still the last forward's
    ws = crnn_run.ws[9]
    assert crnn_run.c.lib.b2o_crnn_forward(crnn_run.c.handle, crnn_run.x.data_ptr(), 9, crnn_run.labels.data_ptr(),
                                           ws.data_ptr(), ws.numel() - 1, _stream()) == ERR_WORKSPACE
    assert crnn_run.tap("l2")[0] == OK


def test_crnn_without_stn_has_no_theta_tap(cuda_device):
    c = _lib.Context(0)
    c.load_crnn(W.synthetic_crnn_weights(seed=5, stn=False))
    r = _CrnnRun(c)
    r.forward("logits")
    assert r.tap("theta")[0] == ERR_STATE and r.tap("warped")[0] == ERR_STATE
    assert r.tap("features")[0] == OK and r.align() == OK
