"""GPU: the image stages of csrc/image.cu bit for bit against the references of tests/image_refs.py (pinned against
cv2 in tests/test_image_refs.py): the fp64 warp plan on its own, warpBox crops and the CRNN input for gray and colour
over the whole case set, resize + pad at the pipeline's downscales, identity and 1-pixel sources, and RGB -> gray on
every triplet."""
import cv2
import numpy as np
import pytest
import torch

from keras_ocr_b200 import _lib
from tests import image_refs as R

pytestmark = pytest.mark.gpu

GROUPS = R.warp_cases()


def _stream():
    return torch.cuda.current_stream().cuda_stream


@pytest.fixture(scope="module")
def ctx(cuda_device):
    c = _lib.Context(0)
    yield c
    c.close()


def _dev(a, device):
    """A device copy; keep it referenced until the kernel has run (a temporary's memory is reused at once)."""
    return torch.from_numpy(np.ascontiguousarray(a)).to(device)


# ------------------------------------------------------------------------------------------------- warpBox
@pytest.mark.parametrize("group", GROUPS, ids=[g["name"] for g in GROUPS])
def test_warp_plan_bit_exact(ctx, cuda_device, group):
    """plan_warp == inv3(get_persp(order_corners(box), dst)) in every bit of the 9 doubles, the same dsize, and
    valid == 0 exactly where warpBox raises ZeroDivisionError."""
    quads = group["quads"]
    n = len(quads)
    quads_t = _dev(quads, cuda_device)
    plans = torch.full((n * _lib.WARP_PLAN_DTYPE.itemsize,), 0xA5, dtype=torch.uint8, device=cuda_device)
    ctx.warp_plan_test(quads_t.data_ptr(), n, plans.data_ptr(), _stream())
    got = plans.cpu().numpy().view(_lib.WARP_PLAN_DTYPE)
    bad = []
    for k, q in enumerate(quads):
        try:
            m, dw, dh = R.warp_plan(q)
        except ZeroDivisionError:
            if got["valid"][k] != 0 or got["m"][k].any() or got["dw"][k] != 0 or got["dh"][k] != 0:
                bad.append((k, "valid for a degenerate box"))
            continue
        if got["valid"][k] != 1 or (got["dw"][k], got["dh"][k]) != (dw, dh):
            bad.append((k, int(got["valid"][k]), (int(got["dw"][k]), int(got["dh"][k])), (dw, dh)))
        elif (got["m"][k].view(np.uint64) != m.view(np.uint64)).any():
            bad.append((k, q.tolist(), got["m"][k].tolist(), m.tolist()))
    assert not bad, bad


@pytest.mark.parametrize("color", [False, True], ids=["gray", "color"])
@pytest.mark.parametrize("group", GROUPS, ids=[g["name"] for g in GROUPS])
def test_warp_crops_and_crnn_input_bit_exact(ctx, cuda_device, group, color):
    """b2o_warp_boxes(_color) crops == the reference on every box (degenerate boxes all zero), its CRNN input ==
    b2o_crops_to_input(_color) of those crops == crop[::-1].T / 255 in fp16."""
    img = group["rgb"] if color else group["gray"]
    quads, index = group["quads"], group["image_index"]
    b, ch = len(quads), 3 if color else 1
    assert (b * R.CROP_H * R.CROP_W * ch) % 256 != 0
    n, h, w = img.shape[:3]
    shape = (b, R.CROP_H, R.CROP_W) + ((3,) if color else ())
    crops = torch.full(shape, 0x5A, dtype=torch.uint8, device=cuda_device)
    crnn_in = torch.full((b, R.CROP_W, R.CROP_H) + shape[3:], float("nan"), dtype=torch.float16, device=cuda_device)
    img_t, quads_t, index_t = _dev(img, cuda_device), _dev(quads, cuda_device), _dev(index, cuda_device)
    ctx.warp_boxes(img_t.data_ptr(), n, h, w, quads_t.data_ptr(), index_t.data_ptr(), b, crops.data_ptr(),
                   crnn_in.data_ptr(), _stream(), color=color)
    got = crops.cpu().numpy()
    bad = []
    for k, (q, i) in enumerate(zip(quads, index)):
        ref, plan = R.warp_box(img[i], q)                   # an all-zero crop where plan is None
        if not np.array_equal(got[k], ref):
            bad.append((k, q.tolist(), None if plan is None else plan[1:], int((got[k] != ref).sum())))
    assert not bad, bad
    again = torch.full_like(crnn_in, float("nan"))
    ctx.crops_to_input(crops.data_ptr(), b, again.data_ptr(), _stream(), color=color)
    x = crnn_in.cpu().numpy()
    assert np.array_equal(again.cpu().numpy(), x)
    assert np.array_equal(x, R.crops_to_input(got))


# ------------------------------------------------------------------------------------------------- resize + pad
RESIZE = R.resize_cases()


@pytest.mark.parametrize("case", RESIZE, ids=[c[0] for c in RESIZE])
def test_resize_pad_bit_exact(ctx, cuda_device, case):
    """b2o_resize_pad (into slot 1 of 2) and b2o_resize_pad_batch (n = 1, gray fused) == cv2.resize + pad(255)."""
    _, hs, ws, hr, wr = case
    hp, wp = R.padded(hr, wr)
    src = np.random.default_rng(hs * 7919 + ws).integers(0, 256, (hs, ws, 3), dtype=np.uint8)
    ref = R.resize_pad(src, hr, wr, hp, wp)
    src_t = _dev(src, cuda_device)
    dst = torch.zeros((2, hp, wp, 3), dtype=torch.uint8, device=cuda_device)
    ctx.resize_pad(src_t.data_ptr(), hs, ws, hr, wr, dst.data_ptr(), 1, hp, wp, _stream())
    one = dst.cpu().numpy()
    assert np.array_equal(one[1], ref) and not one[0].any()
    batch = torch.zeros((1, hp, wp, 3), dtype=torch.uint8, device=cuda_device)
    gray = torch.zeros((1, hp, wp), dtype=torch.uint8, device=cuda_device)
    ctx.resize_pad_batch(src_t.data_ptr(), 1, hs, ws, hr, wr, batch.data_ptr(), hp, wp, gray.data_ptr(), _stream())
    assert np.array_equal(batch.cpu().numpy()[0], ref)
    assert np.array_equal(gray.cpu().numpy()[0], cv2.cvtColor(ref, cv2.COLOR_RGB2GRAY))


@pytest.mark.parametrize("n,hs,ws,hr,wr", [(1, 77, 93, 206, 250), (3, 131, 197, 232, 350), (8, 45, 67, 100, 150),
                                           (8, 64, 48, 37, 29)])
def test_resize_pad_batch_fused_gray_bit_exact(ctx, cuda_device, n, hs, ws, hr, wr):
    """One launch over n sources: every image == cv2.resize + pad(255), the gray plane == cv2.cvtColor of the padded
    batch, and the launch without a gray plane writes the same images."""
    hp, wp = R.padded(hr, wr)
    src = np.random.default_rng(n * 1000 + hs).integers(0, 256, (n, hs, ws, 3), dtype=np.uint8)
    ref = np.stack([R.resize_pad(s, hr, wr, hp, wp) for s in src])
    src_t = _dev(src, cuda_device)
    batch = torch.zeros((n, hp, wp, 3), dtype=torch.uint8, device=cuda_device)
    gray = torch.zeros((n, hp, wp), dtype=torch.uint8, device=cuda_device)
    ctx.resize_pad_batch(src_t.data_ptr(), n, hs, ws, hr, wr, batch.data_ptr(), hp, wp, gray.data_ptr(), _stream())
    assert np.array_equal(batch.cpu().numpy(), ref)
    assert np.array_equal(gray.cpu().numpy(), np.stack([cv2.cvtColor(r, cv2.COLOR_RGB2GRAY) for r in ref]))
    plain = torch.zeros_like(batch)
    ctx.resize_pad_batch(src_t.data_ptr(), n, hs, ws, hr, wr, plain.data_ptr(), hp, wp, None, _stream())
    assert torch.equal(plain, batch)


# ------------------------------------------------------------------------------------------------- RGB -> gray
def test_gray_every_rgb_triplet(ctx, cuda_device):
    """b2o_rgb_to_gray on all 2^24 triplets == cv2.cvtColor; the gray plane fused into b2o_resize_pad_batch (identity
    resize, so the padded image is the source) agrees on every triplet too."""
    img = R.all_rgb_triplets()
    want = cv2.cvtColor(img, cv2.COLOR_RGB2GRAY)
    t = _dev(img, cuda_device)
    gray = torch.zeros((4096, 4096), dtype=torch.uint8, device=cuda_device)
    ctx.rgb_to_gray(t.data_ptr(), 1, 4096, 4096, gray.data_ptr(), _stream())
    assert np.array_equal(gray.cpu().numpy(), want)
    out = torch.zeros((1, 4096, 4101, 3), dtype=torch.uint8, device=cuda_device)
    fused = torch.zeros((1, 4096, 4101), dtype=torch.uint8, device=cuda_device)
    ctx.resize_pad_batch(t.data_ptr(), 1, 4096, 4096, 4096, 4096, out.data_ptr(), 4096, 4101, fused.data_ptr(), _stream())
    assert np.array_equal(out.cpu().numpy()[0, :, :4096], img)
    f = fused.cpu().numpy()[0]
    assert np.array_equal(f[:, :4096], want) and (f[:, 4096:] == R.gray_of(np.full(3, 255, np.uint8))).all()
