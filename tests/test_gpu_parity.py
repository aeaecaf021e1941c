"""GPU parity tests: every CUDA stage, called through the C-ABI, against the CPU oracle and the
golden vectors generated from the reference.  Run on an H100: ``pytest tests -m gpu``.

Tolerances (stated per test): integer/byte/index work is bit-exact; fp16 tensor-core stages are
compared with the fp32 oracle at the tolerances proposed in SURVEY.md 8(c).
"""
import os

import numpy as np
import pytest
import torch

from keras_ocr_b200 import _lib, weights as W

pytestmark = pytest.mark.gpu


def _stream():
    return torch.cuda.current_stream().cuda_stream


@pytest.fixture(scope="module")
def ctx(cuda_device):
    c = _lib.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def detector(cuda_device):
    from keras_ocr_b200.detection import Detector
    return Detector(weights=W.synthetic_craft_weights(seed=3))


@pytest.fixture(scope="module")
def recognizer(cuda_device):
    from keras_ocr_b200.recognition import Recognizer
    r = Recognizer(weights=W.synthetic_crnn_weights(seed=2))
    r.keep_workspace = True
    return r


# ------------------------------------------------------------------------------- conv engines
CONV_CASES = [
    # n, h, w, cin, cout, k, dil, relu, affine2
    (2, 16, 16, 64, 64, 3, 1, 1, 0),
    (1, 24, 40, 128, 256, 3, 1, 1, 0),
    (1, 9, 13, 512, 1024, 3, 6, 0, 0),      # dilated slice5.1 shape, odd spatial size
    (3, 17, 23, 64, 32, 3, 1, 1, 0),        # ragged tiles, batch-spanning boxes
    (2, 50, 7, 512, 16, 5, 1, 1, 0),        # STN conv_a: 5x5, tiny cout, W smaller than the box
    (2, 50, 7, 512, 512, 3, 1, 1, 1),       # CRNN conv_7: ReLU then BN affine
    (1, 1, 300, 3584, 128, 1, 1, 1, 0),     # fc_9 as a 1x1 conv over rows
    (1, 8, 8, 1536, 512, 1, 1, 1, 0),       # upconv1.conv.0
    (1, 96, 96, 64, 64, 3, 1, 1, 0),        # many tiles per CTA (persistent loop, the stage ring wraps)
    (2, 40, 48, 32, 32, 3, 1, 1, 0),        # conv_cls.0: 32-channel K chunk (64B swizzle), resident filters
    (1, 33, 29, 32, 16, 3, 1, 1, 0),        # conv_cls.4, ragged halo tiles
    (2, 50, 7, 16, 32, 5, 1, 1, 0),         # STN conv_b: 16-channel K chunk (32B swizzle), 5x5
    (1, 48, 40, 128, 128, 3, 1, 1, 0),      # halo tiles with a streamed (non-resident) filter bank
    (1, 32, 24, 256, 512, 3, 1, 1, 0),      # halo tiles, four n-tiles of 128
    (2, 40, 56, 16, 64, 3, 1, 1, 0),        # tensor-core stem shape: 16-channel chunk, resident filters
]

ENGINES = [_lib.CONV_SIMT, _lib.CONV_TC_GENERIC, _lib.CONV_AUTO]
# ids kept from the first tensor-core engine (tcgen05) so that test ids stay stable: "tcgen05_generic" = the tensor-core
# engine without halo tiles (B2O_CONV_TC_GENERIC), "tcgen05" = the product path (B2O_CONV_AUTO, wgmma on sm_90a)
ENGINE_IDS = ["simt", "tcgen05_generic", "tcgen05"]


def _torch_conv_reference(x, wgt, k, dil, s1, t1, relu, s2, t2):
    xt = x.float().permute(0, 3, 1, 2)
    wt = torch.from_numpy(wgt).to(x.device).half().float().permute(0, 3, 1, 2)      # (cout,cin,k,k), fp16-rounded
    y = torch.nn.functional.conv2d(xt, wt, padding=dil * (k // 2), dilation=dil)
    y = y * torch.from_numpy(s1).to(x.device)[None, :, None, None] + torch.from_numpy(t1).to(x.device)[None, :, None, None]
    if relu:
        y = torch.relu(y)
    if s2 is not None:
        y = y * torch.from_numpy(s2).to(x.device)[None, :, None, None] + torch.from_numpy(t2).to(x.device)[None, :, None, None]
    return y.permute(0, 2, 3, 1).contiguous()


@pytest.mark.parametrize("engine", ENGINES, ids=ENGINE_IDS)
@pytest.mark.parametrize("case", CONV_CASES, ids=[f"n{c[0]}_{c[1]}x{c[2]}_{c[3]}to{c[4]}_k{c[5]}d{c[6]}" for c in CONV_CASES])
def test_conv_engine_vs_fp32(ctx, cuda_device, case, engine):
    n, h, w, cin, cout, k, dil, relu, aff = case
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    rng = np.random.default_rng(hash(case) % (2 ** 31))
    x = torch.from_numpy(rng.standard_normal((n, h, w, cin)).astype(np.float32)).to(cuda_device).half().contiguous()
    wgt = (rng.standard_normal((cout, k, k, cin)) * np.sqrt(2.0 / (cin * k * k))).astype(np.float32)
    s1 = rng.uniform(0.7, 1.3, cout).astype(np.float32)
    t1 = (rng.standard_normal(cout) * 0.2).astype(np.float32)
    s2 = rng.uniform(0.7, 1.3, cout).astype(np.float32) if aff else None
    t2 = (rng.standard_normal(cout) * 0.2).astype(np.float32) if aff else None
    out = torch.full((n, h, w, cout), float("nan"), dtype=torch.float16, device=cuda_device)
    ctx.conv2d_test(x.data_ptr(), n, h, w, cin, wgt, cout, k, dil, s1, t1, relu, s2, t2, out.data_ptr(), engine, _stream())
    torch.cuda.synchronize()
    ref = _torch_conv_reference(x, wgt, k, dil, s1, t1, relu, s2, t2)
    err = (out.float() - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert np.isfinite(err), "NaN/unwritten output"
    # fp32 accumulation, one fp16 rounding of the result: |err| <= 2^-10 * |y| (+ accumulation-order noise)
    assert err <= 2.5e-3 * max(scale, 1.0), (err, scale)


# ------------------------------------------------------------------------------- image stages
@pytest.mark.parametrize("tag", ["x2", "capped", "x3"])
def test_resize_pad_bit_exact(ctx, cuda_device, golden_dir, tag):
    g = np.load(os.path.join(golden_dir, "inputs.npz"))
    src, ref = g[f"resize_{tag}_src"], g[f"resize_{tag}_dst"]
    hr, wr = ref.shape[:2]
    hp, wp = hr + 5, wr + 9
    src_t = torch.from_numpy(src).to(cuda_device)
    dst = torch.zeros((2, hp, wp, 3), dtype=torch.uint8, device=cuda_device)
    ctx.resize_pad(src_t.data_ptr(), src.shape[0], src.shape[1], hr, wr, dst.data_ptr(), 1, hp, wp, _stream())
    out = dst.cpu().numpy()[1]
    assert np.array_equal(out[:hr, :wr], ref)                       # cv2.resize, bit-exact
    assert (out[hr:] == 255).all() and (out[:, wr:] == 255).all()   # tools.pad cval=255
    with pytest.raises(_lib.B2OError):                              # tools.pad's assert: target smaller than image
        ctx.resize_pad(src_t.data_ptr(), src.shape[0], src.shape[1], hr, wr, dst.data_ptr(), 0, hr - 1, wr, _stream())


def test_gray_bit_exact(ctx, cuda_device):
    from oracle import imageops
    rng = np.random.default_rng(3)
    img = rng.integers(0, 256, (2, 37, 53, 3), dtype=np.uint8)
    t = torch.from_numpy(img).to(cuda_device)
    gray = torch.empty((2, 37, 53), dtype=torch.uint8, device=cuda_device)
    ctx.rgb_to_gray(t.data_ptr(), 2, 37, 53, gray.data_ptr(), _stream())
    assert np.array_equal(gray.cpu().numpy(), np.stack([imageops.rgb_to_gray(i) for i in img]))


def test_warp_boxes_vs_reference_golden(recognizer, cuda_device, golden_dir):
    g = np.load(os.path.join(golden_dir, "warp.npz"))
    gray = torch.from_numpy(g["warp_gray"][None]).to(cuda_device).contiguous()
    quads = torch.from_numpy(g["warp_quads"]).to(cuda_device).contiguous()
    idx = torch.zeros(len(g["warp_quads"]), dtype=torch.int32, device=cuda_device)
    crnn_in, crops = recognizer.warp_device(gray, quads, idx, want_crops=True)
    crops = crops.cpu().numpy()
    # bit for bit: M differs from cv2's in the last ulps on most quads, but the 1/32-pixel rounding of the sampler
    # absorbs that on every golden crop (the kernel's own plan is pinned bit for bit in test_gpu_image_stages.py)
    assert np.array_equal(crops, g["warp_crops"]), int((crops != g["warp_crops"]).sum())
    # CRNN input layout: x[b, t, j] = crop[b, 30 - j, t] / 255   (recognition.py:215-216, 524)
    expect = (crops[:, ::-1, :].transpose(0, 2, 1).astype(np.float32) / 255).astype(np.float16)
    assert np.array_equal(crnn_in.cpu().numpy(), expect)


# ------------------------------------------------------------------------------- getBoxes
def _match_quads(mine, ref):
    """max corner distance allowing a cyclic shift of the starting corner (argmin(x+y) ties)."""
    return min(np.abs(np.roll(mine, s, 0) - ref).max() for s in range(4))


def _check_boxes(detector, scores, ref_groups, tol=1e-3):
    t = torch.from_numpy(np.ascontiguousarray(scores)).to(detector.device)
    boxes, counts = detector.boxes_device(t)
    boxes = boxes.cpu().numpy()
    assert list(counts) == [len(r) for r in ref_groups]            # same components kept, same order
    worst = 0.0
    for i, ref in enumerate(ref_groups):
        for k in range(len(ref)):
            worst = max(worst, _match_quads(boxes[i, k], ref[k]))
    assert worst <= tol, worst


@pytest.mark.parametrize("tag", ["grid32", "rot12", "dense", "blank", "refmaps"])
def test_get_boxes_vs_reference_golden(detector, golden_dir, tag):
    g = np.load(os.path.join(golden_dir, "boxes.npz"))
    counts = g[f"boxes_{tag}_counts"]
    quads = g[f"boxes_{tag}_quads"]
    groups, start = [], 0
    for c in counts:
        groups.append(quads[start:start + c])
        start += c
    _check_boxes(detector, g[f"boxes_{tag}_scores"], groups)


def test_get_boxes_vs_oracle_large_and_adversarial(detector):
    from oracle import imageops, synth
    maps = synth.score_maps(101, 2, 768, 768, 32)
    # adversarial: component of area 9 / 10 / 11, max text 0.699 / 0.701, border-touching blob,
    # a word split in two by text&link removal, a near-square "diamond" blob
    adv = np.zeros((1, 160, 200, 2), np.float32)
    adv[0, 10:13, 10:13, 0] = 0.9                       # area 9  -> dropped (size_threshold)
    adv[0, 10:12, 30:35, 0] = 0.9                       # area 10 -> kept
    adv[0, 20:25, 60:70, 0] = 0.699                     # max below detection threshold -> dropped
    adv[0, 20:25, 90:100, 0] = 0.701                    # kept
    adv[0, 0:8, 150:200, 0] = 0.8                       # touches top and right borders
    adv[0, 60:70, 20:120, 0] = 0.8                      # long word ...
    adv[0, 60:70, 60:80, 1] = 0.9                       # ... whose middle is text & link (removed, 246)
    adv[0, 100:130, 40:70, 0] = 0.85                    # square blob -> "diamond" branch (276-281)
    yy, xx = np.mgrid[0:160, 0:200]
    adv[0, ..., 0] = np.maximum(adv[0, ..., 0], 0.9 * (np.abs(yy - 120) + np.abs(xx - 150) < 18))   # rotated square
    # components beyond the small shared-memory planes of the quads' first pass: two text blocks whose dilation
    # ROI (973 x 403) exceeds even the large planes (global scratch planes, both in one image: the per-image lock),
    # one of them with its middle removed as text & link, a 195-row block (second pass, large shared-memory planes),
    # and an ordinary word next to them
    big = np.zeros((1, 1000, 1000, 2), np.float32)
    big[0, 10:340, 50:950, 0] = 0.9
    big[0, 420:750, 40:940, 0] = 0.85
    big[0, 500:600, 300:500, 1] = 0.9
    big[0, 830:990, 100:400, 0] = 0.9
    big[0, 900:910, 500:560, 0] = 0.8
    for scores in (maps, adv, big):
        _check_boxes(detector, scores, imageops.get_boxes(scores))


def test_get_boxes_overflow_retry(detector):
    from oracle import imageops, synth
    maps = synth.score_maps(7, 1, 256, 256, 40)
    detector.max_boxes = 4                               # force the count > max_boxes retry path
    try:
        _check_boxes(detector, maps, imageops.get_boxes(maps))
        assert detector.max_boxes >= 32
    finally:
        detector.max_boxes = 256


# ------------------------------------------------------------------------------- CRAFT
@pytest.mark.parametrize("engine", ENGINES, ids=ENGINE_IDS)
def test_craft_forward_vs_reference_golden(detector, golden_dir, engine):
    g = np.load(os.path.join(golden_dir, "craft.npz"))
    detector.ctx.set_conv_engine(engine)
    try:
        for tag in ("even", "odd"):
            img = torch.from_numpy(g[f"craft_{tag}_image"]).to(detector.device)
            scores = detector.predict_device(img).cpu().numpy()
            ref = g[f"craft_{tag}_scores"]              # output of the reference's own torch CRAFT, fp32
            assert scores.shape == ref.shape
            err = np.abs(scores - ref).max() / max(np.abs(ref).max(), 1.0)
            # fp16 activations through 27 layers vs fp32: <= 2e-2 of the map's range (SURVEY.md 8(c))
            assert err <= 2e-2, (tag, err)
    finally:
        detector.ctx.set_conv_engine(_lib.CONV_AUTO)


# ------------------------------------------------------------------------------- CRNN
def test_crnn_vs_oracle(recognizer):
    from oracle import crnn
    wts = W.synthetic_crnn_weights(seed=2)
    rng = np.random.default_rng(5)
    b = 6
    crops = rng.integers(0, 256, (b, 31, 200), dtype=np.uint8)
    crops[:, :, 150:] = 0                                   # zero tail like a real warpBox crop
    texts = recognizer.recognize_crops(crops)
    with torch.no_grad():
        probs, inter = crnn.crnn_logits(wts, crops.astype(np.float32) / 255, return_intermediates=True)
    dev = recognizer.device

    def rel(a, ref):
        return float((a - ref).abs().max() / max(ref.abs().max(), 1e-6))

    feat = recognizer.tap("features", (b, 50, 7, 512), torch.float16).float().cpu()
    assert rel(feat, inter["features"].permute(0, 2, 3, 1)) <= 2e-2
    theta = recognizer.tap("theta", (b, 6), torch.float32).cpu()
    assert float((theta - inter["theta"]).abs().max()) <= 2e-2
    warped = recognizer.tap("warped", (b, 50, 7, 512), torch.float16).float().cpu()
    assert rel(warped, inter["warped"]) <= 5e-2               # sampling positions move with theta
    fc9 = recognizer.tap("fc_9", (b, 50, 128), torch.float16).float().cpu()
    assert rel(fc9, inter["fc_9"]) <= 5e-2
    l2 = recognizer.tap("l2", (b, 50, 256), torch.float16).float().cpu()
    assert float((l2 - inter["l2"]).abs().max()) <= 5e-2       # LSTM outputs live in [-1, 1]
    logits = recognizer.tap("logits", (b, 48, 37), torch.float32).cpu()
    ref_logits = inter["logits"]
    assert float((logits - ref_logits).abs().max()) <= 0.15
    # labels: the exact greedy collapse of the device's own logits (integer work).  String identity against the oracle is
    # asserted for every crop with the decisive weights in tests/test_gpu_baseline_sizes.py (C3: 256 crops, C4: full pages).
    labels = recognizer.predict_device(recognizer_input(recognizer, crops)).cpu().numpy()
    assert np.array_equal(labels, crnn.ctc_greedy(torch.softmax(logits, -1)))
    assert texts == crnn.labels_to_text(labels)


def recognizer_input(rec, crops):
    t = torch.from_numpy(np.ascontiguousarray(crops)).to(rec.device)
    x = torch.empty((t.shape[0], 200, 31), dtype=torch.float16, device=rec.device)
    rec.ctx.crops_to_input(t.data_ptr(), t.shape[0], x.data_ptr(), _stream())
    return x


def test_crnn_vs_reference_source_golden(cuda_device, golden_dir):
    """tests/golden/crnn.npz holds what the reference's own build_model / _transform / CTCDecoder source gives
    (executed on oracle/keras_shim.py, decisive weights) on three noise crops and on the word crops of two rendered
    pages.  fp16 tensor-core chain vs that fp32 result: class probabilities within 5e-2 everywhere; on the word crops
    the padded label rows are IDENTICAL to the reference's CTCDecoder output; on every crop the device's labels are the
    exact greedy collapse of the device's own argmax."""
    from keras_ocr_b200.recognition import Recognizer
    from oracle import crnn
    rec = Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True))
    rec.keep_workspace = True
    g = np.load(os.path.join(golden_dir, "crnn.npz"))
    crops, ref_probs, ref_labels, n_noise = g["crnn_crops"], g["crnn_probs"], g["crnn_labels"], int(g["crnn_n_noise"])
    b = crops.shape[0]
    labels = rec.predict_device(recognizer_input(rec, crops)).cpu().numpy()
    probs = torch.softmax(rec.tap("logits", (b, 48, 37), torch.float32), -1).cpu().numpy()
    assert float(np.abs(probs - ref_probs).max()) <= 5e-2
    assert b - n_noise >= 6
    assert np.array_equal(labels[n_noise:], ref_labels[n_noise:])          # the words: every step, padding included
    assert np.array_equal(labels, crnn.ctc_greedy(torch.from_numpy(probs)))  # integer work: exact on every crop


def test_ctc_collapse_exact(recognizer):
    """Greedy CTC on the device equals the oracle's collapse of the device's own logits."""
    from oracle import crnn
    rng = np.random.default_rng(9)
    crops = rng.integers(0, 256, (16, 31, 200), dtype=np.uint8)
    t = torch.from_numpy(crops).to(recognizer.device)
    crnn_in = torch.empty((16, 200, 31), dtype=torch.float16, device=recognizer.device)
    recognizer.ctx.crops_to_input(t.data_ptr(), 16, crnn_in.data_ptr(), _stream())
    labels = recognizer.predict_device(crnn_in).cpu().numpy()
    logits = recognizer.tap("logits", (16, 48, 37), torch.float32).cpu()
    expect = crnn.ctc_greedy(torch.softmax(logits, -1))
    assert np.array_equal(labels, expect)                      # integer work: bit-exact


@pytest.mark.parametrize("alphabet", ["ab", "".join(chr(c) for c in range(32, 127)),
                                      "".join(chr(c) for c in range(0x4E00, 0x4E00 + 300))])
def test_custom_alphabet(cuda_device, alphabet):
    """recognition.py:362-381: the class count follows the alphabet (K = 3, 96, 301).  Logits against the fp32
    oracle within the CRNN tolerance; the device's greedy CTC equals the collapse of its own logits exactly;
    strings use the caller's alphabet."""
    from keras_ocr_b200 import weights as W
    from keras_ocr_b200.recognition import Recognizer
    from oracle import crnn, synth
    w = W.synthetic_crnn_weights(5, alphabet=alphabet)
    rec = Recognizer(alphabet=alphabet, weights=w)
    assert rec.alphabet == alphabet and rec.blank_label_idx == len(alphabet)
    rec.keep_workspace = True
    rng = np.random.default_rng(4)
    crops = np.stack([synth.noise_gray(rng, 31, 200) for _ in range(6)])
    t = torch.from_numpy(crops).to(rec.device)
    crnn_in = torch.empty((6, 200, 31), dtype=torch.float16, device=rec.device)
    rec.ctx.crops_to_input(t.data_ptr(), 6, crnn_in.data_ptr(), _stream())
    labels = rec.predict_device(crnn_in).cpu().numpy()
    K = len(alphabet) + 1
    logits = rec.tap("logits", (6, 48, K), torch.float32).cpu()
    assert np.array_equal(labels, crnn.ctc_greedy(torch.softmax(logits, -1)))
    l2 = rec.tap("l2", (6, 50, 256), torch.float16).float().cpu()[:, 2:]
    own = l2 @ torch.from_numpy(w["fc_12.kernel"]) + torch.from_numpy(w["fc_12.bias"])
    assert float((logits - own).abs().max()) <= 2e-3          # the Dense layer alone: fp32 on both sides
    with torch.no_grad():
        probs, inter = crnn.crnn_logits(w, crops.astype(np.float32) / 255, return_intermediates=True)
    assert float((logits - inter["logits"]).abs().max()) <= 0.15
    texts = rec.recognize_crops(crops)
    assert texts == crnn.labels_to_text(labels, alphabet)
    assert all(set(tx) <= set(alphabet) for tx in texts)


def test_alphabet_mismatch_uses_backbone_only(cuda_device, capsys):
    """recognition.py:399-411: a checkpoint whose top layer does not fit the alphabet keeps the backbone and
    gets a freshly initialised top (same message as the reference)."""
    from keras_ocr_b200 import weights as W
    from keras_ocr_b200.recognition import Recognizer
    rec = Recognizer(alphabet="xyz", weights=W.synthetic_crnn_weights(2))
    assert "Using backbone weights only" in capsys.readouterr().out
    out = rec.recognize_crops(np.zeros((2, 31, 200), np.uint8))
    assert len(out) == 2 and all(set(tx) <= set("xyz") for tx in out)


def test_recognizer_without_spatial_transformer(cuda_device):
    """build_model(stn=False) (recognition.py:196, 243): ``build_params={"stn": False}`` runs the conv stack straight into
    Reshape + fc_9.  Logits against the fp32 oracle (which takes the same branch), labels = exact collapse of the device's
    own logits; a checkpoint that HAS a transformer can be loaded with it switched off; other build_params are refused."""
    from keras_ocr_b200.recognition import Recognizer
    from oracle import crnn, synth
    w = W.synthetic_crnn_weights(5, stn=False)
    assert not any(k.startswith("stn.") for k in w)
    rec = Recognizer(weights=w, build_params={"stn": False})
    rec.keep_workspace = True
    rng = np.random.default_rng(4)
    crops = np.stack([synth.noise_gray(rng, 31, 200) for _ in range(5)])
    texts = rec.recognize_crops(crops)
    logits = rec.tap("logits", (5, 48, 37), torch.float32).cpu()
    with torch.no_grad():
        probs, inter = crnn.crnn_logits(w, crops.astype(np.float32) / 255, return_intermediates=True)
    assert inter["theta"] is None
    assert float((logits - inter["logits"]).abs().max()) <= 0.15
    fc9 = rec.tap("fc_9", (5, 50, 128), torch.float16).float().cpu()
    assert float((fc9 - inter["fc_9"]).abs().max() / inter["fc_9"].abs().max()) <= 5e-2
    assert texts == crnn.labels_to_text(crnn.ctc_greedy(torch.softmax(logits, -1)))
    with pytest.raises(_lib.B2OError):
        rec.tap("theta", (5, 6), torch.float32)
    full = W.synthetic_crnn_weights(5)                               # same seed: identical tensors plus the transformer's
    again = Recognizer(weights=full, build_params={"stn": False})
    assert again.recognize_crops(crops) == texts
    with pytest.raises(ValueError):
        Recognizer(weights=w)                                        # stn=True (default) needs the transformer's tensors
    with pytest.raises(NotImplementedError):
        Recognizer(weights=full, build_params={"rnn_units": (64, 64)})   # other architectures are not implemented


def test_gpu_jpeg_decode(cuda_device, tmp_path):
    """tools.read on the GPU (SURVEY.md 8(f)2): nvJPEG through b2o_decode_jpeg against cv2.imdecode (= what the reference's
    tools.read returns, tools.py:19-38).  The two decoders are not bit-identical (IDCT rounding, chroma upsampling):
    4:4:4 and gray files agree to <= 4 levels (measured 3, mean 0.48); 4:2:0 files differ by up to ~25 levels at sharp colour edges (the chroma
    upsampling filters differ: measured 23 on rendered text) with a mean difference below 0.5 level; the pipeline then finds the same words from paths decoded on the GPU as from host-decoded arrays."""
    import cv2
    from keras_ocr_b200 import tools
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    from keras_ocr_b200.recognition import Recognizer
    from oracle import synth
    ctx = _lib.Context(0)
    pages, _ = synth.text_images(seed=41, n=2, h=192, w=384, n_words=4)
    if ctx.jpeg_info(cv2.imencode(".jpg", pages[0])[1].tobytes()) is None:
        pytest.skip("nvJPEG not available on this box")
    rng = np.random.default_rng(3)
    photo = cv2.GaussianBlur(rng.integers(0, 256, (120, 200, 3)).astype(np.float32), (0, 0), 3).clip(0, 255).astype(np.uint8)
    cases = {"text_420": (pages[0], [cv2.IMWRITE_JPEG_QUALITY, 95]),
             "photo_444": (photo, [cv2.IMWRITE_JPEG_QUALITY, 90, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_444]),
             "gray": (cv2.cvtColor(photo, cv2.COLOR_RGB2GRAY), [cv2.IMWRITE_JPEG_QUALITY, 90])}
    for tag, (img, params) in cases.items():
        data = cv2.imencode(".jpg", img[..., ::-1] if img.ndim == 3 else img, params)[1].tobytes()
        host = tools.read(__import__("io").BytesIO(data))
        dev = tools.read_device(__import__("io").BytesIO(data), ctx, cuda_device)
        assert isinstance(dev, torch.Tensor) and dev.is_cuda and tuple(dev.shape) == host.shape, tag
        diff = np.abs(dev.cpu().numpy().astype(np.int16) - host.astype(np.int16))
        print(f"jpeg {tag}: max {diff.max()} mean {diff.mean():.3f}")
        assert diff.max() <= (32 if tag == "text_420" else 4) and diff.mean() <= 0.6, (tag, int(diff.max()), float(diff.mean()))
    png = str(tmp_path / "p.png")                                  # not a JPEG: host decode, returned as an array
    cv2.imwrite(png, pages[1][..., ::-1])
    assert isinstance(tools.read_device(png, ctx, cuda_device), np.ndarray)
    paths = []
    for i, page in enumerate(pages):
        paths.append(str(tmp_path / f"page{i}.jpg"))
        cv2.imwrite(paths[-1], page[..., ::-1], [cv2.IMWRITE_JPEG_QUALITY, 95])
    det = Detector(weights=W.synthetic_craft_weights(3, textlike=True))
    rec = Recognizer(weights=W.synthetic_crnn_weights(2))
    on_gpu = Pipeline(detector=det, recognizer=rec, scale=2, gpu_decode=True).recognize(paths)
    on_host = Pipeline(detector=det, recognizer=rec, scale=2).recognize(paths)
    assert [len(g) for g in on_gpu] == [len(g) for g in on_host] and sum(len(g) for g in on_host) >= 6
    for g, h in zip(on_gpu, on_host):
        for (_, bg), (_, bh) in zip(g, h):
            assert np.abs(bg - bh).max() <= 1.0                    # a few grey levels do not move a box by a pixel


def test_color_recognizer(cuda_device):
    """build_model(color=True) (recognition.py:214, 508-510): RGB crops, no gray conversion, 3-channel conv_1.
    b2o_warp_boxes_color == cv2.warpPerspective on the RGB image, every channel bit for bit as for gray crops; logits
    against the fp32 oracle fed the same crops; the full pipeline with a color recognizer against the oracle chain built
    the same way."""
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    from keras_ocr_b200.recognition import Recognizer
    from oracle import crnn, imageops, synth
    from oracle.pipeline import OraclePipeline
    w = W.synthetic_crnn_weights(6, color=True)
    assert w["conv_1.kernel"].shape == (3, 3, 3, 64)
    rec = Recognizer(weights=w, build_params={"color": True})
    rec.keep_workspace = True
    rng = np.random.default_rng(23)
    image = np.stack([synth.noise_gray(rng, 240, 320) for _ in range(3)], -1)          # three independent channels
    quads = synth.random_quads(rng, 12, 240, 320, min_side=16, max_side=150)
    img_t = torch.from_numpy(image[None]).to(cuda_device)
    idx = torch.zeros(len(quads), dtype=torch.int32, device=cuda_device)
    crnn_in, crops = rec.warp_device(img_t, torch.from_numpy(quads).to(cuda_device), idx, want_crops=True)
    ref = np.stack([imageops.warp_box(image, q) for q in quads])
    assert crops.shape == ref.shape == (12, 31, 200, 3)
    assert np.array_equal(crops.cpu().numpy(), ref)
    x = torch.empty_like(crnn_in)
    rec.ctx.crops_to_input(crops.data_ptr(), 12, x.data_ptr(), _stream(), color=True)
    assert torch.equal(x, crnn_in)                                  # both routes to the CRNN input agree bit for bit
    texts = rec.recognize_crops(ref)
    logits = rec.tap("logits", (12, 48, 37), torch.float32).cpu()
    with torch.no_grad():
        probs, inter = crnn.crnn_logits(w, ref.astype(np.float32) / 255, return_intermediates=True)
    assert float((logits - inter["logits"]).abs().max()) <= 0.15
    assert texts == crnn.labels_to_text(crnn.ctc_greedy(torch.softmax(logits, -1)))
    assert rec.recognize(ref[0]) == texts[0]                        # single-crop API keeps the colour channels
    with pytest.raises(ValueError):
        Recognizer(weights=w)                                       # a 3-channel conv_1 needs color=True
    cw = W.synthetic_craft_weights(3, textlike=True)
    pages, _ = synth.text_images(seed=21, n=2, h=192, w=384, n_words=4)
    got = Pipeline(detector=Detector(weights=cw), recognizer=rec, scale=2).recognize(pages)
    want = OraclePipeline(cw, w, scale=2, color=True).recognize(pages)
    assert [len(g) for g in got] == [len(r) for r in want] and sum(len(g) for g in got) >= 6


def test_recognize_from_boxes_with_caller_supplied_quads(recognizer):
    """tools.warpBox on quads that are NOT rectangles (reference tools.py:88-95: minimum rotated rectangle first) and on a
    degenerate box (ZeroDivisionError, tools.py:95): the host rectification of ``recognize_from_boxes`` + the CUDA warp
    against the oracle's ``warp_box``, which carries its own restatement of the same rule."""
    from keras_ocr_b200 import tools
    from oracle import imageops, synth
    rng = np.random.default_rng(17)
    gray = synth.noise_gray(rng, 300, 400)
    rects = synth.random_quads(rng, 24, 300, 400, min_side=20, max_side=160)
    quads = rects + rng.uniform(-6, 6, rects.shape).astype(np.float32)          # skewed: no longer rectangles
    fixed = tools.rectify_boxes(quads)
    assert np.abs(fixed - quads).max() > 1.0                                     # really replaced by their rectangles
    assert np.array_equal(tools.rectify_boxes(rects), rects)                     # rectangles pass through bit for bit
    g = torch.from_numpy(gray[None]).to(recognizer.device)
    idx = torch.zeros(len(fixed), dtype=torch.int32, device=recognizer.device)
    _, crops = recognizer.warp_device(g, torch.from_numpy(fixed).to(recognizer.device), idx, want_crops=True)
    crops = crops.cpu().numpy().astype(np.int16)
    ref = np.stack([imageops.warp_box(gray, q) for q in quads]).astype(np.int16)
    diff = np.abs(crops - ref)
    # the two restatements of the rectangle agree to ~1e-5 px; cv2's fixed-point sampler then differs by at most a level
    assert diff.max() <= 2 and (diff > 0).mean() <= 5e-3, (int(diff.max()), float((diff > 0).mean()))
    image = np.repeat(gray[..., None], 3, axis=2)
    texts = recognizer.recognize_from_boxes([image], [quads])
    assert len(texts) == 1 and len(texts[0]) == len(quads)
    with pytest.raises(ZeroDivisionError):
        recognizer.recognize_from_boxes([image], [np.array([[[10, 10], [10.4, 10], [10.4, 60], [10, 60]]], np.float32)])
    with pytest.raises(ZeroDivisionError):
        imageops.warp_box(gray, np.array([[10, 10], [10.4, 10], [10.4, 60], [10, 60]], np.float32))


# ------------------------------------------------------------------------------- API behaviour
def test_reference_api_contract(detector, recognizer):
    rng = np.random.default_rng(0)
    blank = np.full((1, 64, 96, 3), 255, np.uint8)
    boxes = detector.detect(blank)
    assert len(boxes) == 1
    groups = [np.array([])]
    assert recognizer.recognize_from_boxes(blank, groups) == [[]]
    with pytest.raises(AssertionError):                         # recognition.py:501-503
        recognizer.recognize_from_boxes(blank, [])


# ------------------------------------------------------------------------------- end to end
def test_pipeline_recognize_vs_oracle_chain(cuda_device):
    """Whole Pipeline.recognize on rendered pages, fp16 GPU chain vs fp32 oracle chain.
    Tolerance (SURVEY.md 8(c), chained): same box count and order, corners within 2 px at
    detector-input scale (= 1 px in source pixels at scale 2), EVERY decoded string identical
    (decisive recognizer weights: the argmax margins are far above the fp16 noise)."""
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    from keras_ocr_b200.recognition import Recognizer
    from oracle import synth
    from oracle.pipeline import OraclePipeline

    cw, rw = W.synthetic_craft_weights(3, textlike=True), W.synthetic_crnn_weights(2, decisive=True)
    pages, words = synth.text_images(seed=21, n=2, h=192, w=384, n_words=4)
    pipe = Pipeline(detector=Detector(weights=cw), recognizer=Recognizer(weights=rw), scale=2)
    got = pipe.recognize(pages)
    ref = OraclePipeline(cw, rw, scale=2).recognize(pages)
    assert [len(g) for g in got] == [len(r) for r in ref]
    assert sum(len(r) for r in ref) >= 6                        # the synthetic pages really produce word boxes
    worst = 0.0
    for g, r in zip(got, ref):
        for (tg, bg), (tr, br) in zip(g, r):
            assert bg.shape == (4, 2) and bg.dtype == np.float32
            worst = max(worst, _match_quads(bg, br))
    assert worst <= 1.0, worst                                  # source-image pixels (scale 2)
    assert [[t for t, _ in g] for g in got] == [[t for t, _ in r] for r in ref]         # every string
    assert sorted(t for g in got for t, _ in g) == sorted(w for page in words for w in page)   # ... and they are the rendered words
    # same call with a list input and with device-resident sources gives the same result
    again = pipe.recognize([p for p in pages])
    assert [[t for t, _ in g] for g in again] == [[t for t, _ in g] for g in got]
    dev = pipe.recognize(torch.from_numpy(pages).to(cuda_device))
    assert [[t for t, _ in g] for g in dev] == [[t for t, _ in g] for g in got]


def test_blank_page_gives_no_predictions(cuda_device):
    """reference tests/test_pipeline.py:9-12 (blank image -> zero predictions)."""
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    from keras_ocr_b200.recognition import Recognizer
    pipe = Pipeline(detector=Detector(weights=W.synthetic_craft_weights(3, textlike=True)),
                    recognizer=Recognizer(weights=W.synthetic_crnn_weights(2)), scale=2)
    out = pipe.recognize([np.full((256, 256, 3), 255, np.uint8)])
    assert out == [[]]


def test_pipeline_ragged_batch_max_size_and_injection(cuda_device):
    """Different-sized inputs are resized per image (scale capped by max_size for the large one),
    padded with 255 to the batch maximum (pipeline.py:44-57) and the boxes come back in each
    image's own pixels; injecting this package's Detector/Recognizer into a *generic* Pipeline flow
    (duck typing, pipeline.py:18-26) gives the same answer as the all-device flow."""
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    from keras_ocr_b200.recognition import Recognizer
    from oracle import synth
    from oracle.pipeline import OraclePipeline

    cw, rw = W.synthetic_craft_weights(3, textlike=True), W.synthetic_crnn_weights(2)
    rng = np.random.default_rng(33)
    pages = [synth.text_image(rng, 192, 384, 4)[0], synth.text_image(rng, 160, 256, 2)[0], synth.text_image(rng, 256, 640, 4)[0]]
    det, rec = Detector(weights=cw), Recognizer(weights=rw)
    pipe = Pipeline(detector=det, recognizer=rec, scale=2, max_size=1024)     # 640 * 2 > 1024 -> scale 1.6 for page 3
    got = pipe.recognize(pages)
    ref = OraclePipeline(cw, rw, scale=2, max_size=1024).recognize(pages)
    assert [len(g) for g in got] == [len(r) for r in ref]
    for g, r in zip(got, ref):
        for (tg, bg), (tr, br) in zip(g, r):
            assert _match_quads(bg, br) <= 1.0

    class Wrapped:                      # hides the native types -> Pipeline takes its generic (host array) path
        def __init__(self, obj):
            self.obj = obj
        def detect(self, images, **kw):
            return self.obj.detect(images, **kw)
        def recognize_from_boxes(self, images, box_groups, **kw):
            return self.obj.recognize_from_boxes(images, box_groups, **kw)
    generic = Pipeline(detector=Wrapped(det), recognizer=Wrapped(rec), scale=2, max_size=1024).recognize(pages)
    assert [[t for t, _ in g] for g in generic] == [[t for t, _ in g] for g in got]
    for g, r in zip(generic, got):
        for (_, bg), (_, br) in zip(g, r):
            assert np.abs(bg - br).max() <= 1e-3


def test_results_are_bit_reproducible(detector, recognizer):
    """Same inputs -> bit-identical scores and labels on every call (fixed MMA accumulation order)."""
    rng = np.random.default_rng(12)
    img = torch.from_numpy(rng.integers(0, 256, (2, 160, 224, 3), dtype=np.uint8)).to(detector.device)
    a = detector.predict_device(img).clone()
    for _ in range(3):
        assert torch.equal(detector.predict_device(img), a)
    crops = torch.from_numpy(rng.integers(0, 256, (24, 31, 200), dtype=np.uint8)).to(recognizer.device)
    x = torch.empty((24, 200, 31), dtype=torch.float16, device=recognizer.device)
    recognizer.ctx.crops_to_input(crops.data_ptr(), 24, x.data_ptr(), _stream())
    la = recognizer.predict_device(x).clone()
    logits = recognizer.tap("logits", (24, 48, 37), torch.float32).clone()
    for _ in range(3):
        assert torch.equal(recognizer.predict_device(x), la)
        assert torch.equal(recognizer.tap("logits", (24, 48, 37), torch.float32), logits)


def test_crop_result_does_not_depend_on_its_batch(recognizer):
    """A crop's logits are bit-identical whatever batch it is recognised in (kernel configurations that change
    the accumulation order are chosen from the per-image shape only)."""
    rng = np.random.default_rng(3)
    crops = torch.from_numpy(rng.integers(0, 256, (24, 31, 200), dtype=np.uint8)).to(recognizer.device)

    def run(c):
        n = c.shape[0]
        x = torch.empty((n, 200, 31), dtype=torch.float16, device=recognizer.device)
        recognizer.ctx.crops_to_input(c.contiguous().data_ptr(), n, x.data_ptr(), _stream())
        labels = recognizer.predict_device(x).clone()
        return labels, recognizer.tap("logits", (n, 48, 37), torch.float32).clone()

    labels, logits = run(crops)
    for lo, hi in ((0, 10), (10, 24), (3, 4), (5, 18)):
        la, lg = run(crops[lo:hi])
        assert torch.equal(lg, logits[lo:hi]) and torch.equal(la, labels[lo:hi])


def test_pipelined_sub_batches_give_identical_results(cuda_device):
    """Pipeline(inflight=2) splits the batch into software-pipelined sub-batches; every (text, box) must equal
    the unsplit run exactly, for same-size arrays and for ragged lists (whole-batch padding is kept)."""
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    from keras_ocr_b200.recognition import Recognizer
    from oracle import synth
    det = Detector(weights=W.synthetic_craft_weights(3, textlike=True))
    rec = Recognizer(weights=W.synthetic_crnn_weights(2))
    pages, _ = synth.text_images(seed=77, n=9, h=256, w=320, n_words=6)
    ragged = [pages[i][: 256 - 16 * (i % 3), : 320 - 32 * (i % 2)] for i in range(9)]
    for images in (pages, ragged):
        one = Pipeline(detector=det, recognizer=rec, scale=2, inflight=1).recognize(images)
        two = Pipeline(detector=det, recognizer=rec, scale=2, inflight=2).recognize(images)
        assert len(one) == len(two) == 9
        assert sum(len(g) for g in one) > 0
        for ga, gb in zip(one, two):
            assert [t for t, _ in ga] == [t for t, _ in gb]
            assert all(np.array_equal(ba, bb) for (_, ba), (_, bb) in zip(ga, gb))


def test_recognizer_single_crop_api(recognizer):
    """Recognizer.recognize(image) (recognition.py:467-489) == recognize_from_boxes on the fitted crop."""
    import cv2
    from keras_ocr_b200 import tools
    rng = np.random.default_rng(8)
    img = rng.integers(0, 256, (40, 260, 3), dtype=np.uint8)
    text = recognizer.recognize(img)
    fitted = tools.fit(img, 200, 31, cval=0)
    gray = cv2.cvtColor(fitted, cv2.COLOR_RGB2GRAY)
    assert text == recognizer.recognize_crops(gray[None])[0]
    assert isinstance(text, str)


# ------------------------------------------------------------------------------- batch entry points / records
def test_resize_pad_batch_and_fused_gray_bit_exact(ctx, cuda_device):
    """b2o_resize_pad_batch (one launch for equally sized sources, gray fused) == per-image b2o_resize_pad
    followed by b2o_rgb_to_gray, and the gray plane == cv2.cvtColor of the padded batch (oracle)."""
    from oracle import imageops
    rng = np.random.default_rng(5)
    n, hs, ws, hr, wr, hp, wp = 3, 45, 67, 90, 134, 96, 141
    src = torch.from_numpy(rng.integers(0, 256, (n, hs, ws, 3), dtype=np.uint8)).to(cuda_device)
    one = torch.zeros((n, hp, wp, 3), dtype=torch.uint8, device=cuda_device)
    for i in range(n):
        ctx.resize_pad(src[i].data_ptr(), hs, ws, hr, wr, one.data_ptr(), i, hp, wp, _stream())
    gray_one = torch.empty((n, hp, wp), dtype=torch.uint8, device=cuda_device)
    ctx.rgb_to_gray(one.data_ptr(), n, hp, wp, gray_one.data_ptr(), _stream())
    batch = torch.zeros_like(one)
    gray = torch.zeros_like(gray_one)
    ctx.resize_pad_batch(src.data_ptr(), n, hs, ws, hr, wr, batch.data_ptr(), hp, wp, gray.data_ptr(), _stream())
    assert torch.equal(batch, one) and torch.equal(gray, gray_one)
    assert np.array_equal(gray.cpu().numpy(), np.stack([imageops.rgb_to_gray(i) for i in one.cpu().numpy()]))
    again = torch.zeros_like(one)                                   # gray is optional
    ctx.resize_pad_batch(src.data_ptr(), n, hs, ws, hr, wr, again.data_ptr(), hp, wp, None, _stream())
    assert torch.equal(again, one)
    with pytest.raises(_lib.B2OError):
        ctx.resize_pad_batch(src.data_ptr(), n, hs, ws, hr, wr, again.data_ptr(), hr - 1, wp, None, _stream())


def test_compact_boxes_and_pack_records_match_host_bookkeeping(ctx, cuda_device):
    """b2o_compact_boxes == the running-offset bookkeeping of recognize_from_boxes (recognition.py:511-521);
    b2o_pack_records == distributed.pack_records (the host packer, itself round-trip tested on the CPU), bit for
    bit, including clamped counts, empty images and the padding rows of a short shard."""
    from keras_ocr_b200 import distributed as D
    rng = np.random.default_rng(9)
    n, m, rows, rec_boxes = 5, 8, 7, 6
    counts = np.array([3, 0, 8, 11, 1], np.int32)                    # 11 > m: the table holds only 8
    held = np.minimum(counts, m)
    boxes = rng.uniform(0, 3000, (n, m, 4, 2)).astype(np.float32)
    total = int(held.sum())
    labels = rng.integers(-1, 37, (total, 48)).astype(np.int32)
    inv = np.array([0.5, 1.0, 1 / 1.6, 0.5, 1 / 3], np.float32)
    b_t, c_t = torch.from_numpy(boxes).to(cuda_device), torch.from_numpy(counts).to(cuda_device)
    flat = torch.zeros((n * m, 4, 2), dtype=torch.float32, device=cuda_device)
    index = torch.full((n * m,), -7, dtype=torch.int32, device=cuda_device)
    ctx.compact_boxes(b_t.data_ptr(), c_t.data_ptr(), n, m, flat.data_ptr(), index.data_ptr(), _stream())
    assert np.array_equal(flat.cpu().numpy()[:total], np.concatenate([boxes[i, :held[i]] for i in range(n)]))
    assert np.array_equal(index.cpu().numpy()[:total], np.repeat(np.arange(n), held))
    assert (index.cpu().numpy()[total:] == -7).all()                 # nothing written past the dense list

    rec = torch.zeros((rows, ctx.record_floats(rec_boxes)), dtype=torch.float32, device=cuda_device)
    labels_t, inv_t = torch.from_numpy(labels).to(cuda_device), torch.from_numpy(inv).to(cuda_device)
    ctx.pack_records(b_t.data_ptr(), c_t.data_ptr(), labels_t.data_ptr(), inv_t.data_ptr(), n, m, rows, rec_boxes,
                     rec.data_ptr(), _stream())
    scaled = [boxes[i, :held[i]] * inv[i] for i in range(n)]         # tools.adjust_boxes: float32 * float32
    expect = D.pack_records(held, scaled, labels.astype(np.int8), rows, rec_boxes)
    assert np.array_equal(rec.cpu().numpy().view(np.uint32), expect.numpy().view(np.uint32))
    with pytest.raises(D.RecordOverflow):                            # images 2 and 3 hold 8 words, a record 6: never silent
        D.unpack_blocks([rec], rec_boxes)
    got_counts, got_boxes, got_labels = D.unpack_blocks([rec], rec_boxes, strict=False)
    assert got_counts.tolist() == np.minimum(held, rec_boxes).tolist()


def test_recognize_records_equals_recognize(cuda_device):
    """Pipeline.recognize_records (results stay on the device as records; the multi-GPU payload) decodes to exactly
    what Pipeline.recognize returns: same words, boxes bit-identical, padding rows ignored."""
    from keras_ocr_b200 import distributed as D, recognition
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    from keras_ocr_b200.recognition import Recognizer
    from oracle import synth
    pipe = Pipeline(detector=Detector(weights=W.synthetic_craft_weights(3, textlike=True)),
                    recognizer=Recognizer(weights=W.synthetic_crnn_weights(2)), scale=2, max_size=600)
    pages, _ = synth.text_images(seed=5, n=3, h=192, w=384, n_words=4)      # 384 * 2 > 600: scale 1.5625
    pages = np.concatenate([pages, np.full((1, 192, 384, 3), 255, np.uint8)])      # plus a blank page
    ref = pipe.recognize(pages)
    assert sum(len(g) for g in ref) >= 6 and ref[3] == []
    rec = pipe.recognize_records(pages, rows=6, rec_boxes=16)
    assert rec.is_cuda and rec.shape == (6, pipe.detector.ctx.record_floats(16))
    counts, boxes, labels = D.unpack_blocks([rec], 16)
    assert counts.tolist() == [len(g) for g in ref]
    texts = recognition.labels_to_text(labels, pipe.recognizer.alphabet)
    assert texts == [t for g in ref for t, _ in g]
    assert np.array_equal(boxes, np.concatenate([np.stack([b for _, b in g]) for g in ref if g]))
    # the one-process form of the sharded call goes through the same records
    assert [[t for t, _ in g] for g in D.recognize_sharded(pipe, pages, max_boxes=16)] == [[t for t, _ in g] for g in ref]
    # a record too small for a page is never silent: RecordOverflow names the image; "auto" sizes the records from the counts
    with pytest.raises(D.RecordOverflow):
        D.recognize_sharded(pipe, pages, max_boxes=2)
    auto = D.recognize_sharded(pipe, pages, max_boxes="auto")
    assert [[t for t, _ in g] for g in auto] == [[t for t, _ in g] for g in ref]
    assert all(np.array_equal(a, b) for ga, gb in zip(auto, ref) for (_, a), (_, b) in zip(ga, gb))


# ------------------------------------------------------------------------------- BASELINE.json sizes: properties
def test_full_size_page_results_do_not_depend_on_the_batch(cuda_device):
    """configs[3] geometry (768x768 sources, scale 2 -> 1536x1536 detector input, 32 words per page) on a small
    batch: every rendered word is found, and a page's (word, box) list is bit-identical whether the page is
    recognised alone or inside a batch (images are independent, pipeline.py:28-75)."""
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    from keras_ocr_b200.recognition import Recognizer
    from oracle import synth
    pipe = Pipeline(detector=Detector(weights=W.synthetic_craft_weights(3, textlike=True)),
                    recognizer=Recognizer(weights=W.synthetic_crnn_weights(2)), scale=2)
    pages, _ = synth.text_images(seed=1000, n=3, h=768, w=768, n_words=32)
    together = pipe.recognize(pages)
    assert [len(g) for g in together] == [32, 32, 32] or min(len(g) for g in together) >= 30
    for i in (0, 2):
        alone = pipe.recognize(pages[i:i + 1])[0]
        assert [t for t, _ in alone] == [t for t, _ in together[i]]
        assert all(np.array_equal(a, b) for (_, a), (_, b) in zip(alone, together[i]))


def test_craft_batch8_768_scores_do_not_depend_on_the_batch(detector):
    """configs[1] (CRAFT only, batch 8 at 768x768): image i of the batch gives bit-identical score maps to image i
    alone, and the maps are finite."""
    rng = np.random.default_rng(4)
    img = torch.from_numpy(rng.integers(0, 256, (8, 768, 768, 3), dtype=np.uint8)).to(detector.device)
    scores = detector.predict_device(img).clone()
    assert scores.shape == (8, 384, 384, 2) and bool(torch.isfinite(scores).all())
    for i in (0, 5, 7):
        assert torch.equal(detector.predict_device(img[i:i + 1].contiguous())[0], scores[i])


def test_crnn_batch256_labels_do_not_depend_on_the_batch(recognizer):
    """configs[2] (CRNN only, 256 crops 31x200 + greedy CTC): labels of a crop are the same in the batch of 256
    and in a sub-batch; rows are -1 padded after the decoded prefix and never contain the blank."""
    rng = np.random.default_rng(6)
    crops = torch.from_numpy(rng.integers(0, 256, (256, 31, 200), dtype=np.uint8)).to(recognizer.device)

    def run(c):
        x = torch.empty((c.shape[0], 200, 31), dtype=torch.float16, device=recognizer.device)
        recognizer.ctx.crops_to_input(c.contiguous().data_ptr(), c.shape[0], x.data_ptr(), _stream())
        return recognizer.predict_device(x).clone()

    labels = run(crops)
    assert labels.shape == (256, 48)
    assert torch.equal(run(crops[100:133]), labels[100:133])
    lab = labels.cpu().numpy()
    assert ((lab >= -1) & (lab < 36)).all()
    pad = lab == -1
    assert (pad[:, :-1] <= pad[:, 1:]).all()                        # once padding starts it continues


def test_cta_pairs_give_bit_identical_results(cuda_device, monkeypatch):
    """The CTA-pair convolution path (2-CTA clusters sharing B tiles by TMA multicast, B2O_TC_PAIR=1) and the single-CTA
    path (B2O_TC_PAIR=0, the default; read at context creation) add every output's terms in the same order: score maps and CRNN logits are bit-identical, for
    even and odd numbers of tile columns (the odd one leaves the second CTA of the last pair on a dummy tile)."""
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.recognition import Recognizer
    cw, rw = W.synthetic_craft_weights(3), W.synthetic_crnn_weights(2)

    def build(pair):
        monkeypatch.setenv("B2O_TC_PAIR", "1" if pair else "0")
        det, rec = Detector(weights=cw), Recognizer(weights=rw)
        rec.keep_workspace = True
        return det, rec

    (det1, rec1), (det0, rec0) = build(True), build(False)
    rng = np.random.default_rng(2)
    for h, w in ((160, 224), (144, 200)):                 # 200 / 8 = 25 tile columns at full resolution
        img = torch.from_numpy(rng.integers(0, 256, (2, h, w, 3), dtype=np.uint8)).to(cuda_device)
        assert torch.equal(det1.predict_device(img), det0.predict_device(img))
    crops = torch.from_numpy(rng.integers(0, 256, (9, 31, 200), dtype=np.uint8)).to(cuda_device)
    logits = []
    for rec in (rec1, rec0):
        x = torch.empty((9, 200, 31), dtype=torch.float16, device=cuda_device)
        rec.ctx.crops_to_input(crops.data_ptr(), 9, x.data_ptr(), _stream())
        labels = rec.predict_device(x).clone()
        logits.append((labels, rec.tap("logits", (9, 48, 37), torch.float32).clone()))
    assert torch.equal(logits[0][0], logits[1][0]) and torch.equal(logits[0][1], logits[1][1])


def test_decoder_commute_matches_explicit_upsample(cuda_device, monkeypatch, golden_dir):
    """Decoder glue (detection.py:290-309, 380-390): with B2O_UPCONV_COMMUTE=1 the bilinear 2x upsampling is commuted behind
    the decoder half of each 1x1 ``upconvN.conv.0`` (low-resolution GEMM + upsample-add in the full-resolution layer's
    epilogue); the default runs UpsampleLike + the concat-wide convolution as the reference graph does.  The two are the
    same function up to fp16 rounding of one intermediate: score maps agree to 5e-3 of the range, and BOTH stay within
    the 2e-2 bound against the reference's own output (golden "even" case, whose sizes are multiples of 16)."""
    from keras_ocr_b200.detection import Detector
    cw = W.synthetic_craft_weights(3)
    monkeypatch.setenv("B2O_UPCONV_COMMUTE", "1")
    commuted = Detector(weights=cw)
    monkeypatch.delenv("B2O_UPCONV_COMMUTE")
    explicit = Detector(weights=cw)
    rng = np.random.default_rng(7)
    for h, w in ((160, 224), (768, 768), (144, 200)):          # 144 x 200: 200 / 16 is odd -> one level falls back
        img = torch.from_numpy(rng.integers(0, 256, (2, h, w, 3), dtype=np.uint8)).to(cuda_device)
        a, b = commuted.predict_device(img).clone(), explicit.predict_device(img).clone()
        span = max(float(b.abs().max()), 1.0)
        assert float((a - b).abs().max()) / span <= 5e-3, (h, w)
    g = np.load(os.path.join(golden_dir, "craft.npz"))
    img = torch.from_numpy(g["craft_even_image"]).to(cuda_device)
    ref = g["craft_even_scores"]
    for det in (commuted, explicit):
        err = np.abs(det.predict_device(img).cpu().numpy() - ref).max() / max(np.abs(ref).max(), 1.0)
        assert err <= 2e-2, err


@pytest.mark.parametrize("switch", [("B2O_TC_PAIR", "2"), ("B2O_FUSED_TAIL", "0"), ("B2O_TC_AFF", "smem"), ("B2O_GLUE", "v1")],
                         ids=["generic_pairs", "separate_head_tail", "epilogue_constants_in_smem", "round1_upsample2x"])
def test_conv_variants_are_bit_identical(cuda_device, monkeypatch, switch):
    """Kernel variants that keep the MMA / fmaf order of the default path must not change a bit of the CRAFT score
    maps or the CRNN logits:  B2O_TC_PAIR=2 -- CTA pairs on the generic tiles too;  B2O_FUSED_TAIL=0 -- conv_cls.6 / conv_cls.8 as the separate head_tail_kernel instead of conv_cls.4's epilogue;
    B2O_TC_AFF=smem -- the per-channel epilogue constants staged in shared memory / read from global memory (round 1)
    instead of the kernel-parameter constant bank;  B2O_GLUE=v1 -- the round-1 2x upsampling kernel (64-bit index chain, each output
    pixel blending its four taps on its own) instead of the one that shares a quad column's two horizontal blends.
    Sizes: odd tile columns (200 / 8 = 25), several tiles per CTA, and the 768 x 768 case of BASELINE configs[1]."""
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.recognition import Recognizer
    cw, rw = W.synthetic_craft_weights(3), W.synthetic_crnn_weights(2)

    def build(on):
        if on:
            monkeypatch.setenv(*switch)
        else:
            monkeypatch.delenv(switch[0], raising=False)
        det, rec = Detector(weights=cw), Recognizer(weights=rw)
        rec.keep_workspace = True
        return det, rec

    (det1, rec1), (det0, rec0) = build(True), build(False)
    rng = np.random.default_rng(2)
    for h, w in ((160, 224), (144, 200), (768, 768)):
        img = torch.from_numpy(rng.integers(0, 256, (2, h, w, 3), dtype=np.uint8)).to(cuda_device)
        assert torch.equal(det1.predict_device(img), det0.predict_device(img)), (h, w)
    crops = torch.from_numpy(rng.integers(0, 256, (9, 31, 200), dtype=np.uint8)).to(cuda_device)
    got = []
    for rec in (rec1, rec0):
        x = torch.empty((9, 200, 31), dtype=torch.float16, device=cuda_device)
        rec.ctx.crops_to_input(crops.data_ptr(), 9, x.data_ptr(), _stream())
        labels = rec.predict_device(x).clone()
        got.append((labels, rec.tap("logits", (9, 48, 37), torch.float32).clone()))
    assert torch.equal(got[0][0], got[1][0]) and torch.equal(got[0][1], got[1][1])
