"""Train the whole CRNN recognizer on rendered words -- TEST INFRASTRUCTURE, meant to run where torch has a GPU
(``python -m oracle.train_crnn_full`` on a CUDA machine; a few minutes on one GPU, PyTorch/cuDNN doing the training arithmetic).

(An earlier fixture fitted only the head on frozen random features: it memorised its pages and its strings changed when a
box moved by a pixel.)  This script trains every layer of the reference architecture (``build_model``,
recognition.py:187-350, restated with torch.nn modules in exactly ``oracle/crnn.py``'s arithmetic -- the export is checked
against ``oracle.crnn.crnn_logits``) with CTC loss on

* synthetic word crops made on the fly: a random word rendered as ``oracle.synth.text_image`` renders it (cv2 Hershey
  font, thickness 2, anti-aliased, dark colour on white), up-scaled 2x like ``tools.resize_image``, converted to gray and cut
  out by ``imageops.warp_box`` from a box with the margins the oracle detector leaves around a word (statistics measured
  on oracle-pipeline boxes: 0.30 / 0.26 / 0.40 / 0.23 of the glyph height left / right / top / bottom) plus jitter;
* the real crops the ORACLE pipeline cuts out of the test / bench pages (``oracle/_train_data/real_crops.npz``, written by
  ``python -m oracle.word_crops``), including box-jittered copies; four pages are held out to measure generalisation.

The result is a small model that actually READS the Hershey font: it generalises to pages it has not seen, and its strings
do not change when a box moves by a pixel -- which is what lets the chained parity test assert every string.
Writes ``keras-ocr_b200/data/crnn_hershey.npz`` (all CRNN tensors, Keras names / layouts, float16).
"""
import os
import sys
import time

import cv2
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import crnn, imageops, synth                      # noqa: E402

OUT = os.environ.get("B2O_TRAIN_OUT", os.path.join(ROOT, "keras-ocr_b200", "data", "crnn_hershey.npz"))
REAL = os.path.join(ROOT, "oracle", "_train_data", "real_crops.npz")
MARGIN_MEAN = np.array([0.30, 0.26, 0.40, 0.23])               # left, right, top, bottom, in glyph heights (measured)
MARGIN_STD = np.array([0.11, 0.12, 0.18, 0.22])


def synth_crop(seed):
    """One (crop uint8 31x200, word) rendered and cut as the oracle pipeline would."""
    rng = np.random.default_rng(seed)
    word = synth.random_word(rng)
    cell_w, cell_h = float(rng.uniform(120, 260)), float(rng.uniform(60, 100))
    (tw, th), _ = cv2.getTextSize(word, cv2.FONT_HERSHEY_SIMPLEX, 0.9, 2)
    scale = 0.9 * min(0.8 * cell_w / tw, 0.45 * cell_h / th)
    (tw, th), base = cv2.getTextSize(word, cv2.FONT_HERSHEY_SIMPLEX, scale, 2)
    pad = 48
    img = np.full((th + base + 2 * pad, tw + 2 * pad, 3), 255, np.uint8)
    colour = tuple(int(c) for c in rng.integers(0, 90, 3))
    cv2.putText(img, word, (pad, pad + th), cv2.FONT_HERSHEY_SIMPLEX, scale, colour, 2, cv2.LINE_AA)
    big = cv2.resize(img, dsize=(img.shape[1] * 2, img.shape[0] * 2))      # tools.resize_image at scale 2
    gray = imageops.rgb_to_gray(big)
    x0, y0, x1, y1 = 2.0 * pad, 2.0 * pad, 2.0 * (pad + tw), 2.0 * (pad + th + base)
    gh = y1 - y0
    m = np.maximum(rng.normal(MARGIN_MEAN, MARGIN_STD), -0.05) * gh
    box = np.array([[x0 - m[0], y0 - m[2]], [x1 + m[1], y0 - m[2]], [x1 + m[1], y1 + m[3]], [x0 - m[0], y1 + m[3]]], np.float32)
    box += rng.uniform(-2.0, 2.0, (4, 2)).astype(np.float32)
    return imageops.warp_box(gray, box), word


class TorchCRNN(nn.Module):
    """oracle/crnn.py with trainable torch.nn layers (same tensor layouts: NCHW with H = 200 time steps, W = 31)."""

    def __init__(self, classes=37):
        super().__init__()
        chans = [(1, 64), (64, 128), (128, 256), (256, 256), (256, 512), (512, 512), (512, 512)]
        self.convs = nn.ModuleList([nn.Conv2d(i, o, 3, padding=1) for i, o in chans])
        self.bns = nn.ModuleDict({k: nn.BatchNorm2d(c, eps=crnn.KERAS_BN_EPS, momentum=0.01) for k, c in (("3", 256), ("5", 512), ("7", 512))})
        self.stn_a, self.stn_b = nn.Conv2d(512, 16, 5, padding=2), nn.Conv2d(16, 32, 5, padding=2)
        self.stn_d1, self.stn_d2 = nn.Linear(11200, 64), nn.Linear(64, 6)
        with torch.no_grad():                                   # the transformer starts (and is kept) at the identity
            self.stn_d2.weight.zero_()
            self.stn_d2.bias.copy_(torch.tensor([1.0, 0, 0, 0, 1, 0]))
        for p in self.stn_d2.parameters():
            p.requires_grad_(False)
        self.fc9 = nn.Linear(3584, 128)
        self.l10, self.l10b = nn.LSTM(128, 128, batch_first=True), nn.LSTM(128, 128, batch_first=True)
        self.l11, self.l11b = nn.LSTM(128, 128, batch_first=True), nn.LSTM(128, 128, batch_first=True)
        self.fc12 = nn.Linear(256, classes)

    def forward(self, crops):                                  # crops: (B,31,200) float in [0,1]
        x = torch.flip(crops.permute(0, 2, 1), [2]).unsqueeze(1)
        for i, conv in enumerate(self.convs, 1):
            x = F.relu(conv(x))
            if str(i) in self.bns:
                x = self.bns[str(i)](x)
                if i in (3, 5):
                    x = F.max_pool2d(x, 2, 2)
        feat = x.float()
        y = F.relu(self.stn_b(F.relu(self.stn_a(feat))))
        y = y.permute(0, 2, 3, 1).reshape(y.shape[0], -1)
        theta = self.stn_d2(F.relu(self.stn_d1(y)))
        warped = crnn.stn_sample(feat.permute(0, 2, 3, 1).contiguous(), theta)
        seq = F.relu(self.fc9(warped.reshape(warped.shape[0], warped.shape[1], -1)))
        l1 = self.l10(seq)[0] + self.l10b(torch.flip(seq, [1]))[0]
        l2 = torch.cat([self.l11(l1)[0], self.l11b(torch.flip(l1, [1]))[0]], -1)
        return self.fc12(l2)[:, crnn.STEPS_TO_DISCARD:]

    def export(self):
        out = {}
        for i, conv in enumerate(self.convs, 1):
            out[f"conv_{i}.kernel"], out[f"conv_{i}.bias"] = conv.weight.permute(2, 3, 1, 0), conv.bias
        for k, bn in self.bns.items():
            out[f"bn_{k}.gamma"], out[f"bn_{k}.beta"] = bn.weight, bn.bias
            out[f"bn_{k}.moving_mean"], out[f"bn_{k}.moving_variance"] = bn.running_mean, bn.running_var
        for name, conv in (("stn.conv_a", self.stn_a), ("stn.conv_b", self.stn_b)):
            out[name + ".kernel"], out[name + ".bias"] = conv.weight.permute(2, 3, 1, 0), conv.bias
        for name, lin in (("stn.dense_a", self.stn_d1), ("stn.dense_b", self.stn_d2), ("fc_9", self.fc9), ("fc_12", self.fc12)):
            out[name + ".kernel"], out[name + ".bias"] = lin.weight.T, lin.bias
        for name, m in (("lstm_10", self.l10), ("lstm_10_back", self.l10b), ("lstm_11", self.l11), ("lstm_11_back", self.l11b)):
            out[name + ".kernel"], out[name + ".recurrent_kernel"] = m.weight_ih_l0.T, m.weight_hh_l0.T
            out[name + ".bias"] = m.bias_ih_l0 + m.bias_hh_l0
        return {k: v.detach().float().cpu().contiguous().numpy().astype(np.float16) for k, v in out.items()}


def encode(words):
    flat = torch.tensor([crnn.ALPHABET.index(c) for wd in words for c in wd], dtype=torch.long)
    return flat, torch.tensor([len(wd) for wd in words], dtype=torch.long)


def texts_of(model, crops, device, batch=256):
    out = []
    model.eval()
    with torch.no_grad():
        for i in range(0, len(crops), batch):
            x = torch.from_numpy(crops[i:i + batch].astype(np.float32) / 255).to(device)
            out += crnn.labels_to_text(crnn.ctc_greedy(torch.softmax(model(x).float().cpu(), -1)))
    model.train()
    return out


def main():
    import multiprocessing as mp
    device = torch.device("cuda" if torch.cuda.is_available() else "cpu")
    steps = int(os.environ.get("B2O_TRAIN_STEPS", 6000))
    n_synth = int(os.environ.get("B2O_TRAIN_SYNTH", 120000))
    torch.manual_seed(0)
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cuda.matmul.allow_tf32 = True
    t0 = time.time()
    real = np.load(REAL, allow_pickle=True)
    real_crops, real_labels = real["crops"], [str(x) for x in real["labels"]]
    hold_crops, hold_labels = real["hold_crops"], [str(x) for x in real["hold_labels"]]
    with mp.Pool(min(48, os.cpu_count() or 8)) as pool:
        made = pool.map(synth_crop, range(10_000_000, 10_000_000 + n_synth), chunksize=256)
    syn_crops = np.stack([m[0] for m in made])
    syn_words = [m[1] for m in made]
    val_crops, val_words = syn_crops[-2000:], syn_words[-2000:]
    syn_crops, syn_words = syn_crops[:-2000], syn_words[:-2000]
    print(f"[{time.time() - t0:5.0f}s] {len(syn_crops)} synthetic + {len(real_crops)} real crops, device {device}", flush=True)

    model = TorchCRNN().to(device)
    opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-3, weight_decay=1e-4)
    sched = torch.optim.lr_scheduler.OneCycleLR(opt, max_lr=2e-3, total_steps=steps, pct_start=0.1)
    rng = np.random.default_rng(1)
    bs = 128
    for step in range(steps):
        k = bs // 2
        ia, ib = rng.integers(0, len(syn_crops), bs - k), rng.integers(0, len(real_crops), k)
        crops = np.concatenate([syn_crops[ia], real_crops[ib]]).astype(np.float32)
        crops += rng.normal(0, 2.0, crops.shape).astype(np.float32)                     # sensor-like noise, in gray levels
        words = [syn_words[i] for i in ia] + [real_labels[i] for i in ib]
        x = torch.from_numpy(np.clip(crops, 0, 255) / 255).to(device)
        with torch.autocast(device_type=device.type, dtype=torch.bfloat16, enabled=device.type == "cuda"):
            logits = model(x)
        lp = F.log_softmax(logits.float(), -1).permute(1, 0, 2)
        tgt, tl = encode(words)
        loss = F.ctc_loss(lp, tgt, torch.full((bs,), lp.shape[0], dtype=torch.long), tl, blank=crnn.BLANK, zero_infinity=True)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        nn.utils.clip_grad_norm_(model.parameters(), 5.0)
        opt.step(); sched.step()
        if step % 250 == 249 or step == steps - 1:
            va = np.mean([a == b for a, b in zip(texts_of(model, val_crops, device), val_words)])
            ha = np.mean([a == b for a, b in zip(texts_of(model, hold_crops, device), hold_labels)])
            ra = np.mean([a == b for a, b in zip(texts_of(model, real_crops[:2000], device), real_labels[:2000])])
            print(f"[{time.time() - t0:5.0f}s] step {step + 1}: loss {float(loss):.4f}  synthetic val {va:.4f}  real train {ra:.4f}  "
                  f"real hold-out pages {ha:.4f}", flush=True)

    exported = model.export()
    weights = {k: v.astype(np.float32) for k, v in exported.items()}
    with torch.no_grad():                                        # the export is the oracle's network
        mine = model.eval().float()(torch.from_numpy(hold_crops[:16].astype(np.float32) / 255).to(device)).cpu()
        _, inter = crnn.crnn_logits(weights, hold_crops[:16].astype(np.float32) / 255, return_intermediates=True)
    print("export vs oracle.crnn logits: max|diff|", float((mine - inter["logits"]).abs().max()), "of", float(inter["logits"].abs().max()))
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    np.savez(OUT, **exported)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
