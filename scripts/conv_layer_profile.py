"""conv_layer_profile.py -- time of every ``conv_tc_kernel`` launch of one bench.py step, layer by layer.

    python scripts/conv_layer_profile.py OUT_DIR [--warmup W]

Runs the workload of bench.py (its 32 seeded pages, weights and ``Pipeline(scale=2, max_size=2048)``): W warm-up
steps, one step under ``torch.profiler`` with CUDA activity (its trace goes to OUT_DIR), then a few steps without the
profiler for the step time.  The trace's ``conv_tc_kernel`` launches, in launch order, are matched to the layer
sequence of ``b2o_craft_forward`` and ``b2o_crnn_forward``; for each layer the script prints its shape, the kernel
instance, the time, the algorithmic FLOPs (2 * pixels * taps * cin * cout with the reference's channel counts, as
``launch()`` in csrc/conv_tc.cu counts them) and the rate, then totals for CRAFT, the CRNN and the step, and the share of
the step spent outside ``conv_tc_kernel``.  The same data goes to OUT_DIR/conv_layer_profile.json, with the card's name,
power limit and clocks (read-only nvidia-smi query).  Only the public Python API is used.
"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# b2o_craft_forward's tensor-core launches: (name, resolution divisor, ksize, cin, cout).  The stem runs as a 16-channel
# layer but counts its 3 real input channels; conv_cls.6 / conv_cls.8 ride in conv_cls.4's epilogue (not counted).
CRAFT_LAYERS = [
    ("stem16 (basenet.slice1.0)", 1, 3, 3, 64),
    ("basenet.slice1.3 +pool", 1, 3, 64, 64),
    ("basenet.slice1.7", 2, 3, 64, 128),
    ("basenet.slice1.10 +pool", 2, 3, 128, 128),
    ("basenet.slice2.14", 4, 3, 128, 256),
    ("basenet.slice2.17", 4, 3, 256, 256),
    ("basenet.slice3.20 +pool", 4, 3, 256, 256),
    ("basenet.slice3.24", 8, 3, 256, 512),
    ("basenet.slice3.27", 8, 3, 512, 512),
    ("basenet.slice4.30 +pool", 8, 3, 512, 512),
    ("basenet.slice4.34", 16, 3, 512, 512),
    ("basenet.slice4.37", 16, 3, 512, 512),
    ("basenet.slice5.1 (dil 6)", 16, 3, 512, 1024),
    ("basenet.slice5.2", 16, 1, 1024, 1024),
    ("upconv1.conv.0", 16, 1, 1536, 512),
    ("upconv1.conv.3", 16, 3, 512, 256),
    ("upconv2.conv.0", 8, 1, 768, 256),
    ("upconv2.conv.3", 8, 3, 256, 128),
    ("upconv3.conv.0", 4, 1, 384, 128),
    ("upconv3.conv.3", 4, 3, 128, 64),
    ("upconv4.conv.0", 2, 1, 192, 64),
    ("upconv4.conv.3", 2, 3, 64, 32),
    ("conv_cls.0", 2, 3, 32, 32),
    ("conv_cls.2", 2, 3, 32, 32),
    ("conv_cls.4 +tail", 2, 3, 32, 16),
]


def crnn_layers(b):
    """b2o_crnn_forward's tensor-core launches for b crops: (name, (n, h, w), ksize, cin, cout)."""
    return [
        ("conv_2", (b, 200, 31), 3, 64, 128),
        ("conv_3 +pool", (b, 200, 31), 3, 128, 256),
        ("conv_4", (b, 100, 15), 3, 256, 256),
        ("conv_5 +pool", (b, 100, 15), 3, 256, 512),
        ("conv_6", (b, 50, 7), 3, 512, 512),
        ("conv_7", (b, 50, 7), 3, 512, 512),
        ("stn.conv_a (as 1x1 GEMM)", (b, 50, 7), 1, 512, 400),
        ("stn.conv_b", (b, 50, 7), 5, 16, 32),
        ("stn.dense_a", (1, 1, b), 1, 11200, 64),
        ("fc_9", (1, 1, b * 50), 1, 3584, 128),
        ("lstm_in_1 (fp32 out)", (1, 1, b * 50), 1, 128, 1024),
        ("lstm_in_2 (fp32 out)", (1, 1, b * 50), 1, 128, 1024),
    ]


def card_info(device_index):
    """Name, power limit (W), max and current SM clock (MHz) of the card (read-only nvidia-smi query)."""
    fields = ["name", "power.limit", "clocks.max.sm", "clocks.sm"]
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={','.join(fields)}", "--format=csv,noheader,nounits",
                              "-i", str(device_index)], capture_output=True, text=True, timeout=30).stdout.strip()
        vals = [v.strip() for v in out.split(",")]
        return {"gpu": vals[0], "power_limit_w": float(vals[1]), "sm_max_mhz": float(vals[2]), "sm_mhz": float(vals[3])}
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return {"gpu": None, "power_limit_w": None, "sm_max_mhz": None, "sm_mhz": None}


def kernel_events(trace_path):
    """GPU kernel events of a chrome trace, in start order: [(name, start_us, dur_us)]."""
    with open(trace_path) as f:
        trace = json.load(f)
    ev = [(e["name"], float(e["ts"]), float(e["dur"])) for e in trace.get("traceEvents", [])
          if e.get("cat") == "kernel" and "dur" in e]
    return sorted(ev, key=lambda e: e[1])


def instance(name):
    m = re.search(r"conv_tc_kernel<([^>]*)>", name)
    return m.group(1).replace(" ", "") if m else name


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("out_dir")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5, help="unprofiled steps timed for the step time")
    args = ap.parse_args()
    os.makedirs(args.out_dir, exist_ok=True)

    import torch

    import bench
    from keras_ocr_b200 import weights as W
    from keras_ocr_b200.detection import Detector
    from keras_ocr_b200.pipeline import Pipeline
    from keras_ocr_b200.recognition import Recognizer

    assert torch.cuda.is_available(), "conv_layer_profile.py needs a CUDA device"
    device = torch.device("cuda", 0)
    det = Detector(weights=W.synthetic_craft_weights(3, textlike=True), device=0)
    rec = Recognizer(weights=W.synthetic_crnn_weights(2, decisive=True), device=0)
    pipe = Pipeline(detector=det, recognizer=rec, scale=bench.SCALE, max_size=2048)
    pages = torch.from_numpy(bench.make_pages(0)).to(device)
    n_pages, hp, wp, _ = pipe.prepare_device(pages)[0].shape     # the detector's (resized, padded) input

    for _ in range(max(args.warmup, 1)):
        result = pipe.recognize(pages)
    crops = sum(len(g) for g in result)
    torch.cuda.synchronize()

    # the conv kernel's own FLOP count of one step (b2o_profile_*), to check the layer table against
    det.ctx.profile_enable(1); rec.ctx.profile_enable(1)
    pipe.recognize(pages)
    torch.cuda.synchronize()
    _, flop_d, n_d = det.ctx.profile_read()
    _, flop_r, n_r = rec.ctx.profile_read()
    det.ctx.profile_enable(0); rec.ctx.profile_enable(0)

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        pipe.recognize(pages)
        torch.cuda.synchronize()
    trace_path = os.path.join(args.out_dir, "step.pt.trace.json")
    prof.export_chrome_trace(trace_path)

    step_ms = []
    for _ in range(args.steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        pipe.recognize(pages)
        e1.record()
        torch.cuda.synchronize()
        step_ms.append(e0.elapsed_time(e1))
    card = card_info(0)

    kernels = kernel_events(trace_path)
    conv = [k for k in kernels if "conv_tc_kernel" in k[0]]
    table = [(name, (n_pages, hp // div, wp // div), k, cin, cout) for name, div, k, cin, cout in CRAFT_LAYERS]
    n_craft = len(table)
    table += crnn_layers(crops)
    matched = len(conv) == len(table) and n_d == n_craft and n_r == len(table) - n_craft
    rows = []
    for i, (kname, _, dur) in enumerate(conv):
        row = {"launch": i, "instance": instance(kname), "ms": dur / 1e3}
        if matched:
            name, (n, h, w), k, cin, cout = table[i]
            flop = 2.0 * n * h * w * k * k * cin * cout
            row.update({"net": "craft" if i < n_craft else "crnn", "layer": name, "shape": [n, h, w, cin, cout],
                        "ksize": k, "flop": flop, "tflops": flop / (dur * 1e-6) / 1e12})
        rows.append(row)

    def total(sel):
        ms = sum(r["ms"] for r in sel)
        fl = sum(r.get("flop", 0.0) for r in sel)
        return {"launches": len(sel), "ms": ms, "flop": fl, "tflops": fl / (ms * 1e-3) / 1e12 if ms > 0 else None}

    span_ms = (kernels[-1][1] + kernels[-1][2] - kernels[0][1]) / 1e3 if kernels else 0.0
    step = statistics.median(step_ms)
    out = {
        "card": card, "workload": bench.workload_config(1)["workload"], "detector_input": [n_pages, hp, wp],
        "crops": crops, "matched_to_layers": matched,
        "layer_flop_sum": sum(r.get("flop", 0.0) for r in rows), "kernel_flop_count": flop_d + flop_r,
        "layers": rows,
        "craft": total([r for r in rows if r.get("net") == "craft"]),
        "crnn": total([r for r in rows if r.get("net") == "crnn"]),
        "conv_total": total(rows),
        "step_ms_unprofiled_median": step, "step_ms_unprofiled": step_ms,
        "profiled_step_gpu_span_ms": span_ms,
        "kernels_in_profiled_step": len(kernels),
        "share_outside_conv_tc": 1.0 - total(rows)["ms"] / step,
        "trace": os.path.basename(trace_path),
    }
    with open(os.path.join(args.out_dir, "conv_layer_profile.json"), "w") as f:
        json.dump(out, f, indent=1)

    print(f"{card['gpu']}, power limit {card['power_limit_w']} W, SM clock {card['sm_mhz']} of {card['sm_max_mhz']} MHz; "
          f"{n_pages} pages {hp}x{wp}, {crops} crops")
    if not matched:
        print(f"WARNING: {len(conv)} conv_tc_kernel launches, {len(table)} layers in the table "
              f"(kernel counts craft {n_d}, crnn {n_r}): layers not named")
    print(f"{'#':>3} {'layer':<28} {'n x h x w x cin -> cout':<28} {'k':>1} {'instance':<26} {'ms':>8} {'GFLOP':>9} {'TFLOP/s':>8}")
    for r in rows:
        shape = "x".join(str(v) for v in r["shape"][:4]) + f"->{r['shape'][4]}" if "shape" in r else ""
        print(f"{r['launch']:>3} {r.get('layer', '?'):<28} {shape:<28} {r.get('ksize', ''):>1} {r['instance']:<26} "
              f"{r['ms']:8.3f} {r.get('flop', 0) / 1e9:9.1f} {r.get('tflops') or 0:8.1f}")
    for key in ("craft", "crnn", "conv_total"):
        t = out[key]
        print(f"{key:<10} {t['launches']:>3} launches {t['ms']:9.3f} ms {t['flop'] / 1e12:8.3f} TFLOP "
              f"{t['tflops'] or 0:7.1f} TFLOP/s")
    print(f"step {step:.3f} ms unprofiled (median of {len(step_ms)}), profiled GPU span {span_ms:.3f} ms; "
          f"outside conv_tc_kernel {100 * out['share_outside_conv_tc']:.1f} %; "
          f"layer FLOPs {out['layer_flop_sum'] / 1e12:.4f} T vs kernel count {out['kernel_flop_count'] / 1e12:.4f} T")


if __name__ == "__main__":
    main()
