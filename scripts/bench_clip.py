"""CLIP-ReID ViT-B/16 on bench.py's default workload: the BoT-SORT tracker, detection stream and frame ring of BASELINE
config 2 with clip_market1501-shaped seeded weights (256x128 crops, 129 tokens, 1280-d rows) as the ReID backbone,
alternated in one process with ResNet50 on the same workload, timed with bench.py's own device and end-to-end legs;
per-kernel time from a separate torch.profiler run over the same number of crops; parity of the first frames against
the oracle tracker fed by the oracle CLIP.  Prints one JSON line.

    python scripts/bench_clip.py [--steps 100] [--warmup 10] [--rounds 2] [--parity-frames 2]

Writes nothing into the tree (the blobs go to a temporary directory).  The linear layers run as three-term TF32
wgmma, so their share of peak is against the data sheet's dense TF32 rate with the three MMAs per product counted; the
attention runs in float32 on the CUDA cores."""
from __future__ import annotations

import argparse
import json
import sys
import tempfile
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

import bench  # noqa: E402
from scripts.bench_resnet import FP32_PEAK_TFLOPS, TC_TERMS, TF32_PEAK_TFLOPS, power_limit  # noqa: E402

KERNELS = ("k_conv_tc", "k_vit_attention", "k_vit_layernorm", "k_vit_head", "k_vit_patchify", "k_crop_resize_norm")


def clip_gflop_per_crop(tokens=129, width=768, layers=12, proj=512):
    """Algorithmic GFLOP of one crop (2 x MAC): the patch embedding, per block in_proj, out_proj, c_fc, c_proj
    ("linears") and the two attention products q.k and p.v, and the head projection.  At 129 tokens: 21.9 linears +
    0.15 embedding + 0.61 attention = 22.7."""
    p = tokens - 1
    embed = 2 * p * 768 * width
    linears = layers * 2 * tokens * width * (3 * width + width + 4 * width + 4 * width)
    attention = layers * 2 * 2 * tokens * tokens * width
    head = 2 * width * proj
    return {"embed": embed / 1e9, "linears": linears / 1e9, "attention": attention / 1e9,
            "total": (embed + linears + attention + head) / 1e9}


def kernel_profile(blob, n_crops, reps=5):
    """Device time per kernel name over `reps` forwards of `n_crops` crops (torch.profiler, CUDA activities)."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    from boxmot_b200.reid import B200ReID

    reid = B200ReID(str(blob))
    rng = np.random.default_rng(0)
    img = rng.integers(0, 255, size=(1080, 1920, 3), dtype=np.uint8)
    cx, cy = rng.uniform(0, 1920, n_crops), rng.uniform(0, 1080, n_crops)
    bw, bh = rng.uniform(20, 160, n_crops), rng.uniform(40, 320, n_crops)
    boxes = np.stack([cx - bw / 2, cy - bh / 2, cx + bw / 2, cy + bh / 2], 1).astype(np.float32)
    reid.get_features(boxes, img)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            reid.get_features(boxes, img)
        torch.cuda.synchronize()
    ms = {k: 0.0 for k in KERNELS}
    other = 0.0
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        name = next((k for k in KERNELS if k in ev.key), None)
        if name:
            ms[name] += t / 1e3 / reps
        elif "memcpy" not in ev.key.lower() and "memset" not in ev.key.lower():
            other += t / 1e3 / reps
    reid.close()
    total = sum(ms.values())
    return {"crops": n_crops, "ms_per_forward": ms, "other_kernels_ms": other, "total_ms": total,
            "attention_share": ms["k_vit_attention"] / total if total else None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=2, help="alternations of CLIP and ResNet50")
    ap.add_argument("--parity-frames", type=int, default=2, help="first frames of stream 0 checked against the oracle (CPU)")
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_clip.py needs a CUDA device: boxmot_b200 has no CPU fallback")
    torch.cuda.set_device(0)
    from boxmot_b200.synthetic import make_clip_state, make_resnet_state
    from boxmot_b200.weights import export_blob

    base = bench.CONFIGS[2]
    tmp = Path(tempfile.mkdtemp(prefix="b200clip_"))
    sd = make_clip_state(0)
    models = {
        "clip_market1501": (dict(base, id=2, arch="clip_market1501", feat=1280),
                            export_blob(sd, tmp / "clip_market1501_synthetic.b200reid")),
        "resnet50": (dict(base, id=2, arch="resnet50", feat=2048),
                     export_blob(make_resnet_state(50, seed=0), tmp / "resnet50_synthetic.b200reid")),
    }
    K, Wm = args.steps, max(3, args.warmup)
    runs = {name: [] for name in models}
    for _ in range(args.rounds):
        for name, (cfg, blob) in models.items():
            dev = bench.device_run(cfg, blob, K, Wm, None)
            e2e_ms, _, api = bench.e2e_run(cfg, blob, dev["per_stream"], K, Wm, None, pinned=False)
            reid_ms = sum(dev["prof"][c]["ms_per_step"] for c in bench.CLASSES if c != "association")
            runs[name].append(dict(dev=dev, e2e_ms=e2e_ms, api=api, reid_ms=reid_ms))

    cfg, blob = models["clip_market1501"]
    first = runs["clip_market1501"][0]["dev"]
    ps = first["per_stream"][0]
    from oracle.clip import OracleCLIP
    from oracle.trackers import BotSortOracle

    orc = BotSortOracle(reid_model=OracleCLIP(sd), **cfg["params"])
    rows = [np.asarray(orc.update(ps[1][f], ps[0][f % cfg["ring"]]), np.float32).reshape(-1, 8)
            for f in range(args.parity_frames)]
    parity = bench.parity_check(cfg, blob, rows, first["per_stream"])

    def summary(name):
        rs = runs[name]
        best = min(rs, key=lambda r: r["dev"]["value_ms"])
        return {
            "device_fps": [K / (r["dev"]["value_ms"] * 1e-3) for r in rs],
            "e2e_fps": [K / (r["e2e_ms"] * 1e-3) for r in rs],
            "reid_device_ms_per_frame": [r["reid_ms"] for r in rs],
            "crops_per_frame": best["dev"]["crops"],
            "kernel_classes": best["dev"]["prof"],
        }

    flop = clip_gflop_per_crop()
    res = summary("clip_market1501")
    reid_ms = min(res["reid_device_ms_per_frame"])
    gflop_frame = res["crops_per_frame"] * flop["total"]
    achieved = gflop_frame / reid_ms   # GFLOP per ms = TFLOP/s
    kp = kernel_profile(blob, int(round(res["crops_per_frame"])))
    gemm_ms = kp["ms_per_forward"]["k_conv_tc"]
    gemm_tflops = kp["crops"] * (flop["linears"] + flop["embed"]) / gemm_ms if gemm_ms else None
    line = {
        "metric": "tracker.update() frames/sec with CLIP-ReID ViT-B/16", "value": max(res["device_fps"]),
        "unit": "frames/s", "steps": K, "warmup": Wm, "rounds": args.rounds, "data": "synthetic",
        "workload": f"botsort workload of BASELINE config 2 ({base['dets']} dets/frame, {base['hw'][0]}x{base['hw'][1]}) "
                    f"with ReID in update(); clip_market1501 and resnet50 alternated in one process",
        "card": power_limit(),
        "clip_market1501": res,
        "resnet50": summary("resnet50"),
        "kernels": kp,
        "roofline": {"kernel": "CLIP ReID (all kernels of a frame, serialised device time)",
                     "gflop_per_crop": flop, "algorithmic_gflop_per_frame": gflop_frame,
                     "achieved_tflops": achieved,
                     "gemm_tflops": gemm_tflops,
                     "gemm_tf32x3_frac": gemm_tflops * TC_TERMS / TF32_PEAK_TFLOPS if gemm_tflops else None,
                     "fp32_floor_ms_per_frame": gflop_frame / FP32_PEAK_TFLOPS,
                     "peak_source": "H100 SXM data sheet (dense TF32 495 TFLOP/s, FP32 67 TFLOP/s, 700 W), not measured"},
        "parity": parity,
    }
    print(json.dumps(line))


if __name__ == "__main__":
    main()
