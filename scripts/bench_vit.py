"""ViT-Nano / ViT-Tiny on bench.py's default workload: the BoT-SORT tracker, detection stream and frame ring of BASELINE
config 2 with seeded vit_tiny_parts3 (384x128 crops, 311 tokens, 2048-d rows) and vit_nano_ain_os (256x128, 129
tokens, 192-d rows) weights as the ReID backbone, alternated in one process with OSNet_x1_0 on the same workload, timed
with bench.py's own device and end-to-end legs; per-kernel time from a separate torch.profiler run over the same number
of crops; parity of the first frames against the oracle tracker fed by the float64 oracle ViT (PyTorch on the GPU).
Prints one JSON line.

    python scripts/bench_vit.py [--steps 100] [--warmup 10] [--rounds 2] [--parity-frames 2]

Writes nothing into the tree (the blobs go to a temporary directory).  The linear layers run as three-term TF32 wgmma;
the attention, norms and heads run in float32 on the CUDA cores."""
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
from scripts.bench_resnet import power_limit  # noqa: E402

KERNELS = ("k_conv_tc", "k_vit_attention", "k_vits_layernorm", "k_vits_ain", "k_vits_head", "k_vits_tokens",
           "k_vit_patchify", "k_crop_resize_norm")
VARIANTS = ("vit_tiny_parts3", "vit_nano_ain_os")


def vit_gflop_per_crop(variant):
    """Algorithmic GFLOP of one crop (2 x MAC), counted from the shapes: the patch embedding, per block qkv, proj, fc1,
    fc2 ("linears") and the two attention products q.k and p.v, and the head projections.  vit_nano*: 0.80 (attention
    10 %), vit_tiny*: 4.29 (attention 21 %)."""
    from boxmot_b200.weights import VIT_VARIANTS, vit_grid

    depth, _, _, parts, *_ = VIT_VARIANTS[variant]
    tokens, d = vit_grid(variant)[5], 192
    p = tokens - 1
    embed = 2 * p * 768 * d
    linears = depth * 2 * tokens * d * (3 * d + d + 4 * d + 4 * d)
    attention = depth * 2 * 2 * tokens * tokens * d
    head = (1 + parts) * 2 * d * 512 if variant.startswith("vit_tiny") else 0
    total = embed + linears + attention + head
    return {"embed": embed / 1e9, "linears": linears / 1e9, "attention": attention / 1e9, "total": total / 1e9,
            "attention_share": attention / total}


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


class _DeviceOracle:
    """The float64 oracle ViT on the GPU (PyTorch), on crops staged by the oracle's CPU restatement."""

    def __init__(self, sd, variant):
        import torch

        from tests import vit_oracle as ov

        self.ov, self.torch = ov, torch
        self.sd = {k: v.cuda() for k, v in ov.double_state(sd).items()}
        self.variant = variant

    def get_features(self, xyxys, img):
        ov, torch = self.ov, self.torch
        xyxys = np.asarray(xyxys, dtype=np.float32)
        if xyxys.size == 0:
            return np.array([])
        x = ov.get_crops(xyxys, img, "resize", ov.input_hw(self.variant))
        f = torch.cat([ov.vit_forward(self.sd, self.variant, x[i:i + 64].cuda().double())
                       for i in range(0, len(x), 64)]).cpu().numpy()
        return (f / np.linalg.norm(f, axis=-1, keepdims=True)).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=2, help="alternations of the ViTs and OSNet_x1_0")
    ap.add_argument("--parity-frames", type=int, default=2, help="first frames of stream 0 checked against the oracle")
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_vit.py needs a CUDA device: boxmot_b200 has no CPU fallback")
    torch.cuda.set_device(0)
    from boxmot_b200.synthetic import make_osnet_state, make_vit_state
    from boxmot_b200.weights import export_blob, read_blob

    base = bench.CONFIGS[2]
    tmp = Path(tempfile.mkdtemp(prefix="b200vit_"))
    states = {v: make_vit_state(v, 0) for v in VARIANTS}
    models = {}
    for v in VARIANTS:
        blob = export_blob(states[v], tmp / f"{v}_synthetic.b200reid")
        models[v] = (dict(base, id=2, arch=v, feat=int(read_blob(blob)[0][7])), blob)
    models["osnet_x1_0"] = (dict(base, id=2, arch="osnet_x1_0", feat=512),
                            export_blob(make_osnet_state("osnet_x1_0", seed=0), tmp / "osnet_x1_0_synthetic.b200reid"))
    K, Wm = args.steps, max(3, args.warmup)
    runs = {name: [] for name in models}
    for _ in range(args.rounds):
        for name, (cfg, blob) in models.items():
            dev = bench.device_run(cfg, blob, K, Wm, None)
            e2e_ms, _, api = bench.e2e_run(cfg, blob, dev["per_stream"], K, Wm, None, pinned=False)
            reid_ms = sum(dev["prof"][c]["ms_per_step"] for c in bench.CLASSES if c != "association")
            runs[name].append(dict(dev=dev, e2e_ms=e2e_ms, api=api, reid_ms=reid_ms))

    from oracle.trackers import BotSortOracle

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

    line = {"metric": "tracker.update() frames/sec with ViT ReID (vit_tiny_parts3)", "unit": "frames/s", "steps": K,
            "warmup": Wm, "rounds": args.rounds, "data": "synthetic",
            "workload": f"botsort workload of BASELINE config 2 ({base['dets']} dets/frame, {base['hw'][0]}x{base['hw'][1]}) "
                        f"with ReID in update(); {', '.join(models)} alternated in one process",
            "card": power_limit(), "osnet_x1_0": summary("osnet_x1_0")}
    for v in VARIANTS:
        cfg, blob = models[v]
        first = runs[v][0]["dev"]
        ps = first["per_stream"][0]
        orc = BotSortOracle(reid_model=_DeviceOracle(states[v], v), **cfg["params"])
        rows = [np.asarray(orc.update(ps[1][f], ps[0][f % cfg["ring"]]), np.float32).reshape(-1, 8)
                for f in range(args.parity_frames)]
        res = summary(v)
        flop = vit_gflop_per_crop(v)
        reid_ms = min(res["reid_device_ms_per_frame"])
        gflop_frame = res["crops_per_frame"] * flop["total"]
        res.update(gflop_per_crop=flop, algorithmic_gflop_per_frame=gflop_frame,
                   achieved_tflops=gflop_frame / reid_ms,   # GFLOP per ms = TFLOP/s
                   kernels=kernel_profile(blob, int(round(res["crops_per_frame"]))),
                   parity=bench.parity_check(cfg, blob, rows, first["per_stream"]))
        line[v] = res
    line["value"] = max(line["vit_tiny_parts3"]["device_fps"])
    print(json.dumps(line))


if __name__ == "__main__":
    main()
