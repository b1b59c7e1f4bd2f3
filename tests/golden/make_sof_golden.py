"""Regenerate tests/golden/cmc_sof.npz from the UNMODIFIED reference SOF class (boxmot/motion/cmc/sof.py).

* `<seq>_warps` -- what SOF().apply(frame, dets) returned on seeded synthetic sequences: camera_similarity_sequence
  (pan + rotation + zoom) at 360p and 720p, camera_pan_sequence at 360p, with each frame's detections passed.
* `mot17_reg`   -- BaseCMC.preprocess (162 x 288) of the first frames of the reference's assets/MOT17-mini sequences.
* `mot17_warps` -- what SOF().apply returned on those frames (no detections), per sequence.

Needs the reference package (located by tests/golden/refharness.py):  python tests/golden/make_sof_golden.py
"""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT))
from tests.golden.refharness import REFERENCE_ROOT, install_reference  # noqa: E402

install_reference()
import cv2  # noqa: E402
from boxmot.motion.cmc.sof import SOF  # noqa: E402

from boxmot_b200.synthetic import camera_pan_sequence, camera_similarity_sequence  # noqa: E402

SEQS = {"sim360": ("sim", (360, 640), 21), "sim720": ("sim", (720, 1280), 22), "pan360": ("pan", (360, 640), 23)}
N_FRAMES = 8


def frames_of(kind, hw, seed):
    if kind == "sim":
        f, d, _ = camera_similarity_sequence(N_FRAMES, hw=hw, seed=seed)
    else:
        f, d, _, _ = camera_pan_sequence(N_FRAMES, hw=hw, seed=seed)
    return f, d


out = {}
for name, (kind, hw, seed) in SEQS.items():
    frames, dets = frames_of(kind, hw, seed)
    ref = SOF()
    out[f"{name}_warps"] = np.stack([ref.apply(f, d) for f, d in zip(frames, dets)]).astype(np.float32)
regs, warps = [], []
for seq in ("MOT17-02-FRCNN", "MOT17-04-FRCNN"):
    files = sorted((REFERENCE_ROOT / "assets" / "MOT17-mini" / "train" / seq / "img1").glob("*.jpg"))[:5]
    ref = SOF()
    for f in files:
        img = cv2.imread(str(f))
        warps.append(ref.apply(img))
        regs.append(ref.prev_frame.copy())
out["mot17_reg"] = np.stack(regs)
out["mot17_warps"] = np.stack(warps).astype(np.float32)
np.savez_compressed(ROOT / "tests" / "golden" / "cmc_sof.npz", **out)
print({k: v.shape for k, v in out.items()})
