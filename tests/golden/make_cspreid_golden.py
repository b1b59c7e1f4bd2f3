"""Embeddings of the reference's CSPReID-n ReID model (reid/backbones/cspreid_n.py, built by
`ReIDModelRegistry.build_model` with pretrained=False) with seeded weights, on a handful of boxes of a seeded frame
(outside and clipped boxes included), through the reference backend's own `get_features`, in both preprocess modes,
plus the sha256 of the staged float32 NCHW crops.  Two checkpoints: `cspreid_n_market1501.pt` (256x128 crops) and
`cspreid_n_veri.pt` (256x256 crops, base_backend.py's vehicle rule), each saved as a training checkpoint
(`{"state_dict": module.-prefixed}`) and loaded by `ReIDModelRegistry.load_pretrained_weights`; every tensor of the
model must come from the file.  `make_cspreid_state` randomises every BatchNorm, so no bottleneck is the identity the
reference's own initialisation makes of it.
Pins `tests/cspreid_oracle.py`.  Writes tests/golden/reid_cspreid_reference.npz.
Run: python tests/golden/make_cspreid_golden.py"""
from __future__ import annotations

import hashlib
import sys
import tempfile
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parents[1]))
import refharness  # noqa: E402
from make_reid_arch_golden import boxes_for  # noqa: E402

IMAGE_SEED, NUM_CLASSES = 411, 751
FILES = {"cspreid_n_market1501.pt": 61, "cspreid_n_veri.pt": 62}
MODES = ("resize", "resize_pad")
OUT = HERE / "reid_cspreid_reference.npz"


def compute():
    refharness.install_reference()
    import torch
    from boxmot.reid.backends.base_backend import BaseModelBackend
    from boxmot.reid.core.preprocessing import get_preprocess_fn
    from boxmot.reid.core.registry import ReIDModelRegistry

    from boxmot_b200.synthetic import make_cspreid_state

    threads = torch.get_num_threads()
    torch.set_num_threads(1)   # one summation order for the float32 convolutions: the file regenerates bit for bit
    try:
        return _compute(torch, BaseModelBackend, get_preprocess_fn, ReIDModelRegistry, make_cspreid_state)
    finally:
        torch.set_num_threads(threads)


def _compute(torch, BaseModelBackend, get_preprocess_fn, ReIDModelRegistry, make_cspreid_state):

    class RefBackend(BaseModelBackend):
        def __init__(self, model, preprocess, input_shape):
            self.device = torch.device("cpu")
            self.half = False
            self.input_shape = input_shape
            self.nhwc = False
            self.preprocess_fn = get_preprocess_fn(preprocess)
            self.mean_array = torch.tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1)
            self.std_array = torch.tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1)
            self.model = model

        def forward(self, x):
            return self.model(x)

        def load_model(self, w):
            pass

    img = np.random.default_rng(IMAGE_SEED).integers(0, 255, size=(540, 960, 3), dtype=np.uint8)
    boxes = boxes_for(seed=19)
    out = {"boxes": boxes, "image_seed": np.int64(IMAGE_SEED), "num_classes": np.int64(NUM_CLASSES)}
    for fname, seed in FILES.items():
        key = Path(fname).stem
        sd = make_cspreid_state(seed, num_classes=NUM_CLASSES)
        with tempfile.TemporaryDirectory() as d:
            pt = Path(d) / fname
            torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, pt)
            name = ReIDModelRegistry.get_model_name(pt)
            assert name == "cspreid_n", name
            m = ReIDModelRegistry.build_model(name, pt, num_classes=NUM_CLASSES, pretrained=False)
            assert set(m.state_dict()) == set(sd), sorted(set(m.state_dict()) ^ set(sd))[:8]
            ReIDModelRegistry.load_pretrained_weights(m, pt)
        for k, v in m.state_dict().items():   # every tensor came from the checkpoint
            assert torch.equal(v, sd[k]), k
        m.eval()
        input_shape = (256, 256) if "vehicleid" in fname or "veri" in fname else (256, 128)   # base_backend.py's rule
        out[f"{key}_seed"] = np.int64(seed)
        out[f"{key}_input_hw"] = np.array(input_shape, np.int64)
        for mode in MODES:
            be = RefBackend(m, mode, input_shape)
            crops = be.get_crops(boxes, img)
            out[f"{key}_crops_sha256_{mode}"] = hashlib.sha256(np.ascontiguousarray(crops.numpy()).tobytes()).hexdigest()
            with torch.no_grad():
                out[f"{key}_features_{mode}"] = np.asarray(be.get_features(boxes, img), np.float32)
    return out


def main():
    out = compute()
    np.savez_compressed(OUT, **out)
    print({k: getattr(v, "shape", v) for k, v in out.items()})


if __name__ == "__main__":
    main()
