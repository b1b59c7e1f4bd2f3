"""Embeddings of the reference's ViT-Nano / ViT-Tiny ReID models (vit_nano, vit_nano_ain, vit_nano_ain_os, vit_tiny,
vit_tiny_parts, vit_tiny_parts3; reid/backbones/vit_nano.py and vit_tiny.py, built by `ReIDModelRegistry.build_model`
with pretrained=False) with seeded weights, on a handful of boxes of a seeded frame (outside and clipped boxes
included), through the reference backend's own `get_features`, in both preprocess modes, plus the sha256 of the
staged float32 NCHW crops.  Each variant's `make_vit_state` weights are saved as the reference trainer saves them
(`{"state_dict": module.-prefixed, "model_name": ...}`) and loaded by `ReIDModelRegistry.load_pretrained_weights`;
every tensor of the model must come from the file.
Pins `tests/vit_oracle.vit_forward`.  Writes tests/golden/reid_vit_reference.npz.
Run: python tests/golden/make_vit_golden.py"""
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

IMAGE_SEED, NUM_CLASSES = 337, 751
SEEDS = {"vit_nano": 51, "vit_nano_ain": 52, "vit_nano_ain_os": 53, "vit_tiny": 54, "vit_tiny_parts": 55,
         "vit_tiny_parts3": 56}
MODES = ("resize", "resize_pad")


def main():
    refharness.install_reference()
    import torch
    from boxmot.reid.backends.base_backend import BaseModelBackend
    from boxmot.reid.core.preprocessing import get_preprocess_fn
    from boxmot.reid.core.registry import ReIDModelRegistry

    from boxmot_b200.synthetic import make_vit_state

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
    boxes = boxes_for(seed=17)
    out = {"boxes": boxes, "image_seed": np.int64(IMAGE_SEED), "num_classes": np.int64(NUM_CLASSES)}
    for variant, seed in SEEDS.items():
        sd = make_vit_state(variant, seed, num_classes=NUM_CLASSES)
        with tempfile.TemporaryDirectory() as d:
            pt = Path(d) / f"{variant}_market1501.pt"
            torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}, "model_name": variant}, pt)
            name = ReIDModelRegistry.get_model_name(pt)
            assert name == variant, name
            m = ReIDModelRegistry.build_model(name, pt, num_classes=NUM_CLASSES, pretrained=False)
            assert set(m.state_dict()) == set(sd), sorted(set(m.state_dict()) ^ set(sd))[:8]
            ReIDModelRegistry.load_pretrained_weights(m, pt)
        for k, v in m.state_dict().items():   # every tensor came from the checkpoint
            assert torch.equal(v, sd[k]), k
        m.eval()
        input_shape = (384, 128) if "vit_tiny" in name else (256, 128)   # base_backend.py's rule
        out[f"{variant}_seed"] = np.int64(seed)
        for mode in MODES:
            be = RefBackend(m, mode, input_shape)
            crops = be.get_crops(boxes, img)
            out[f"{variant}_crops_sha256_{mode}"] = hashlib.sha256(np.ascontiguousarray(crops.numpy()).tobytes()).hexdigest()
            with torch.no_grad():
                out[f"{variant}_features_{mode}"] = np.asarray(be.get_features(boxes, img), np.float32)
    np.savez_compressed(HERE / "reid_vit_reference.npz", **out)
    print({k: getattr(v, "shape", v) for k, v in out.items()})


if __name__ == "__main__":
    main()
