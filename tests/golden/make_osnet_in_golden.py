"""Embeddings of the reference's osnet_ain_x1_0, osnet_ain_x0_25 (reid/backbones/osnet_ain.py) and osnet_ibn_x1_0
(reid/backbones/osnet.py:548) classes with seeded weights loaded by `load_state_dict(strict=True)`, on a handful of boxes
of a seeded frame (a fully outside box, i.e. a blank crop, and a clipped box included), through the reference backend's
own `get_features` at 256x128, in both preprocess modes.  Pins `oracle.osnet_in`.
Writes tests/golden/reid_osnet_in_reference.npz.   Run: python tests/golden/make_osnet_in_golden.py"""
from __future__ import annotations

import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parents[1]))
import refharness  # noqa: E402
from make_reid_arch_golden import boxes_for  # noqa: E402

IMAGE_SEED, NUM_CLASSES = 323, 4101
MODELS = {"osnet_ain_x1_0": 31, "osnet_ain_x0_25": 32, "osnet_ibn_x1_0": 33}   # name -> weight seed
MODES = ("resize", "resize_pad")


def main():
    refharness.install_reference()
    import torch
    from boxmot.reid.backbones import osnet, osnet_ain
    from boxmot.reid.backends.base_backend import BaseModelBackend
    from boxmot.reid.core.preprocessing import get_preprocess_fn

    from boxmot_b200.synthetic import make_osnet_ain_state, make_osnet_ibn_state

    class RefBackend(BaseModelBackend):
        def __init__(self, model, preprocess):
            self.device = torch.device("cpu")
            self.half = False
            self.input_shape = (256, 128)
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
    boxes = boxes_for(seed=11)
    out = {"boxes": boxes, "image_seed": np.int64(IMAGE_SEED), "num_classes": np.int64(NUM_CLASSES)}
    for name, seed in MODELS.items():
        if name.startswith("osnet_ain"):
            m = getattr(osnet_ain, name)(num_classes=NUM_CLASSES, pretrained=False)
            sd = make_osnet_ain_state(name, seed=seed, num_classes=NUM_CLASSES)
        else:
            m = osnet.osnet_ibn_x1_0(num_classes=NUM_CLASSES, pretrained=False)
            sd = make_osnet_ibn_state(seed=seed, num_classes=NUM_CLASSES)
        m.load_state_dict(sd, strict=True)
        m.eval()
        out[f"weight_seed_{name}"] = np.int64(seed)
        for mode in MODES:
            out[f"{name}_{mode}"] = np.asarray(RefBackend(m, mode).get_features(boxes, img), np.float32)
    np.savez_compressed(HERE / "reid_osnet_in_reference.npz", **out)
    print({k: getattr(v, "shape", v) for k, v in out.items()})


if __name__ == "__main__":
    main()
