"""Embeddings of the reference's LMBN_n class (`reid/backbones/lmbn/lmbn_n.py`) with seeded weights loaded by
`load_state_dict(strict=True)`, on a handful of boxes of a seeded frame (outside and clipped boxes included), through
the reference backend's own `get_features` at `input_shape=(384, 128)` (base_backend.py:59-60), in both preprocess
modes, plus the sha256 of the staged float32 NCHW crops of each mode.  Pins `oracle.lmbn.lmbn_n_forward` and the
384x128 crop staging.  Writes tests/golden/reid_lmbn_n_reference.npz.   Run: python tests/golden/make_lmbn_golden.py"""
from __future__ import annotations

import hashlib
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parents[1]))
import refharness  # noqa: E402
from make_reid_arch_golden import boxes_for  # noqa: E402

IMAGE_SEED, LMBN_SEED, NUM_CLASSES = 322, 17, 702
MODES = ("resize", "resize_pad")


def main():
    refharness.install_reference()
    import torch
    from boxmot.reid.backbones.lmbn.lmbn_n import LMBN_n
    from boxmot.reid.backends.base_backend import BaseModelBackend
    from boxmot.reid.core.preprocessing import get_preprocess_fn

    from boxmot_b200.synthetic import make_lmbn_n_state

    class RefBackend(BaseModelBackend):
        def __init__(self, model, preprocess):
            self.device = torch.device("cpu")
            self.half = False
            self.input_shape = (384, 128)
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
    boxes = boxes_for(seed=10)
    out = {"boxes": boxes, "image_seed": np.int64(IMAGE_SEED), "weight_seed": np.int64(LMBN_SEED),
           "num_classes": np.int64(NUM_CLASSES)}
    m = LMBN_n(num_classes=NUM_CLASSES, loss="softmax", pretrained=False, use_gpu=False)
    m.load_state_dict(make_lmbn_n_state(seed=LMBN_SEED, num_classes=NUM_CLASSES), strict=True)
    m.eval()
    for mode in MODES:
        be = RefBackend(m, mode)
        crops = be.get_crops(boxes, img)
        out[f"crops_sha256_{mode}"] = hashlib.sha256(np.ascontiguousarray(crops.numpy()).tobytes()).hexdigest()
        out[f"features_{mode}"] = np.asarray(be.get_features(boxes, img), np.float32)
    np.savez_compressed(HERE / "reid_lmbn_n_reference.npz", **out)
    print({k: getattr(v, "shape", v) for k, v in out.items()})


if __name__ == "__main__":
    main()
