"""Embeddings of the reference's HACNN (`reid/backbones/hacnn.py`) with seeded weights, on a handful of boxes of a seeded
frame (outside and clipped boxes included), through the reference backend's own `get_features` at 160x64, in both
preprocess modes, plus the sha256 of the staged float32 NCHW crops of each mode.  Two cases:
    strict       make_hacnn_state loaded with strict=True
    checkpoint   make_hacnn_state saved as {"state_dict": {"module." + k}} under the name hacnn_market1501.pt and loaded by
                 ReIDModelRegistry.load_pretrained_weights into the model get_model_name picks for that name
Pins `oracle.hacnn.hacnn_forward`.  Writes tests/golden/reid_hacnn_reference.npz.
Run: python tests/golden/make_hacnn_golden.py"""
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

IMAGE_SEED, NUM_CLASSES = 331, 751
CASES = {"strict": 51, "checkpoint": 52}
MODES = ("resize", "resize_pad")


def main():
    refharness.install_reference()
    import torch
    from boxmot.reid.backbones import hacnn as ref_hacnn
    from boxmot.reid.backends.base_backend import BaseModelBackend
    from boxmot.reid.core.preprocessing import get_preprocess_fn
    from boxmot.reid.core.registry import ReIDModelRegistry

    from boxmot_b200.synthetic import make_hacnn_state

    class RefBackend(BaseModelBackend):
        def __init__(self, model, preprocess):
            self.device = torch.device("cpu")
            self.half = False
            self.input_shape = (160, 64)
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
    boxes = boxes_for(seed=13)
    out = {"boxes": boxes, "image_seed": np.int64(IMAGE_SEED), "num_classes": np.int64(NUM_CLASSES)}
    for case, seed in CASES.items():
        sd = make_hacnn_state(seed=seed, num_classes=NUM_CLASSES)
        m = ref_hacnn.HACNN(NUM_CLASSES)
        if case == "checkpoint":
            assert ReIDModelRegistry.get_model_name("hacnn_market1501.pt") == "hacnn"
            with tempfile.TemporaryDirectory() as d:
                pt = Path(d) / "hacnn_market1501.pt"
                torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, pt)
                ReIDModelRegistry.load_pretrained_weights(m, pt)
        else:
            m.load_state_dict(sd, strict=True)
        m.eval()
        out[f"{case}_seed"] = np.int64(seed)
        for mode in MODES:
            be = RefBackend(m, mode)
            if case == "strict":
                crops = be.get_crops(boxes, img)
                out[f"crops_sha256_{mode}"] = hashlib.sha256(np.ascontiguousarray(crops.numpy()).tobytes()).hexdigest()
            out[f"{case}_features_{mode}"] = np.asarray(be.get_features(boxes, img), np.float32)
    np.savez_compressed(HERE / "reid_hacnn_reference.npz", **out)
    print({k: getattr(v, "shape", v) for k, v in out.items()})


if __name__ == "__main__":
    main()
