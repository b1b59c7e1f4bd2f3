"""Embeddings of the reference's resnet50 / resnet101 (`reid/backbones/resnet.py`) with seeded weights, on a handful of
boxes of a seeded frame (outside and clipped boxes included), through the reference backend's own `get_features` at
256x128, in both preprocess modes, plus the sha256 of the staged float32 NCHW crops of each mode.  Three cases:
    resnet50     make_resnet_state(50) loaded with strict=True
    resnet101    make_resnet_state(101) loaded with strict=True
    fc512        a resnet50_fc512-shaped state dict (fc.0 / fc.1 head, 512-wide classifier) loaded by
                 ReIDModelRegistry.load_pretrained_weights into the model get_model_name("resnet50_fc512_market1501.pt")
                 picks (plain resnet50: the fc and classifier tensors are discarded)
Pins `oracle.resnet.resnet_forward`.  Writes tests/golden/reid_resnet_reference.npz.
Run: python tests/golden/make_resnet_golden.py"""
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

IMAGE_SEED, NUM_CLASSES = 323, 751
CASES = {"resnet50": (50, 31, False), "resnet101": (101, 32, False), "fc512": (50, 33, True)}
MODES = ("resize", "resize_pad")


def main():
    refharness.install_reference()
    import torch
    from boxmot.reid.backbones import resnet as ref_resnet
    from boxmot.reid.backends.base_backend import BaseModelBackend
    from boxmot.reid.core.preprocessing import get_preprocess_fn
    from boxmot.reid.core.registry import ReIDModelRegistry

    from boxmot_b200.synthetic import make_resnet_state

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
    for case, (depth, seed, fc512) in CASES.items():
        sd = make_resnet_state(depth, seed=seed, with_fc512=fc512, num_classes=NUM_CLASSES)
        if fc512:
            name = ReIDModelRegistry.get_model_name("resnet50_fc512_market1501.pt")
            assert name == "resnet50", name
            m = getattr(ref_resnet, name)(num_classes=NUM_CLASSES, pretrained=False)
            with tempfile.TemporaryDirectory() as d:
                pt = Path(d) / "resnet50_fc512_market1501.pt"
                torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, pt)
                ReIDModelRegistry.load_pretrained_weights(m, pt)
        else:
            m = getattr(ref_resnet, f"resnet{depth}")(num_classes=NUM_CLASSES, pretrained=False)
            m.load_state_dict(sd, strict=True)
        m.eval()
        out[f"{case}_depth"] = np.int64(depth)
        out[f"{case}_seed"] = np.int64(seed)
        out[f"{case}_fc512"] = np.int64(fc512)
        for mode in MODES:
            be = RefBackend(m, mode)
            if case == "resnet50":
                crops = be.get_crops(boxes, img)
                out[f"crops_sha256_{mode}"] = hashlib.sha256(np.ascontiguousarray(crops.numpy()).tobytes()).hexdigest()
            out[f"{case}_features_{mode}"] = np.asarray(be.get_features(boxes, img), np.float32)
    np.savez_compressed(HERE / "reid_resnet_reference.npz", **out)
    print({k: getattr(v, "shape", v) for k, v in out.items()})


if __name__ == "__main__":
    main()
