"""Embeddings of the reference's CLIP-ReID ViT-B/16 (`reid/backbones/clip`, built by `ReIDModelRegistry.build_model`)
with seeded weights, on a handful of boxes of a seeded frame (outside and clipped boxes included), through the
reference backend's own `get_features`, in both preprocess modes, plus the sha256 of the staged float32 NCHW crops.
Two cases, each a `make_clip_state` checkpoint (`state_dict`, `module.` prefixes, with discarded extra keys) loaded by
`ReIDModelRegistry.load_pretrained_weights`:
    market   clip_market1501.pt   256x128 crops, 129 positions
    veri     clip_veri.pt         256x256 crops, 257 positions
`make_model.load_clip_to_cpu` downloads OpenAI's ViT-B-16; it is replaced by a call to the reference's own
`clip.build_model` on an OpenAI-layout state dict (ViT-B/16 vision tower with 197 positions, a tiny text tower, which
the head never uses), so `resize_pos_embed` and `convert_weights` run as in the reference.  The reference mutates its
module-level cfg for vehicle names; it is restored after each build.
Pins `oracle.clip.clip_forward`.  Writes tests/golden/reid_clip_reference.npz.
Run: python tests/golden/make_clip_golden.py"""
from __future__ import annotations

import copy
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
CASES = {"market": ("clip_market1501.pt", 41, False), "veri": ("clip_veri.pt", 42, True)}
MODES = ("resize", "resize_pad")


def openai_vit_b16_state():
    """State dict in the layout of OpenAI's ViT-B-16 release (visual.* at 224x224: 197 positions) with a tiny text
    tower, from the reference's own CLIP class."""
    import torch
    from boxmot.reid.backbones.clip.clip.model import CLIP

    torch.manual_seed(0)
    m = CLIP(embed_dim=512, image_resolution=224, vision_layers=12, vision_width=768, vision_patch_size=16,
             vision_stride_size=16, context_length=4, vocab_size=8, transformer_width=64, transformer_heads=1,
             transformer_layers=1, h_resolution=14, w_resolution=14)
    return {k: v.clone() for k, v in m.state_dict().items()}


def main():
    refharness.install_reference()
    import torch
    from boxmot.reid.backbones.clip import make_model as ref_make_model
    from boxmot.reid.backbones.clip.clip import clip as ref_clip
    from boxmot.reid.backbones.clip.config.defaults import _C as cfg
    from boxmot.reid.backends.base_backend import BaseModelBackend
    from boxmot.reid.core.preprocessing import get_preprocess_fn
    from boxmot.reid.core.registry import ReIDModelRegistry

    from boxmot_b200.synthetic import make_clip_state

    openai_sd = openai_vit_b16_state()

    def load_clip_to_cpu(backbone_name, h_resolution, w_resolution, vision_stride_size):
        assert backbone_name == "ViT-B-16"
        return ref_clip.build_model(copy.deepcopy(openai_sd), h_resolution, w_resolution, vision_stride_size)

    ref_make_model.load_clip_to_cpu = load_clip_to_cpu
    size_train, size_test = list(cfg.INPUT.SIZE_TRAIN), list(cfg.INPUT.SIZE_TEST)

    class RefBackend(BaseModelBackend):
        def __init__(self, model, preprocess, input_shape):
            self.device = torch.device("cpu")
            self.half = False
            self.input_shape = input_shape
            self.nhwc = False
            self.preprocess_fn = get_preprocess_fn(preprocess)
            self.mean_array = torch.tensor([0.5, 0.5, 0.5]).view(1, 3, 1, 1)
            self.std_array = torch.tensor([0.5, 0.5, 0.5]).view(1, 3, 1, 1)
            self.model = model

        def forward(self, x):
            return self.model(x)

        def load_model(self, w):
            pass

    img = np.random.default_rng(IMAGE_SEED).integers(0, 255, size=(540, 960, 3), dtype=np.uint8)
    boxes = boxes_for(seed=13)
    out = {"boxes": boxes, "image_seed": np.int64(IMAGE_SEED), "num_classes": np.int64(NUM_CLASSES)}
    for case, (fname, seed, vehicle) in CASES.items():
        sd = make_clip_state(seed, vehicle=vehicle, num_classes=NUM_CLASSES)
        name = ReIDModelRegistry.get_model_name(fname)
        assert name == "clip", name
        try:
            m = ReIDModelRegistry.build_model(name, Path(fname), num_classes=NUM_CLASSES, pretrained=False)
        finally:
            cfg.INPUT.SIZE_TRAIN, cfg.INPUT.SIZE_TEST = list(size_train), list(size_test)
        ref_keys = {k for k in m.state_dict()}
        assert ref_keys == {k for k in sd if not k.startswith(("prompt_learner.", "text_encoder."))}, \
            sorted(ref_keys ^ set(sd))[:8]
        with tempfile.TemporaryDirectory() as d:
            pt = Path(d) / fname
            torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, pt)
            ReIDModelRegistry.load_pretrained_weights(m, pt)
        for k, v in m.state_dict().items():   # every tensor came from the checkpoint
            assert torch.equal(v, sd[k]), k
        m.eval()
        input_shape = (256, 256) if vehicle else (256, 128)
        out[f"{case}_seed"] = np.int64(seed)
        out[f"{case}_vehicle"] = np.int64(vehicle)
        for mode in MODES:
            be = RefBackend(m, mode, input_shape)
            crops = be.get_crops(boxes, img)
            out[f"{case}_crops_sha256_{mode}"] = hashlib.sha256(np.ascontiguousarray(crops.numpy()).tobytes()).hexdigest()
            out[f"{case}_features_{mode}"] = np.asarray(be.get_features(boxes, img), np.float32)
    np.savez_compressed(HERE / "reid_clip_reference.npz", **out)
    print({k: getattr(v, "shape", v) for k, v in out.items()})


if __name__ == "__main__":
    main()
