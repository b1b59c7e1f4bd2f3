"""Oracle restatement of the Bottleneck ResNet ReID backbones resnet50 / resnet101 (reid/backbones/resnet.py, eval mode,
last_stride 2, no fc: the embedding is the 2048-d average pool of layer4) on the raw, unfolded state dict -- TEST
INFRASTRUCTURE ONLY.  Crops are staged at 256x128 exactly as for OSNet (oracle/reid.py)."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle.reid import _bn, get_crops

RESNET_BLOCKS = {50: (3, 4, 6, 3), 101: (3, 4, 23, 3)}


def resnet_depth(sd) -> int:
    n3 = len({k.split(".")[1] for k in sd if k.startswith("layer3.")})
    return next(d for d, b in RESNET_BLOCKS.items() if b[2] == n3)


def is_resnet(sd) -> bool:
    return "conv1.weight" in sd and "layer1.0.conv1.weight" in sd


def _bottleneck(sd, name, x, stride):
    out = F.relu(_bn(sd, name + ".bn1", F.conv2d(x, sd[name + ".conv1.weight"])))
    out = F.relu(_bn(sd, name + ".bn2", F.conv2d(out, sd[name + ".conv2.weight"], stride=stride, padding=1)))
    out = _bn(sd, name + ".bn3", F.conv2d(out, sd[name + ".conv3.weight"]))
    identity = x
    if (name + ".downsample.0.weight") in sd:
        identity = _bn(sd, name + ".downsample.1", F.conv2d(x, sd[name + ".downsample.0.weight"], stride=stride))
    return F.relu(out + identity)


@torch.no_grad()
def resnet_forward(sd, x: torch.Tensor, return_stages: bool = False):
    """x (N,3,256,128) float32 -> (N, 2048) un-normalised embedding.  Stage taps (NCHW): "stem" (conv1 + bn1 + ReLU),
    "pool" (max pool), "layer{l}.{j}" after every Bottleneck, and "feature" (the average pool)."""
    stages = {}
    x = F.relu(_bn(sd, "bn1", F.conv2d(x, sd["conv1.weight"], stride=2, padding=3)))
    stages["stem"] = x
    x = F.max_pool2d(x, 3, stride=2, padding=1)
    stages["pool"] = x
    for li, n_blocks in enumerate(RESNET_BLOCKS[resnet_depth(sd)]):
        for j in range(n_blocks):
            name = f"layer{li + 1}.{j}"
            x = _bottleneck(sd, name, x, 2 if (j == 0 and li > 0) else 1)
            stages[name] = x
    v = F.adaptive_avg_pool2d(x, 1).flatten(1)
    stages["feature"] = v
    return (v, stages) if return_stages else v


def get_features(sd, xyxys: np.ndarray, img: np.ndarray, preprocess: str = "resize") -> np.ndarray:
    """(N, 2048) float32 L2-normalised embeddings, as BaseModelBackend.get_features returns them."""
    xyxys = np.asarray(xyxys, dtype=np.float32)
    if xyxys.size == 0:
        return np.array([])
    feats = resnet_forward(sd, get_crops(xyxys, img, preprocess)).numpy()
    return feats / np.linalg.norm(feats, axis=-1, keepdims=True)


class OracleResNet:
    """Minimal `reid_model` object for the oracle trackers (get_features only)."""

    def __init__(self, sd, preprocess: str = "resize"):
        self.sd = sd
        self.preprocess = preprocess

    def get_features(self, xyxys, img):
        return get_features(self.sd, xyxys, img, self.preprocess)
