"""Oracle restatement of the OSNet networks with instance norms -- TEST INFRASTRUCTURE ONLY.

Follows (relative to /root/reference/boxmot):
  * reid/backbones/osnet_ain.py  ConvLayer(IN=True) stem, OSBlock / OSBlockINin (IN on conv3's output, before the
    residual add), OSNet with `conv1_IN=True`, blocks [[INin, INin], [OSBlock, INin], [INin, OSBlock]], transitions
    pool2 / pool3 (osnet_ain_x1_0 / _x0_75 / _x0_5 / _x0_25)
  * reid/backbones/osnet.py:215-262,548  OSBlock(IN=True) (IN after the residual add, conv2.0 / conv2.1) and the IN stem
    of osnet_ibn_x1_0
InstanceNorm2d(affine=True, track_running_stats=False): per crop and channel, biased variance over H x W, eps 1e-5.
Built on oracle/reid.py's `_bn` / `_light` / `_gate` and crop staging; stage taps are named as in `osnet_forward`.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from boxmot_b200.synthetic import OSNET_AIN_ININ
from oracle import reid
from oracle.reid import OracleReID, _bn, _gate, _light, _osblock, get_crops


def _in(sd, name, x):
    return F.instance_norm(x, weight=sd[name + ".weight"], bias=sd[name + ".bias"], eps=1e-5)


def is_osnet_ain(sd) -> bool:
    return "pool2.0.conv.weight" in sd


def is_osnet_ibn(sd) -> bool:
    return "conv1.conv.weight" in sd and "conv2.0.IN.weight" in sd and "pool2.0.conv.weight" not in sd


def _ain_block(sd, name, x, inin):
    identity = x
    x1 = F.relu(_bn(sd, name + ".conv1.bn", F.conv2d(x, sd[name + ".conv1.conv.weight"])))
    x2 = 0
    for t in range(4):
        y = x1
        for i in range(t + 1):
            y = _light(sd, f"{name}.conv2.{t}.layers.{i}", y)
        x2 = x2 + _gate(sd, name + ".gate", y)
    x3 = F.conv2d(x2, sd[name + ".conv3.conv.weight"])
    x3 = _in(sd, name + ".IN", x3) if inin else _bn(sd, name + ".conv3.bn", x3)
    if (name + ".downsample.conv.weight") in sd:
        identity = _bn(sd, name + ".downsample.bn", F.conv2d(identity, sd[name + ".downsample.conv.weight"]))
    return F.relu(x3 + identity)


def _ibn_block(sd, name, x):
    identity = x
    x1 = F.relu(_bn(sd, name + ".conv1.bn", F.conv2d(x, sd[name + ".conv1.conv.weight"])))
    branches = [_light(sd, name + ".conv2a", x1)]
    for br, depth in (("conv2b", 2), ("conv2c", 3), ("conv2d", 4)):
        y = x1
        for k in range(depth):
            y = _light(sd, f"{name}.{br}.{k}", y)
        branches.append(y)
    x2 = sum(_gate(sd, name + ".gate", b) for b in branches)
    x3 = _bn(sd, name + ".conv3.bn", F.conv2d(x2, sd[name + ".conv3.conv.weight"]))
    if (name + ".downsample.conv.weight") in sd:
        identity = _bn(sd, name + ".downsample.bn", F.conv2d(identity, sd[name + ".downsample.conv.weight"]))
    return F.relu(_in(sd, name + ".IN", x3 + identity))


def _head(sd, x, stages, return_stages):
    x = F.relu(_bn(sd, "conv5.bn", F.conv2d(x, sd["conv5.conv.weight"])))
    stages["conv5"] = x
    v = F.adaptive_avg_pool2d(x, 1).flatten(1)
    v = F.relu(_bn(sd, "fc.1", F.linear(v, sd["fc.0.weight"], sd["fc.0.bias"])))
    return (v, stages) if return_stages else v


def _stem(sd, x, stages):
    x = F.relu(_in(sd, "conv1.bn", F.conv2d(x, sd["conv1.conv.weight"], stride=2, padding=3)))
    stages["stem"] = x
    x = F.max_pool2d(x, 3, stride=2, padding=1)
    stages["pool"] = x
    return x


@torch.no_grad()
def osnet_ain_forward(sd, x: torch.Tensor, return_stages: bool = False):
    """x (N,3,256,128) float32 -> (N, 512) un-normalised osnet_ain embedding (eval mode).  Taps (NCHW): stem (after
    IN + ReLU), pool, conv{2,3,4}.{0,1}, the transitions conv2.2 / conv3.2 (pool2 / pool3) and conv5."""
    stages = {}
    x = _stem(sd, x, stages)
    for s in range(3):
        for j in range(2):
            x = _ain_block(sd, f"conv{s + 2}.{j}", x, OSNET_AIN_ININ[s][j])
            stages[f"conv{s + 2}.{j}"] = x
        if s < 2:
            x = F.relu(_bn(sd, f"pool{s + 2}.0.bn", F.conv2d(x, sd[f"pool{s + 2}.0.conv.weight"])))
            x = F.avg_pool2d(x, 2, stride=2)
            stages[f"conv{s + 2}.2"] = x
    return _head(sd, x, stages, return_stages)


@torch.no_grad()
def osnet_ibn_forward(sd, x: torch.Tensor, return_stages: bool = False):
    """x (N,3,256,128) float32 -> (N, 512) un-normalised osnet_ibn_x1_0 embedding (eval mode); taps as osnet_ain_forward."""
    stages = {}
    x = _stem(sd, x, stages)
    for s in range(3):
        for j in range(2):
            name = f"conv{s + 2}.{j}"
            x = _ibn_block(sd, name, x) if (name + ".IN.weight") in sd else _osblock(sd, name, x)
            stages[name] = x
        if s < 2:
            x = F.relu(_bn(sd, f"conv{s + 2}.2.0.bn", F.conv2d(x, sd[f"conv{s + 2}.2.0.conv.weight"])))
            x = F.avg_pool2d(x, 2, stride=2)
            stages[f"conv{s + 2}.2"] = x
    return _head(sd, x, stages, return_stages)


def osnet_in_forward(sd, x, return_stages: bool = False):
    fn = osnet_ain_forward if is_osnet_ain(sd) else osnet_ibn_forward
    return fn(sd, x, return_stages)


def get_features_in(sd, xyxys: np.ndarray, img: np.ndarray, preprocess: str = "resize") -> np.ndarray:
    """(N, 512) float32 L2-normalised embeddings of an OSNet-AIN / OSNet-IBN state dict."""
    xyxys = np.asarray(xyxys, dtype=np.float32)
    if xyxys.size == 0:
        return np.array([])
    feats = osnet_in_forward(sd, get_crops(xyxys, img, preprocess)).numpy()
    return feats / np.linalg.norm(feats, axis=-1, keepdims=True)


def get_features(sd, xyxys: np.ndarray, img: np.ndarray, preprocess: str = "resize") -> np.ndarray:
    """`get_features` dispatching on the state dict: OSNet-AIN / OSNet-IBN here, every other backbone in oracle.reid."""
    if is_osnet_ain(sd) or is_osnet_ibn(sd):
        return get_features_in(sd, xyxys, img, preprocess)
    return reid.get_features(sd, xyxys, img, preprocess)


class OracleReIDIn(OracleReID):
    """`OracleReID` for the OSNet networks with instance norms (and every backbone of oracle.reid)."""

    def get_features(self, xyxys, img):
        return get_features(self.sd, xyxys, img)
