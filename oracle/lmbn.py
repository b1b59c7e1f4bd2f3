"""Oracle restatement of LMBN_n (reid/backbones/lmbn/lmbn_n.py, eval mode) and of its 384x128 crop staging
(reid/backends/base_backend.py:59-60) -- TEST INFRASTRUCTURE ONLY.  Built on the OSNet pieces of oracle/reid.py: the
trunk and the three branches are OSNet_x1_0 OSBlocks and transitions; the head restates lmbn_n.py:96-146 with
bnneck.py's BNNeck3 / BNNeck (1x1 conv + BatchNorm1d, BatchNorm1d) and attention.py's BatchDropTop (identity in eval).
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle.reid import INPUT_HW, MEAN, STD, OracleReID, _bn, _osblock, get_features, resize_linear_u8, resize_pad_u8

LMBN_INPUT_HW = (384, 128)
LMBN_BRANCHES = ("global_branch", "partial_branch", "channel_branch")


def crop_boxes_hw(xyxys: np.ndarray, img: np.ndarray, preprocess: str = "resize", input_hw=INPUT_HW):
    """`crop_boxes` at any network input size: uint8 RGB crops (N, H, W, 3)."""
    h, w = img.shape[:2]
    th, tw = input_hw
    xyxys = np.asarray(xyxys, dtype=np.float32).reshape(-1, 4)
    out = np.zeros((len(xyxys), th, tw, 3), np.uint8)
    for i, box in enumerate(xyxys):
        x1, y1, x2, y2 = box.round().astype("int")
        cx1, cy1 = max(0, x1), max(0, y1)
        cx2, cy2 = min(w, x2), min(h, y2)
        if cx2 > cx1 and cy2 > cy1:
            fn = resize_pad_u8 if preprocess == "resize_pad" else resize_linear_u8
            crop = fn(img[cy1:cy2, cx1:cx2], th, tw)
        else:
            crop = np.zeros((th, tw, 3), np.uint8)
        out[i] = crop[:, :, ::-1]
    return out


def get_crops_hw(xyxys: np.ndarray, img: np.ndarray, preprocess: str = "resize", input_hw=INPUT_HW) -> torch.Tensor:
    """`get_crops` at any network input size: float32 NCHW (N, 3, H, W)."""
    u8 = crop_boxes_hw(xyxys, img, preprocess, input_hw)
    x = torch.from_numpy(u8).to(torch.float32).permute(0, 3, 1, 2).contiguous()
    x = x / 255.0
    mean = torch.tensor(MEAN).view(1, 3, 1, 1)
    std = torch.tensor(STD).view(1, 3, 1, 1)
    return (x - mean) / std


def is_lmbn_n(sd) -> bool:
    return "backone.0.conv.weight" in sd


def _transition(sd, name, x):
    return F.avg_pool2d(F.relu(_bn(sd, name + ".bn", F.conv2d(x, sd[name + ".conv.weight"]))), 2, stride=2)


@torch.no_grad()
def lmbn_n_forward(sd, x: torch.Tensor, return_stages: bool = False):
    """x (N,3,384,128) float32 -> (N, 3584) un-normalised LMBN_n embedding (eval mode).  Stage taps (NCHW): stem, pool,
    backone.2.0, backone.2.1, backone.2.2, trunk, and per branch <name>.0.1, .0.2, .1.0, .1.1, .2, plus bottleneck."""
    stages = {}
    x = F.relu(_bn(sd, "backone.0.bn", F.conv2d(x, sd["backone.0.conv.weight"], stride=2, padding=3)))
    stages["stem"] = x
    x = F.max_pool2d(x, 3, stride=2, padding=1)
    stages["pool"] = x
    x = _osblock(sd, "backone.2.0", x)
    stages["backone.2.0"] = x
    x = _osblock(sd, "backone.2.1", x)
    stages["backone.2.1"] = x
    x = _transition(sd, "backone.2.2.0", x)
    stages["backone.2.2"] = x
    trunk = _osblock(sd, "backone.3", x)
    stages["trunk"] = trunk
    outs = {}
    for br in LMBN_BRANCHES:
        y = _osblock(sd, f"{br}.0.1", trunk)
        stages[f"{br}.0.1"] = y
        y = _transition(sd, f"{br}.0.2.0", y)
        stages[f"{br}.0.2"] = y
        y = _osblock(sd, f"{br}.1.0", y)
        stages[f"{br}.1.0"] = y
        y = _osblock(sd, f"{br}.1.1", y)
        stages[f"{br}.1.1"] = y
        y = F.relu(_bn(sd, f"{br}.2.bn", F.conv2d(y, sd[f"{br}.2.conv.weight"])))
        stages[f"{br}.2"] = y
        outs[br] = y
    # BatchFeatureErase_Top in eval: the bottleneck OSBlock, and BatchDropTop is the identity, so glo == glo_drop
    glo = _osblock(sd, "batch_drop_block.drop_batch_bottleneck", outs["global_branch"])
    stages["bottleneck"] = glo
    par, cha = outs["partial_branch"], outs["channel_branch"]
    h = par.shape[2]
    pooled = [F.adaptive_avg_pool2d(glo, 1), F.adaptive_max_pool2d(glo, 1), F.adaptive_max_pool2d(par, 1),
              par[:, :, : h // 2].mean(dim=(2, 3), keepdim=True), par[:, :, h // 2:].mean(dim=(2, 3), keepdim=True)]
    necks = (0, 4, 1, 2, 3)   # f_glo, f_glo_drop, f_p0, f_p1, f_p2
    feats = [_bn(sd, f"reduction_{k}.bn", F.conv2d(p, sd[f"reduction_{k}.reduction.weight"]).flatten(1))
             for k, p in zip(necks, pooled)]
    cha = F.adaptive_avg_pool2d(cha, 1)
    for j, half in enumerate((cha[:, :256], cha[:, 256:])):
        c = F.relu(_bn(sd, "shared.1", F.conv2d(half, sd["shared.0.weight"]))).flatten(1)
        feats.append(_bn(sd, f"reduction_ch_{j}.bn", c))
    v = torch.stack(feats, dim=2).flatten(1, 2)   # element c*7 + k = channel c of vector k
    return (v, stages) if return_stages else v


def lmbn_get_features(sd, xyxys: np.ndarray, img: np.ndarray, preprocess: str = "resize") -> np.ndarray:
    """(N, 3584) float32 L2-normalised LMBN_n embeddings of 384x128 crops."""
    xyxys = np.asarray(xyxys, dtype=np.float32)
    if xyxys.size == 0:
        return np.array([])
    feats = lmbn_n_forward(sd, get_crops_hw(xyxys, img, preprocess, LMBN_INPUT_HW)).numpy()
    return feats / np.linalg.norm(feats, axis=-1, keepdims=True)


def get_features_any(sd, xyxys: np.ndarray, img: np.ndarray, preprocess: str = "resize") -> np.ndarray:
    """`get_features` for every backbone the oracle restates (LMBN_n at 384x128, the others at 256x128)."""
    fn = lmbn_get_features if is_lmbn_n(sd) else get_features
    return fn(sd, xyxys, img, preprocess)


class OracleReIDAny(OracleReID):
    """`OracleReID` for every backbone the oracle restates."""

    def get_features(self, xyxys, img):
        return get_features_any(self.sd, xyxys, img)
