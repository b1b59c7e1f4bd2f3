"""Oracle restatement of the MLFN ReID backbone (reid/backbones/mlfn.py, eval mode, groups 32, embed_dim 1024) on the
raw, unfolded state dict -- TEST INFRASTRUCTURE ONLY.  Crops are staged at 256x128 exactly as for OSNet
(oracle/reid.py)."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle.reid import _bn, get_crops

GROUPS = 32
STAGES = ((3, 256), (4, 512), (6, 1024), (3, 2048))   # MLFNBlocks and output width per stage


def _block(sd, name, x, stride):
    """MLFNBlock.forward: (out, s) with s the (N, 32) factor-selection gates."""
    s = x.mean(dim=(2, 3), keepdim=True)
    s = F.relu(_bn(sd, name + ".fsm.2", F.conv2d(s, sd[name + ".fsm.1.weight"], sd[name + ".fsm.1.bias"])))
    s = F.relu(_bn(sd, name + ".fsm.5", F.conv2d(s, sd[name + ".fsm.4.weight"], sd[name + ".fsm.4.bias"])))
    s = torch.sigmoid(_bn(sd, name + ".fsm.8", F.conv2d(s, sd[name + ".fsm.7.weight"], sd[name + ".fsm.7.bias"])))
    y = F.relu(_bn(sd, name + ".fm_bn1", F.conv2d(x, sd[name + ".fm_conv1.weight"])))
    y = F.relu(_bn(sd, name + ".fm_bn2", F.conv2d(y, sd[name + ".fm_conv2.weight"], stride=stride, padding=1,
                                                   groups=GROUPS)))
    y = y * s.flatten(1).repeat_interleave(y.shape[1] // GROUPS, dim=1)[:, :, None, None]   # channel c: s[c // gw]
    y = F.relu(_bn(sd, name + ".fm_bn3", F.conv2d(y, sd[name + ".fm_conv3.weight"])))
    residual = x
    if (name + ".downsample.0.weight") in sd:
        residual = _bn(sd, name + ".downsample.1", F.conv2d(x, sd[name + ".downsample.0.weight"], stride=stride))
    return F.relu(residual + y), s.flatten(1)


@torch.no_grad()
def mlfn_forward(sd, x: torch.Tensor, return_stages: bool = False):
    """x (N,3,256,128) -> (N, 1024) un-normalised embedding v.  Stage taps (NCHW maps, rows otherwise): "stem"
    (conv1 + bn1 + ReLU), "pool", "feature.{i}" after every MLFNBlock, "s_hat" (N, 512) and "v" (N, 1024)."""
    stages = {}
    x = F.relu(_bn(sd, "bn1", F.conv2d(x, sd["conv1.weight"], sd["conv1.bias"], stride=2, padding=3)))
    stages["stem"] = x
    x = F.max_pool2d(x, 3, stride=2, padding=1)
    stages["pool"] = x
    gates, i = [], 0
    for s, (n_blocks, _) in enumerate(STAGES):
        for j in range(n_blocks):
            x, g = _block(sd, f"feature.{i}", x, 2 if (j == 0 and s > 0) else 1)
            gates.append(g)
            stages[f"feature.{i}"] = x
            i += 1
    s_hat = torch.cat(gates, 1)
    stages["s_hat"] = s_hat
    xv = F.relu(_bn(sd, "fc_x.1", F.conv2d(x.mean(dim=(2, 3), keepdim=True), sd["fc_x.0.weight"])))
    sv = F.relu(_bn(sd, "fc_s.1", F.conv2d(s_hat[:, :, None, None], sd["fc_s.0.weight"])))
    v = ((xv + sv) * 0.5).flatten(1)
    stages["v"] = v
    return (v, stages) if return_stages else v


def get_features(sd, xyxys: np.ndarray, img: np.ndarray, preprocess: str = "resize") -> np.ndarray:
    """(N, 1024) float32 L2-normalised embeddings, as BaseModelBackend.get_features returns them."""
    xyxys = np.asarray(xyxys, dtype=np.float32)
    if xyxys.size == 0:
        return np.array([])
    feats = mlfn_forward(sd, get_crops(xyxys, img, preprocess)).numpy()
    return feats / np.linalg.norm(feats, axis=-1, keepdims=True)
