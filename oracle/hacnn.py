"""Oracle restatement of the HACNN ReID backbone (reid/backbones/hacnn.py, eval mode, nchannels 128 / 256 / 384,
feat_dim 512, learn_region=True) on the raw, unfolded state dict -- TEST INFRASTRUCTURE ONLY.  Crops are staged at
160x64 (base_backend.py) with the ImageNet mean / std."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle.lmbn import get_crops_hw
from oracle.reid import _bn

INPUT_HW = (160, 64)
LOCAL_HW = ((24, 28), (12, 14), (6, 7))


def _cb(sd, name, x, stride=1):
    w = sd[name + ".conv.weight"]
    y = F.conv2d(x, w, sd[name + ".conv.bias"], stride=stride, padding=w.shape[-1] // 2)
    return F.relu(_bn(sd, name + ".bn", y))


def inception_a(sd, p, x):
    s = [_cb(sd, f"{p}.stream{i}.1", _cb(sd, f"{p}.stream{i}.0", x)) for i in (1, 2, 3)]
    s.append(_cb(sd, f"{p}.stream4.1", F.avg_pool2d(x, 3, stride=1, padding=1)))   # count_include_pad: / 9
    return torch.cat(s, 1)


def inception_b(sd, p, x):
    s1 = _cb(sd, f"{p}.stream1.1", _cb(sd, f"{p}.stream1.0", x), 2)
    s2 = _cb(sd, f"{p}.stream2.2", _cb(sd, f"{p}.stream2.1", _cb(sd, f"{p}.stream2.0", x)), 2)
    s3 = _cb(sd, f"{p}.stream3.1", F.max_pool2d(x, 3, stride=2, padding=1))
    return torch.cat([s1, s2, s3], 1)


def harm_attn(sd, p, x):
    """HarmAttn.forward: (soft attention map, theta (N, 4, 2))."""
    sp = _cb(sd, p + ".soft_attn.spatial_attn.conv1", x.mean(1, keepdim=True), 2)
    sp = F.interpolate(sp, (sp.shape[2] * 2, sp.shape[3] * 2), mode="bilinear", align_corners=True)
    sp = _cb(sd, p + ".soft_attn.spatial_attn.conv2", sp)
    ch = F.avg_pool2d(x, x.shape[2:])
    ch = _cb(sd, p + ".soft_attn.channel_attn.conv2", _cb(sd, p + ".soft_attn.channel_attn.conv1", ch))
    y = sp * ch
    attn = torch.sigmoid(_cb(sd, p + ".soft_attn.conv", y))   # a ConvBlock: the ReLU comes before the sigmoid
    g = x.mean(dim=(2, 3))
    theta = torch.tanh(F.linear(g, sd[p + ".hard_attn.fc.weight"], sd[p + ".hard_attn.fc.bias"]))
    return attn, theta.view(-1, 4, 2)


def stn(x, theta_r):
    """HACNN.stn with the region's [[1, 0, tx], [0, 0.25, ty]] affine (theta_r (N, 2) = (tx, ty))."""
    th = torch.zeros(x.shape[0], 2, 3, dtype=x.dtype, device=x.device)
    th[:, 0, 0], th[:, 1, 1] = 1.0, 0.25
    th[:, :, 2] = theta_r
    grid = F.affine_grid(th, list(x.shape), align_corners=False)
    return F.grid_sample(x, grid, align_corners=False)


@torch.no_grad()
def hacnn_forward(sd, x: torch.Tensor, return_stages: bool = False):
    """x (N,3,160,64) -> (N, 1024) un-normalised row [fc_global | fc_local].  Stage taps (NCHW maps, rows otherwise):
    "stem", "x1_out" .. "x3_out", "local1" .. "local3" ((N, 4, C, h, w), regions in order), "theta" (N, 3, 8) and
    "v" (N, 1024)."""
    st = {}
    x = _cb(sd, "conv", x, 2)
    st["stem"] = x
    prev, local, thetas = x, None, []
    for i in (1, 2, 3):
        xi = inception_b(sd, f"inception{i}.1", inception_a(sd, f"inception{i}.0", prev))
        attn, theta = harm_attn(sd, f"ha{i}", xi)
        thetas.append(theta.reshape(-1, 8))
        regions = []
        for r in range(4):
            t = F.interpolate(stn(prev, theta[:, r]), LOCAL_HW[i - 1], mode="bilinear", align_corners=True)
            if local is not None:
                t = t + local[r]
            regions.append(inception_b(sd, f"local_conv{i}", t))
        local = regions
        st[f"local{i}"] = torch.stack(regions, 1)
        prev = xi * attn
        st[f"x{i}_out"] = prev
    st["theta"] = torch.stack(thetas, 1)
    xg = F.linear(prev.mean(dim=(2, 3)), sd["fc_global.0.weight"], sd["fc_global.0.bias"])
    xg = F.relu(_bn(sd, "fc_global.1", xg))
    xl = torch.cat([r.mean(dim=(2, 3)) for r in local], 1)
    xl = F.relu(_bn(sd, "fc_local.1", F.linear(xl, sd["fc_local.0.weight"], sd["fc_local.0.bias"])))
    v = torch.cat([xg, xl], 1)
    st["v"] = v
    return (v, st) if return_stages else v


def embed(v: torch.Tensor) -> torch.Tensor:
    """The model's eval output (each half L2-normalised, concatenated), normalised again by get_features."""
    g, l = v[:, :512], v[:, 512:]
    e = torch.cat([g / g.norm(dim=1, keepdim=True), l / l.norm(dim=1, keepdim=True)], 1)
    return e / e.norm(dim=1, keepdim=True)


def get_crops(xyxys: np.ndarray, img: np.ndarray, preprocess: str = "resize") -> torch.Tensor:
    return get_crops_hw(xyxys, img, preprocess, INPUT_HW)


def get_features(sd, xyxys: np.ndarray, img: np.ndarray, preprocess: str = "resize") -> np.ndarray:
    """(N, 1024) float32 L2-normalised embeddings, as BaseModelBackend.get_features returns them."""
    xyxys = np.asarray(xyxys, dtype=np.float32)
    if xyxys.size == 0:
        return np.array([])
    return embed(hacnn_forward(sd, get_crops(xyxys, img, preprocess))).numpy()
