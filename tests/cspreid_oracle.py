"""Float64 functional restatement of the reference's CSPReID_n (reid/backbones/cspreid_n.py, eval mode) on its state
dict, with the stage outputs the device path taps.  No folding: every BatchNorm runs as written, so comparing this
against the folded blob checks the fold as well as the kernels.

Taps (NHWC per crop, as `boxmot_b200_reid_debug_stage` returns them): 0 crop (H, W, 3), 1 stem (H/4, W/4, 64),
2-4 stage1..3 after their downsample (H/8 x 128, H/16 x 256, H/32 x 384), 5 stage4's C3k2 (512), 6 SPPF (512),
7 LightSelfAttention (512), 8 the interleaved 1536-d head row before the L2 norm.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from boxmot_b200.weights import CSPREID_HEADS, CSPREID_STAGES

EPS = 1e-5
TAPS = 9


def double_state(sd):
    return {k: (v.double() if torch.is_tensor(v) and v.is_floating_point() else v) for k, v in sd.items()}


def _bn(sd, name, x):
    return F.batch_norm(x, sd[name + ".running_mean"], sd[name + ".running_var"], sd[name + ".weight"],
                        sd[name + ".bias"], False, 0.0, EPS)


def _cbs(sd, name, x, stride=1):
    w = sd[name + ".conv.weight"]
    return F.silu(_bn(sd, name + ".bn", F.conv2d(x, w, None, stride, w.shape[-1] // 2)))


def _c3k2(sd, name, x, n):
    y = _cbs(sd, name + ".cv1", x)
    outs = list(y.chunk(2, dim=1))
    cur = outs[-1]
    for i in range(n):
        b = f"{name}.bottlenecks.{i}"
        cur = cur + _cbs(sd, b + ".cv2", _cbs(sd, b + ".cv1", cur))
        outs.append(cur)
    return _cbs(sd, name + ".cv2", torch.cat(outs, dim=1))


def sppf(sd, name, x):
    x = _cbs(sd, name + ".cv1", x)
    y1 = F.max_pool2d(x, 3, 1, 1)
    y2 = F.max_pool2d(y1, 3, 1, 1)
    y3 = F.max_pool2d(y2, 3, 1, 1)
    return _cbs(sd, name + ".cv2", torch.cat([x, y1, y2, y3], dim=1))


def attention(sd, name, x):
    ca = torch.sigmoid(F.conv2d(F.silu(F.conv2d(x.mean(dim=(2, 3), keepdim=True), sd[name + ".fc.0.weight"])),
                                sd[name + ".fc.2.weight"]))
    x = x * ca
    d = F.conv2d(x, sd[name + ".spatial.0.weight"], None, 1, 1, 1, x.shape[1])
    sa = torch.sigmoid(F.conv2d(F.silu(_bn(sd, name + ".spatial.1", d)), sd[name + ".spatial.3.weight"]))
    return x * sa


def head(sd, x):
    """x (n, 512, h, w) -> the interleaved (n, 1536) row before the L2 norm: element 3 c + branch."""
    g = F.adaptive_avg_pool2d(x, (1, 1))
    p = F.adaptive_avg_pool2d(x, (2, 1))
    outs = []
    for h, v in zip(CSPREID_HEADS, (g, p[:, :, 0:1], p[:, :, 1:2])):
        r = F.conv2d(v, sd[f"head.{h}.reduction.weight"]).flatten(1)
        outs.append(_bn(sd, f"head.{h}.bn", r))
    return torch.stack(outs, dim=2).flatten(1, 2)


def forward_taps(sd, x):
    """x (n, 3, H, W) float64, already normalised -> [tap 0 .. 8] as NCHW tensors (the head row as (n, 1536))."""
    taps = [x]
    x = _cbs(sd, "stem.1", _cbs(sd, "stem.0", x, 2), 2)
    taps.append(x)
    for s, (_, _, n) in enumerate(CSPREID_STAGES[:3], 1):
        x = _cbs(sd, f"stage{s}.1", _c3k2(sd, f"stage{s}.0", x, n), 2)
        taps.append(x)
    x = _c3k2(sd, "stage4.0", x, CSPREID_STAGES[3][2])
    taps.append(x)
    x = sppf(sd, "stage4.1", x)
    taps.append(x)
    x = attention(sd, "stage4.2", x)
    taps.append(x)
    taps.append(head(sd, x))
    return taps


def embed(sd, x):
    """L2-normalised rows, as the reference's get_features returns them."""
    return F.normalize(forward_taps(sd, x)[-1], dim=1)


def nhwc(t):
    """A tap as the device stores it per crop: NHWC, flattened."""
    return (t.permute(0, 2, 3, 1) if t.dim() == 4 else t).reshape(t.shape[0], -1)
