"""Oracle restatement of the ViT-Nano / ViT-Tiny ReID family (reid/backbones/vit_nano.py ViTNano, vit_tiny.py
ViTTinyParts, eval mode) on the raw, unfolded state dict -- TEST INFRASTRUCTURE ONLY.  Runs in the dtype of its inputs
(float64 for the tests).  Crops are staged at 384x128 for vit_tiny* and 256x128 otherwise (base_backend.py:56-64),
with ImageNet's mean / std."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from boxmot_b200.weights import VIT_VARIANTS, vit_grid
from oracle.lmbn import crop_boxes_hw

D, HEADS = 192, 3
MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def input_hw(variant) -> tuple:
    return vit_grid(variant)[:2]


def get_crops(xyxys: np.ndarray, img: np.ndarray, preprocess: str = "resize", hw=(256, 128)) -> torch.Tensor:
    """float32 NCHW network input (N, 3, H, W), normalised with ImageNet's mean / std."""
    u8 = crop_boxes_hw(xyxys, img, preprocess, hw)
    x = torch.from_numpy(u8).to(torch.float32).permute(0, 3, 1, 2).contiguous()
    x = x / 255.0
    return (x - torch.tensor(MEAN).view(1, 3, 1, 1)) / torch.tensor(STD).view(1, 3, 1, 1)


def _ln(sd, name, x):
    return F.layer_norm(x, (D,), sd[name + ".weight"], sd[name + ".bias"], eps=1e-5)


def _bn1d(sd, name, x):
    return F.batch_norm(x, sd[name + ".running_mean"], sd[name + ".running_var"], sd[name + ".weight"],
                        sd[name + ".bias"], training=False, eps=1e-5)


def ain(sd, name, x):
    """AdaptiveINLN: sigmoid(gate) * InstanceNorm1d over the tokens + (1 - sigmoid(gate)) * LayerNorm."""
    ln = _ln(sd, name + ".ln", x)
    xin = F.instance_norm(x.transpose(1, 2), weight=sd[name + ".in_norm.weight"], bias=sd[name + ".in_norm.bias"],
                          eps=1e-5).transpose(1, 2)
    g = torch.sigmoid(sd[name + ".gate"])
    return g * xin + (1.0 - g) * ln


def attention(x, w_qkv, b_qkv, w_proj, b_proj):
    n, t, _ = x.shape
    q, k, v = (x @ w_qkv.T + b_qkv).reshape(n, t, 3, HEADS, D // HEADS).permute(2, 0, 3, 1, 4)
    p = torch.softmax((q @ k.transpose(-1, -2)) * (D // HEADS) ** -0.5, dim=-1)
    return (p @ v).transpose(1, 2).reshape(n, t, D) @ w_proj.T + b_proj


def omni_scale(sd, patch, gh, gw):
    """OmniScaleAggregation over the patch tokens (N, P, 192) on a gh x gw grid."""
    n = patch.shape[0]
    spatial = patch.transpose(1, 2).reshape(n, D, gh, gw)
    fused = torch.zeros(n, D, dtype=patch.dtype, device=patch.device)
    for i, s in enumerate((1, 2, 4, 8)):
        p = F.adaptive_avg_pool2d(spatial, (s, 1)).squeeze(-1).mean(dim=-1)
        p = _ln(sd, f"os_agg.scale_norms.{i}", p)
        h = torch.relu(p @ sd["os_agg.gate.fc.0.weight"].T + sd["os_agg.gate.fc.0.bias"])
        g = torch.sigmoid(h @ sd["os_agg.gate.fc.2.weight"].T + sd["os_agg.gate.fc.2.bias"])
        fused = fused + g * p
    return fused


@torch.no_grad()
def vit_forward(sd, variant, x: torch.Tensor, return_stages: bool = False):
    """x (N, 3, H, W) -> the un-normalised embedding of `variant`.  Stage taps: "patch" (N, P, 192), "tokens"
    (N, T, 192), "block{i}" (N, T, 192), "norm" (N, T, 192), "feature"."""
    depth, n_ain, omni, parts, *_ = VIT_VARIANTS[variant]
    _, _, stride, gh, gw, _ = vit_grid(variant)
    stages = {}
    x = F.conv2d(x, sd["patch_embed.proj.weight"], sd["patch_embed.proj.bias"], stride=stride)
    x = x.flatten(2).transpose(1, 2)
    stages["patch"] = x
    cls = sd["cls_token"].to(x.dtype).expand(x.shape[0], -1, -1)
    x = torch.cat([cls, x], dim=1) + sd["pos_embed"]
    stages["tokens"] = x
    for i in range(depth):
        b = f"blocks.{i}."
        y = ain(sd, b + "norm1", x) if i < n_ain else _ln(sd, b + "norm1", x)
        x = x + attention(y, sd[b + "attn.qkv.weight"], sd[b + "attn.qkv.bias"], sd[b + "attn.proj.weight"],
                          sd[b + "attn.proj.bias"])
        h = _ln(sd, b + "norm2", x) @ sd[b + "mlp.fc1.weight"].T + sd[b + "mlp.fc1.bias"]
        x = x + F.gelu(h) @ sd[b + "mlp.fc2.weight"].T + sd[b + "mlp.fc2.bias"]
        stages[f"block{i}"] = x
    x = _ln(sd, "norm", x)
    stages["norm"] = x
    if omni:
        v = omni_scale(sd, x[:, 1:], gh, gw)
    else:
        v = x[:, 0]
    if "proj.weight" in sd:
        v = v @ sd["proj.weight"].T
    feats = [_bn1d(sd, "bottleneck", v)]
    if parts:
        spatial = x[:, 1:].transpose(1, 2).reshape(x.shape[0], D, gh, gw)
        sh = gh // parts
        for i in range(parts):
            h1 = (i + 1) * sh if i < parts - 1 else gh
            p = spatial[:, :, i * sh:h1, :].mean(dim=[2, 3])
            feats.append(_bn1d(sd, f"part_bns.{i}", p @ sd[f"part_projs.{i}.weight"].T))
    v = torch.cat(feats, dim=1)
    stages["feature"] = v
    return (v, stages) if return_stages else v


def attention_row_max(sd, variant, x: torch.Tensor, block: int = 0) -> torch.Tensor:
    """Largest softmax probability of every attention row of `block` (N, heads, T): 1/T for uniform attention."""
    _, st = vit_forward(sd, variant, x, return_stages=True)
    h = st["tokens"] if block == 0 else st[f"block{block - 1}"]
    b = f"blocks.{block}."
    y = ain(sd, b + "norm1", h) if block < VIT_VARIANTS[variant][1] else _ln(sd, b + "norm1", h)
    n, t, _ = y.shape
    q, k, _ = (y @ sd[b + "attn.qkv.weight"].T + sd[b + "attn.qkv.bias"]).reshape(n, t, 3, HEADS, 64).permute(2, 0, 3, 1, 4)
    return torch.softmax((q / 8) @ k.transpose(-1, -2), dim=-1).amax(-1)


def double_state(sd):
    return {k: v.double() for k, v in sd.items() if torch.is_floating_point(v)}


def get_features(sd, variant, xyxys: np.ndarray, img: np.ndarray, preprocess: str = "resize") -> np.ndarray:
    """(N, row) float32 L2-normalised embeddings, as BaseModelBackend.get_features returns them (computed in float64
    from the float32 crops)."""
    xyxys = np.asarray(xyxys, dtype=np.float32)
    if xyxys.size == 0:
        return np.array([])
    x = get_crops(xyxys, img, preprocess, input_hw(variant)).double()
    feats = vit_forward(double_state(sd), variant, x).numpy()
    return (feats / np.linalg.norm(feats, axis=-1, keepdims=True)).astype(np.float32)
