"""Oracle restatement of the CLIP-ReID ViT-B/16 backbone (reid/backbones/clip/make_model.py build_transformer with
clip/config/defaults.py: NECK_FEAT "after", SIE off; clip/clip/model.py VisionTransformer / ResidualAttentionBlock) on
the raw, unfolded state dict -- TEST INFRASTRUCTURE ONLY.  Runs in the dtype of its inputs (float64 for the tests).
Crops are staged at 256x128, or at 256x256 for weights whose file name says `veri` / `vehicleid`
(base_backend.py:57), with mean = std = 0.5 (base_backend.py:52-54)."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle.lmbn import crop_boxes_hw

E = "image_encoder."
WIDTH, HEADS = 768, 12
CLIP_MEAN = CLIP_STD = (0.5, 0.5, 0.5)


def input_hw(sd) -> tuple:
    return (256, 256) if sd[E + "positional_embedding"].shape[0] == 257 else (256, 128)


def get_crops(xyxys: np.ndarray, img: np.ndarray, preprocess: str = "resize", hw=(256, 128)) -> torch.Tensor:
    """float32 NCHW network input (N, 3, H, W), normalised with CLIP's mean / std."""
    u8 = crop_boxes_hw(xyxys, img, preprocess, hw)
    x = torch.from_numpy(u8).to(torch.float32).permute(0, 3, 1, 2).contiguous()
    x = x / 255.0
    return (x - torch.tensor(CLIP_MEAN).view(1, 3, 1, 1)) / torch.tensor(CLIP_STD).view(1, 3, 1, 1)


def _ln(sd, name, x):
    return F.layer_norm(x, (WIDTH,), sd[name + ".weight"], sd[name + ".bias"], eps=1e-5)


def _bn1d(sd, name, x):
    return F.batch_norm(x, sd[name + ".running_mean"], sd[name + ".running_var"], sd[name + ".weight"],
                        sd[name + ".bias"], training=False, eps=1e-5)


def attention(x, w_in, b_in, w_out, b_out):
    """nn.MultiheadAttention(768, 12) self-attention without a mask on x (N, T, 768)."""
    n, t, _ = x.shape
    q, k, v = (x @ w_in.T + b_in).split(WIDTH, dim=-1)
    q, k, v = (z.reshape(n, t, HEADS, WIDTH // HEADS).transpose(1, 2) for z in (q, k, v))
    p = torch.softmax((q * (WIDTH // HEADS) ** -0.5) @ k.transpose(-1, -2), dim=-1)
    o = (p @ v).transpose(1, 2).reshape(n, t, WIDTH)
    return o @ w_out.T + b_out


@torch.no_grad()
def clip_forward(sd, x: torch.Tensor, return_stages: bool = False):
    """x (N, 3, H, W) -> (N, 1280) un-normalised embedding cat(bottleneck(x0), bottleneck_proj(x0 @ proj)), x0 the
    ln_post'ed class token.  Stage taps: "patch" (N, P, 768), "ln_pre" (N, T, 768), "block{i}" (N, T, 768)."""
    stages = {}
    x = F.conv2d(x, sd[E + "conv1.weight"], stride=16).flatten(2).transpose(1, 2)   # (N, P, 768)
    stages["patch"] = x
    cls = sd[E + "class_embedding"].to(x.dtype).expand(x.shape[0], 1, WIDTH)
    x = torch.cat([cls, x], dim=1) + sd[E + "positional_embedding"]
    x = _ln(sd, E + "ln_pre", x)
    stages["ln_pre"] = x
    for i in range(12):
        b = f"{E}transformer.resblocks.{i}."
        x = x + attention(_ln(sd, b + "ln_1", x), sd[b + "attn.in_proj_weight"], sd[b + "attn.in_proj_bias"],
                          sd[b + "attn.out_proj.weight"], sd[b + "attn.out_proj.bias"])
        h = _ln(sd, b + "ln_2", x) @ sd[b + "mlp.c_fc.weight"].T + sd[b + "mlp.c_fc.bias"]
        h = h * torch.sigmoid(1.702 * h)
        x = x + h @ sd[b + "mlp.c_proj.weight"].T + sd[b + "mlp.c_proj.bias"]
        stages[f"block{i}"] = x
    x0 = _ln(sd, E + "ln_post", x)[:, 0]
    v = torch.cat([_bn1d(sd, "bottleneck", x0), _bn1d(sd, "bottleneck_proj", x0 @ sd[E + "proj"])], dim=1)
    stages["feature"] = v
    return (v, stages) if return_stages else v


def attention_row_max(sd, x: torch.Tensor, block: int = 0) -> torch.Tensor:
    """Largest softmax probability of every attention row of `block` (N, heads, T): 1/T for uniform attention."""
    with torch.no_grad():
        _, st = clip_forward(sd, x, return_stages=True)
        h = st["ln_pre"] if block == 0 else st[f"block{block - 1}"]
        b = f"{E}transformer.resblocks.{block}."
        n, t, _ = h.shape
        q, k, _ = (_ln(sd, b + "ln_1", h) @ sd[b + "attn.in_proj_weight"].T + sd[b + "attn.in_proj_bias"]).split(WIDTH, -1)
        q, k = (z.reshape(n, t, HEADS, 64).transpose(1, 2) for z in (q, k))
        return torch.softmax((q / 8) @ k.transpose(-1, -2), dim=-1).amax(-1)


def double_state(sd):
    return {k: v.double() for k, v in sd.items() if torch.is_floating_point(v)}


def get_features(sd, xyxys: np.ndarray, img: np.ndarray, preprocess: str = "resize") -> np.ndarray:
    """(N, 1280) float32 L2-normalised embeddings, as BaseModelBackend.get_features returns them (computed in
    float64 from the float32 crops)."""
    xyxys = np.asarray(xyxys, dtype=np.float32)
    if xyxys.size == 0:
        return np.array([])
    x = get_crops(xyxys, img, preprocess, input_hw(sd)).double()
    feats = clip_forward(double_state(sd), x).numpy()
    return (feats / np.linalg.norm(feats, axis=-1, keepdims=True)).astype(np.float32)


class OracleCLIP:
    """Minimal `reid_model` object for the oracle trackers (get_features only)."""

    def __init__(self, sd, preprocess: str = "resize"):
        self.sd = double_state(sd)
        self.preprocess = preprocess

    def get_features(self, xyxys, img):
        return get_features(self.sd, xyxys, img, self.preprocess)
