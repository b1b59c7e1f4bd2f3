"""ReID weight preparation: reference state dict (.pt) -> BN-folded `.b200reid` blob for the CUDA kernels.

Plays the role of the reference's automatic `.pt -> .onnx` export for its native ReID path
(boxmot/native/_common.py:453-570) and of its checkpoint loader (boxmot/reid/core/registry.py:126-164:
unwrap `state_dict`, strip `module.`).  Pure tensor plumbing on the host; no inference happens here.

Blob layout (little endian): 16 int32 header words
    [magic 'B2RE', version, arch (1 = OSNet), c0, c1, c2, c3, feat_dim, n_floats, 0...]
followed by float32 parameters in the exact order csrc/reid_model.cu walks them:
    stem      W[147][c0] (k = (kh*7+kw)*3 + ci, BN folded), b[c0]
    per stage s=0..2, per block j=0..1 (cin, cout, mid = cout/4, hid = mid/16):
        conv1      W[cin][mid], b[mid]
        10 x light (a0 | b0 b1 | c0 c1 c2 | d0 d1 d2 d3):  pw W[mid][mid], dw W[9][mid] (BN folded), b[mid]
        gate       fc1 W[mid][hid], b[hid], fc2 W[hid][mid], b[mid]
        combine    W[mid (+ cin if downsample)][cout]  (conv3 rows, then downsample rows), b[cout] (summed)
      transition (s < 2)  W[cout][cout], b[cout]
    conv5     W[c3][c3], b[c3]
    fc        W[c3][feat] (BatchNorm1d folded), b[feat]
Arch 3 (LMBN_n, `fold_lmbn_n`) keeps the OSNet header dims (64, 256, 384, 512, feat 3584) and records the input
height (384) in header word 9; its tensors reuse the OSBlock / transition layouts above.
Arch 4 (OSNet-AIN / OSNet-IBN, `fold_osnet_in`) keeps the arch-1 layout and header dims; header word 9 flags the
stem's instance norm and words 10-15 hold each block's IN placement (0 none, 1 before the residual add, 2 after it),
with the gamma / beta arrays stored right after the tensors of the stem or block they belong to.
Arch 5 (Bottleneck ResNet50 / ResNet101, `fold_resnet`) records the Bottleneck counts of layer1..4 in words 3-6 and
the 2048-d feature in word 7; its layout is listed above `fold_resnet`.
Arch 6 (CLIP-ReID ViT-B/16, `fold_clip`) records width, layers, heads, the 512-d projection and the 1280-d feature
in words 3-7, the input height / width in words 9-10 and the patch grid in words 11-12; its layout is listed above
`fold_clip`.
Arch 7 (MLFN, `fold_mlfn`) records the stem width, the last block width, the groups, the block count and the 1024-d
feature in words 3-7; its layout is listed above `fold_mlfn`.
Arch 8 (HACNN, `fold_hacnn`) records the stem width and the three Inception widths and the 1024-d feature in words
3-7 and the 160x64 input in words 9-10; its layout is listed above `fold_hacnn`.
Arch 9 (ViT-Nano / ViT-Tiny, `fold_vit`) records width 192, depth, 3 heads, the AIN block count and the row width in
words 3-7, the crop height / width in words 9-10, the patch grid in words 11-12, the patch stride in word 13, the
pooling (0 class token, 1 omni-scale, P >= 2 class token + P strips) in word 14 and the projection width (0 or 512)
in word 15; its layout is listed above `fold_vit`.
Arch 10 (CSPReID-n, `fold_cspreid`) records the stage widths 128, 256, 384, 512 and the 1536-d row in words 3-7 and the
crop height / width (256x128, or 256x256 for a vehicle file name) in words 9-10; its layout is listed above
`cspreid_layout`.
All 1x1 weights are stored K-major ([cin][cout]) so a thread owning consecutive output channels loads
consecutive floats; every tensor is zero-padded to a multiple of 4 floats (16-byte aligned float4 loads).
"""
from __future__ import annotations

import hashlib
import struct
from pathlib import Path
from typing import Dict, List, Tuple

import numpy as np

MAGIC = 0x45523242  # 'B2RE'
VERSION = 1
ARCH_OSNET = 1
ARCH_MOBILENETV2 = 2
ARCH_LMBN_N = 3
ARCH_OSNET_IN = 4
ARCH_RESNET = 5
RESNET_FEAT = 2048
ARCH_CLIP = 6
ARCH_MLFN = 7
MLFN_FEAT = 1024
ARCH_HACNN = 8
HACNN_FEAT = 1024
ARCH_VIT = 9
ARCH_CSPREID = 10
BRANCHES = (("conv2a", 1), ("conv2b", 2), ("conv2c", 3), ("conv2d", 4))
EPS = 1e-5


def _np(t) -> np.ndarray:
    if hasattr(t, "detach"):
        t = t.detach().cpu().numpy()
    return np.asarray(t, dtype=np.float64)


def load_state_dict(path) -> Dict[str, np.ndarray]:
    return _load_checkpoint(path)[0]


def _load_checkpoint(path):
    """(state dict without `module.` prefixes, the top-level `model_name` a reference training checkpoint records or
    None)."""
    import torch

    ckpt = torch.load(str(path), map_location="cpu", weights_only=False)
    sd = ckpt["state_dict"] if isinstance(ckpt, dict) and "state_dict" in ckpt else ckpt
    name = ckpt.get("model_name") if isinstance(ckpt, dict) else None
    sd = {(k[7:] if k.startswith("module.") else k): v for k, v in sd.items()}
    return sd, (name if isinstance(name, str) and name else None)


def _bn_fold(sd, name) -> Tuple[np.ndarray, np.ndarray]:
    scale = _np(sd[name + ".weight"]) / np.sqrt(_np(sd[name + ".running_var"]) + EPS)
    shift = _np(sd[name + ".bias"]) - _np(sd[name + ".running_mean"]) * scale
    return scale, shift


def _pw(sd, name, bn=None):
    """1x1 conv weight [co][ci][1][1] -> K-major [ci][co] with an optional BN folded in; returns (W, b)."""
    w = _np(sd[name + ".weight"])[:, :, 0, 0]
    co = w.shape[0]
    b = np.zeros(co)
    if (name + ".bias") in sd:
        b = _np(sd[name + ".bias"])
    if bn is not None:
        scale, shift = _bn_fold(sd, bn)
        w = w * scale[:, None]
        b = b * scale + shift
    return w.T.copy(), b


def _fold_osblock(sd, name, cin, cout) -> List[np.ndarray]:
    mid = cout // 4
    assert sd[name + ".conv1.conv.weight"].shape[:2] == (mid, cin)
    out = list(_pw(sd, name + ".conv1.conv", name + ".conv1.bn"))
    for br, depth in BRANCHES:
        for k in range(depth):
            lname = f"{name}.{br}" if br == "conv2a" else f"{name}.{br}.{k}"
            wpw, _ = _pw(sd, lname + ".conv1")
            sc, sh = _bn_fold(sd, lname + ".bn")
            wdw = _np(sd[lname + ".conv2.weight"])[:, 0] * sc[:, None, None]  # [c][3][3]
            out += [wpw, wdw.reshape(mid, 9).T.copy(), sh]
    w1, b1 = _pw(sd, name + ".gate.fc1")
    w2, b2 = _pw(sd, name + ".gate.fc2")
    out += [w1, b1, w2, b2]
    w3, b3 = _pw(sd, name + ".conv3.conv", name + ".conv3.bn")
    if (name + ".downsample.conv.weight") in sd:
        wd, bd = _pw(sd, name + ".downsample.conv", name + ".downsample.bn")
        out += [np.concatenate([w3, wd], 0), b3 + bd]
    else:
        assert cin == cout
        out += [w3, b3]
    return out


def _fold_stem(sd, conv, bn) -> List[np.ndarray]:
    w = _np(sd[conv + ".weight"])  # [c0][3][7][7]
    scale, shift = _bn_fold(sd, bn)
    w = w * scale[:, None, None, None]
    return [w.transpose(2, 3, 1, 0).reshape(147, w.shape[0]), shift]


def fold_osnet(sd) -> Tuple[List[int], List[np.ndarray]]:
    c0 = sd["conv1.conv.weight"].shape[0]
    chans = [c0] + [sd[f"conv{s + 2}.1.conv3.conv.weight"].shape[0] for s in range(3)]
    feat = sd["fc.0.weight"].shape[0]
    out: List[np.ndarray] = _fold_stem(sd, "conv1.conv", "conv1.bn")
    for s in range(3):
        stage = f"conv{s + 2}"
        for j in range(2):
            out += _fold_osblock(sd, f"{stage}.{j}", chans[s] if j == 0 else chans[s + 1], chans[s + 1])
        if s < 2:
            out += list(_pw(sd, f"{stage}.2.0.conv", f"{stage}.2.0.bn"))
    out += list(_pw(sd, "conv5.conv", "conv5.bn"))
    wf = _np(sd["fc.0.weight"])  # [feat][c3]
    bf = _np(sd["fc.0.bias"])
    scale, shift = _bn_fold(sd, "fc.1")
    out += [(wf * scale[:, None]).T.copy(), bf * scale + shift]
    return chans + [feat], out


# LMBN_n (reid/backbones/lmbn/lmbn_n.py): the output row interleaves seven 512-d vectors, element c*7 + k being channel
# c of vector k.  LMBN_NECKS lists, per vector k < 5, the BNNeck3 that produces it (reduction_0 on the average-pooled
# bottleneck output, reduction_4 on its max pool, reduction_1 on the max-pooled partial branch, reduction_2 / _3 on
# the averages of its top / bottom halves); vectors 5 and 6 are the channel halves through `shared` + reduction_ch_*.
LMBN_NECKS = (0, 4, 1, 2, 3)
LMBN_INPUT_H = 384
LMBN_FEAT = 3584


def _lmbn_n_keys():
    from .synthetic import make_lmbn_n_state

    return {k for k in make_lmbn_n_state(0, num_classes=1) if not k.endswith("num_batches_tracked")}


def is_lmbn(sd) -> bool:
    return "backone.0.conv.weight" in sd


def fold_lmbn_n(sd) -> List[np.ndarray]:
    """LMBN_n state dict -> arrays of the arch-3 blob in the order csrc/reid_model.cu walks them:
        stem | trunk: backone.2.0, backone.2.1, transition backone.2.2.0, backone.3 (OSBlocks laid out as in OSNet)
        per branch (global, partial, channel): OSBlock .0.1, transition .0.2.0, OSBlocks .1.0 and .1.1, conv5 .2
        bottleneck OSBlock (batch_drop_block.drop_batch_bottleneck; BatchDropTop is the identity in eval)
        necks: for k in LMBN_NECKS: reduction_k 1x1 with its BatchNorm1d folded, W[512][512], b[512]
        shared: 1x1 256 -> 512 with shared.1 folded, W[256][512], b[512]
        reduction_ch_0, reduction_ch_1: BatchNorm1d as scale[512], shift[512] (it follows a ReLU: not foldable)
    Refuses (ValueError) any state dict whose key set is not exactly LMBN_n's, e.g. lmbn_ain_n's instance norms."""
    keys = {k for k in sd if not k.endswith("num_batches_tracked")}
    want = _lmbn_n_keys()
    if keys != want:
        extra, missing = sorted(keys - want)[:3], sorted(want - keys)[:3]
        raise ValueError(f"not an LMBN_n state dict (unexpected keys {extra}, missing keys {missing})")
    out: List[np.ndarray] = _fold_stem(sd, "backone.0.conv", "backone.0.bn")
    out += _fold_osblock(sd, "backone.2.0", 64, 256)
    out += _fold_osblock(sd, "backone.2.1", 256, 256)
    out += list(_pw(sd, "backone.2.2.0.conv", "backone.2.2.0.bn"))
    out += _fold_osblock(sd, "backone.3", 256, 384)
    from .synthetic import LMBN_BRANCHES

    for br in LMBN_BRANCHES:
        out += _fold_osblock(sd, f"{br}.0.1", 384, 384)
        out += list(_pw(sd, f"{br}.0.2.0.conv", f"{br}.0.2.0.bn"))
        out += _fold_osblock(sd, f"{br}.1.0", 384, 512)
        out += _fold_osblock(sd, f"{br}.1.1", 512, 512)
        out += list(_pw(sd, f"{br}.2.conv", f"{br}.2.bn"))
    out += _fold_osblock(sd, "batch_drop_block.drop_batch_bottleneck", 512, 512)
    for k in LMBN_NECKS:
        out += list(_pw(sd, f"reduction_{k}.reduction", f"reduction_{k}.bn"))
    out += list(_pw(sd, "shared.0", "shared.1"))
    for j in range(2):
        out += list(_bn_fold(sd, f"reduction_ch_{j}.bn"))
    return out


# OSNet with instance norms (arch 4): osnet_ain_x{1_0,0_75,0_5,0_25} (reid/backbones/osnet_ain.py) and osnet_ibn_x1_0
# (reid/backbones/osnet.py:548).  Per-block IN placement, recorded in header words 10-15:
IN_NONE, IN_BEFORE_RESIDUAL, IN_AFTER_RESIDUAL = 0, 1, 2


def _ignored(k: str) -> bool:
    return k.startswith("classifier.") or k.endswith("num_batches_tracked")


def _osnet_in_variant(sd):
    """("ain" | "ibn", width name) for a state dict shaped like one of the OSNet-with-IN networks, else None."""
    from .synthetic import OSNET_ARCHS

    if "conv1.conv.weight" not in sd:
        return None
    c0 = sd["conv1.conv.weight"].shape[0]
    width = next((name for name, ch in OSNET_ARCHS.items() if ch[0] == c0), None)
    if "pool2.0.conv.weight" in sd or any(".layers." in k for k in sd):
        return "ain", width
    if any(".IN." in k for k in sd) or ("conv1.bn.weight" in sd and "conv1.bn.running_var" not in sd):
        return "ibn", width
    return None


def _osnet_in_keys(variant, width):
    from .synthetic import make_osnet_ain_state, make_osnet_ibn_state

    if width is None or (variant == "ibn" and width != "osnet_x1_0"):
        return None
    sd = make_osnet_ain_state(width, 0, num_classes=1) if variant == "ain" else make_osnet_ibn_state(0, num_classes=1)
    return {k for k in sd if not _ignored(k)}


def _in_affine(sd, name):
    return [_np(sd[name + ".weight"]), _np(sd[name + ".bias"])]


def fold_osnet_in(sd):
    """OSNet-AIN / OSNet-IBN state dict -> (dims, IN modes [stem, block 0..5], arrays) of the arch-4 blob.  The arrays
    keep the arch-1 order; where an instance norm sits:
        stem      W[147][c0] (no bias, no fold), gamma[c0], beta[c0]           (IN then ReLU, before the max pool)
        IN_BEFORE_RESIDUAL block (OSBlockINin): ... gate, conv3 W[mid][cout], zero bias[cout],
                  then (downsample) W[cin][cout] with its BN folded, b[cout], then gamma[cout], beta[cout]
        IN_AFTER_RESIDUAL block (IBN conv2.0 / conv2.1): the arch-1 combine (conv3 rows, downsample rows, summed bias),
                  then gamma[cout], beta[cout]
    Refuses (ValueError, naming the keys) any state dict whose key set, apart from `classifier.*` and
    `num_batches_tracked`, is not exactly the one of the variant its structure suggests."""
    from .synthetic import OSNET_AIN_ININ, OSNET_ARCHS

    variant, width = _osnet_in_variant(sd) or (None, None)
    want = _osnet_in_keys(variant, width) if variant else None
    keys = {k for k in sd if not _ignored(k)}
    if want is None or keys != want:
        label = {"ain": "OSNet-AIN", "ibn": "OSNet-IBN x1_0"}.get(variant, "OSNet with instance norms")
        extra, missing = sorted(keys - (want or set()))[:4], sorted((want or set()) - keys)[:4]
        raise ValueError(f"not an {label} state dict of a known width (unexpected keys {extra}, missing keys "
                         f"{missing}); osnet_ain_x1_0 / _x0_75 / _x0_5 / _x0_25 and osnet_ibn_x1_0 are supported")
    chans = list(OSNET_ARCHS[width])
    feat = sd["fc.0.weight"].shape[0]
    w = _np(sd["conv1.conv.weight"])
    out: List[np.ndarray] = [w.transpose(2, 3, 1, 0).reshape(147, chans[0])] + _in_affine(sd, "conv1.bn")
    modes = [1]
    for s in range(3):
        for j in range(2):
            name, cin, cout = f"conv{s + 2}.{j}", chans[s] if j == 0 else chans[s + 1], chans[s + 1]
            if variant == "ain":
                inin = OSNET_AIN_ININ[s][j]
                out += _fold_ain_block(sd, name, cin, cout, inin)
                modes.append(IN_BEFORE_RESIDUAL if inin else IN_NONE)
            else:
                out += _fold_osblock(sd, name, cin, cout)
                if (name + ".IN.weight") in sd:
                    out += _in_affine(sd, name + ".IN")
                modes.append(IN_AFTER_RESIDUAL if (name + ".IN.weight") in sd else IN_NONE)
        if s < 2:
            t = f"pool{s + 2}.0" if variant == "ain" else f"conv{s + 2}.2.0"
            out += list(_pw(sd, t + ".conv", t + ".bn"))
    out += list(_pw(sd, "conv5.conv", "conv5.bn"))
    wf, bf = _np(sd["fc.0.weight"]), _np(sd["fc.0.bias"])
    scale, shift = _bn_fold(sd, "fc.1")
    out += [(wf * scale[:, None]).T.copy(), bf * scale + shift]
    return chans + [feat], modes, out


def _fold_ain_block(sd, name, cin, cout, inin) -> List[np.ndarray]:
    """osnet_ain.py OSBlock / OSBlockINin: the OSNet layout with the branches read from `conv2.{t}.layers.{i}`."""
    mid = cout // 4
    assert sd[name + ".conv1.conv.weight"].shape[:2] == (mid, cin)
    out = list(_pw(sd, name + ".conv1.conv", name + ".conv1.bn"))
    for t in range(4):
        for i in range(t + 1):
            lname = f"{name}.conv2.{t}.layers.{i}"
            wpw, _ = _pw(sd, lname + ".conv1")
            sc, sh = _bn_fold(sd, lname + ".bn")
            wdw = _np(sd[lname + ".conv2.weight"])[:, 0] * sc[:, None, None]
            out += [wpw, wdw.reshape(mid, 9).T.copy(), sh]
    w1, b1 = _pw(sd, name + ".gate.fc1")
    w2, b2 = _pw(sd, name + ".gate.fc2")
    out += [w1, b1, w2, b2]
    has_ds = (name + ".downsample.conv.weight") in sd
    if not inin:
        w3, b3 = _pw(sd, name + ".conv3.conv", name + ".conv3.bn")
        if has_ds:
            wd, bd = _pw(sd, name + ".downsample.conv", name + ".downsample.bn")
            return out + [np.concatenate([w3, wd], 0), b3 + bd]
        return out + [w3, b3]
    w3, _ = _pw(sd, name + ".conv3.conv")   # Conv1x1Linear(bn=False): the instance norm follows directly
    out += [w3, np.zeros(cout)]
    if has_ds:
        out += list(_pw(sd, name + ".downsample.conv", name + ".downsample.bn"))
    return out + _in_affine(sd, name + ".IN")


# Bottleneck ResNet (arch 5): resnet50 / resnet101 of reid/backbones/resnet.py.  Header words 3-6 hold the Bottleneck
# counts of layer1..4 and word 7 the 2048-d feature; the arrays are
#     stem      W[147][64] (k = (kh*7+kw)*3 + ci, bn1 folded), b[64]
#     per Bottleneck (cin, width, cout = 4 width):
#         conv1     W[cin][width], b[width]                      (bn1 folded)
#         conv2     W[9 width][width] (k = (kh*3+kw)*width + ci), b[width]   (bn2 folded)
#         conv3     W[width (+ cin, block 0)][cout], b[cout]     (bn3 folded; block 0 appends the downsample's rows and
#                                                                 adds its folded bias: one GEMM over [conv2 out | x])
def _resnet_ignored(k: str) -> bool:
    return k.startswith(("fc.", "classifier.")) or k.endswith("num_batches_tracked")


def is_resnet(sd) -> bool:
    return "conv1.weight" in sd and any(k.startswith("layer1.0.") for k in sd)


def fold_resnet(sd):
    """ResNet state dict -> (block counts, arrays) of the arch-5 blob.  Only the Bottleneck resnet50 / resnet101 are
    supported: anything else whose keys or shapes differ from those (resnet18/34's BasicBlocks, ResNeXt's grouped 3x3,
    a missing BatchNorm key), apart from `fc.*`, `classifier.*` and `num_batches_tracked`, raises a ValueError naming
    the keys."""
    from .synthetic import RESNET_BLOCKS, resnet_layout

    keys = {k for k in sd if not _resnet_ignored(k)}
    n3 = len({k.split(".")[1] for k in keys if k.startswith("layer3.")})
    depth = next((d for d, b in RESNET_BLOCKS.items() if b[2] == n3), None)
    want = {}
    for name, kind, shape in resnet_layout(depth) if depth else ():
        if kind == "conv":
            want[name + ".weight"] = shape
        else:
            for p in ("weight", "bias", "running_mean", "running_var"):
                want[f"{name}.{p}"] = shape
    bad_shape = sorted(k for k in keys & set(want) if tuple(sd[k].shape) != want[k])[:4]
    if not want or keys != set(want) or bad_shape:
        extra, missing = sorted(keys - set(want))[:4], sorted(set(want) - keys)[:4]
        raise ValueError(f"not a Bottleneck resnet50 / resnet101 state dict (unexpected keys {extra}, missing keys "
                         f"{missing}, unexpected shapes {bad_shape}); BasicBlock ResNets and ResNeXt are not supported")
    out: List[np.ndarray] = _fold_stem(sd, "conv1", "bn1")
    for li, n_blocks in enumerate(RESNET_BLOCKS[depth]):
        for j in range(n_blocks):
            name = f"layer{li + 1}.{j}"
            out += list(_pw(sd, name + ".conv1", name + ".bn1"))
            w2 = _np(sd[name + ".conv2.weight"])   # [co][ci][3][3]
            sc, sh = _bn_fold(sd, name + ".bn2")
            w2 = (w2 * sc[:, None, None, None]).transpose(2, 3, 1, 0).reshape(-1, w2.shape[0])
            out += [w2, sh]
            w3, b3 = _pw(sd, name + ".conv3", name + ".bn3")
            if j == 0:
                wd, bd = _pw(sd, name + ".downsample.0", name + ".downsample.1")
                w3, b3 = np.concatenate([w3, wd], 0), b3 + bd
            out += [w3, b3]
    return list(RESNET_BLOCKS[depth]), out


# CLIP-ReID ViT-B/16 (arch 6): build_transformer of reid/backbones/clip/make_model.py with cfg MODEL.NAME "ViT-B-16",
# NECK_FEAT "after", SIE off.  Every linear weight is stored K-major ([in][out]); the arrays are
#     patch     W[768][768] (k = (ky*16 + kx)*3 + ci), b[768] (zero: conv1 has no bias)
#     pos       [T][768]  positional_embedding, class_embedding added to row 0
#     ln_pre    gamma[768], beta[768]
#     per block ln_1 gamma, beta; in_proj W[768][2304] (q | k | v; the q third and its bias scaled by 1/8, exact),
#               b[2304]; out_proj W[768][768], b; ln_2 gamma, beta; c_fc W[768][3072], b; c_proj W[3072][768], b
#     head      g[768], b[768]: ln_post's affine folded into bottleneck;  W[768][512], b[512]: ln_post's affine, proj
#               and bottleneck_proj folded  (the head normalises token 0 without an affine, then applies both)
CLIP_WIDTH, CLIP_LAYERS, CLIP_HEADS, CLIP_PROJ = 768, 12, 12, 512
CLIP_FEAT = CLIP_WIDTH + CLIP_PROJ
CLIP_GRIDS = {129: (16, 8), 257: (16, 16)}   # positional rows -> patch grid (256x128 and 256x256 crops)


def _clip_ignored(k: str) -> bool:
    """Keys registry.load_pretrained_weights drops for a CLIP model: anything outside build_transformer's state."""
    return k.startswith(("classifier.", "classifier_proj.", "prompt_learner.", "text_encoder.")) or \
        k.endswith("num_batches_tracked")


def is_clip(sd) -> bool:
    return "image_encoder.conv1.weight" in sd and "image_encoder.proj" in sd


def clip_vehicle_name(name: str) -> bool:
    """The reference runs 256x256 crops when the weights file name contains `veri` or `vehicleid` (registry.py:231,
    base_backend.py:57)."""
    return "veri" in name or "vehicleid" in name


def clip_layout(tokens: int = 129):
    """{key: shape} of build_transformer's state dict (ViT-B/16), without the classifiers and num_batches_tracked."""
    d = CLIP_WIDTH
    e = "image_encoder."
    want = {e + "class_embedding": (d,), e + "positional_embedding": (tokens, d), e + "proj": (d, CLIP_PROJ),
            e + "conv1.weight": (d, 3, 16, 16)}
    for ln in ("ln_pre", "ln_post"):
        want[f"{e}{ln}.weight"] = want[f"{e}{ln}.bias"] = (d,)
    for i in range(CLIP_LAYERS):
        b = f"{e}transformer.resblocks.{i}."
        want.update({b + "attn.in_proj_weight": (3 * d, d), b + "attn.in_proj_bias": (3 * d,),
                     b + "attn.out_proj.weight": (d, d), b + "attn.out_proj.bias": (d,),
                     b + "ln_1.weight": (d,), b + "ln_1.bias": (d,), b + "ln_2.weight": (d,), b + "ln_2.bias": (d,),
                     b + "mlp.c_fc.weight": (4 * d, d), b + "mlp.c_fc.bias": (4 * d,),
                     b + "mlp.c_proj.weight": (d, 4 * d), b + "mlp.c_proj.bias": (d,)})
    for bn, n in (("bottleneck", d), ("bottleneck_proj", CLIP_PROJ)):
        for p in ("weight", "bias", "running_mean", "running_var"):
            want[f"{bn}.{p}"] = (n,)
    return want


def fold_clip(sd, name=None):
    """CLIP-ReID state dict -> (header dims, input hw, grid, arrays) of the arch-6 blob.  Only ViT-B/16 is supported:
    any key or shape that differs from build_transformer's (another width or depth, CLIP-RN50's attnpool, a missing
    key), apart from the keys the reference discards, raises a ValueError naming the keys.  `name` is the weights
    file name: a `veri` / `vehicleid` name needs the 257-row positional table of 256x256 crops and any other name the
    129-row one of 256x128, as the reference builds the model for that name."""
    keys = {k for k in sd if not _clip_ignored(k)}
    pos_key = "image_encoder.positional_embedding"
    tokens = tuple(sd[pos_key].shape)[0] if pos_key in sd else 129
    want = clip_layout(tokens if tokens in CLIP_GRIDS else 129)
    bad_shape = sorted(k for k in keys & set(want) if tuple(sd[k].shape) != want[k])[:4]
    if keys != set(want) or bad_shape:
        extra, missing = sorted(keys - set(want))[:4], sorted(set(want) - keys)[:4]
        raise ValueError(f"not a CLIP-ReID ViT-B/16 state dict (unexpected keys {extra}, missing keys {missing}, "
                         f"unexpected shapes {bad_shape}); CLIP-RN50 and other widths or depths are not supported")
    if name is not None and clip_vehicle_name(name) != (tokens == 257):
        raise ValueError(f"CLIP weights '{name}' have a {tokens}-row positional table, but the reference runs "
                         f"{'256x256' if clip_vehicle_name(name) else '256x128'} crops for that file name "
                         f"({257 if clip_vehicle_name(name) else 129} rows) and would discard the table")
    gh, gw = CLIP_GRIDS[tokens]
    e = "image_encoder."
    d = CLIP_WIDTH
    w = _np(sd[e + "conv1.weight"])   # [768][3][16][16]
    pos = _np(sd[e + "positional_embedding"]).copy()
    pos[0] += _np(sd[e + "class_embedding"])
    out: List[np.ndarray] = [w.transpose(2, 3, 1, 0).reshape(-1, d), np.zeros(d), pos,
                             _np(sd[e + "ln_pre.weight"]), _np(sd[e + "ln_pre.bias"])]
    qscale = np.ones(3 * d)
    qscale[:d] = 1.0 / 8.0   # head_dim ** -0.5
    for i in range(CLIP_LAYERS):
        b = f"{e}transformer.resblocks.{i}."
        out += [_np(sd[b + "ln_1.weight"]), _np(sd[b + "ln_1.bias"]),
                (_np(sd[b + "attn.in_proj_weight"]) * qscale[:, None]).T, _np(sd[b + "attn.in_proj_bias"]) * qscale,
                _np(sd[b + "attn.out_proj.weight"]).T, _np(sd[b + "attn.out_proj.bias"]),
                _np(sd[b + "ln_2.weight"]), _np(sd[b + "ln_2.bias"]),
                _np(sd[b + "mlp.c_fc.weight"]).T, _np(sd[b + "mlp.c_fc.bias"]),
                _np(sd[b + "mlp.c_proj.weight"]).T, _np(sd[b + "mlp.c_proj.bias"])]
    g, beta = _np(sd[e + "ln_post.weight"]), _np(sd[e + "ln_post.bias"])
    sc, sh = _bn_fold(sd, "bottleneck")
    scp, shp = _bn_fold(sd, "bottleneck_proj")
    proj = _np(sd[e + "proj"])   # [768][512]
    out += [sc * g, sc * beta + sh, (g[:, None] * proj) * scp[None, :], (beta @ proj) * scp + shp]
    dims = [d, CLIP_LAYERS, CLIP_HEADS, CLIP_PROJ, CLIP_FEAT]
    return dims, (16 * gh, 16 * gw), (gh, gw), out


# MLFN (arch 7): mlfn of reid/backbones/mlfn.py (groups 32, channels 64 / 256 / 512 / 1024 / 2048, embed_dim 1024).
# Header words 3-7 hold the stem width 64, the last block width 2048, the 32 groups, the 16 blocks and the 1024-d
# feature.  Every 1x1 weight is K-major ([cin][cout]) with its BatchNorm (and conv bias) folded; the arrays are
#     stem      W[147][64] (k = (kh*7+kw)*3 + ci), b[64]          (bn1 folded, conv1's bias included)
#     per MLFNBlock i (cin, cout, mid = cout / 2, group width gw = mid / 32, fsm widths f0, f1):
#         fsm       W[cin][f0], b[f0]; W[f0][f1], b[f1]; W[f1][32], b[32]   (fsm.1 / .4 / .7 with .2 / .5 / .8 folded)
#         fm_conv1  W[cin][mid], b[mid]
#         fm_conv2  W[9][gw][mid] (element (tap, i, c) weighs input channel (c / gw) gw + i), b[mid]
#         fm_conv3  W[mid][cout], b[cout]
#         downsample (first block of a stage) W[cin][cout], b[cout]
#     fc_x      W[2048][1024], b[1024];   fc_s  W[512][1024], b[1024]
def _mlfn_ignored(k: str) -> bool:
    return k.startswith("classifier.") or k.endswith("num_batches_tracked")


def is_mlfn(sd) -> bool:
    return "feature.0.fm_conv1.weight" in sd


def fold_mlfn(sd) -> List[np.ndarray]:
    """MLFN state dict -> arrays of the arch-7 blob.  Only the reference's `mlfn` with its default groups, channels and
    embed_dim is supported: any key or shape that differs from it, apart from `classifier.*` and
    `num_batches_tracked`, raises a ValueError naming the keys."""
    from .synthetic import MLFN_GROUPS, mlfn_blocks, mlfn_layout

    keys = {k for k in sd if not _mlfn_ignored(k)}
    want = {}
    for name, kind, shape in mlfn_layout():
        if kind == "bn":
            for p in ("weight", "bias", "running_mean", "running_var"):
                want[f"{name}.{p}"] = shape
        else:
            want[name + ".weight"] = shape
            if kind == "convb":
                want[name + ".bias"] = shape[:1]
    bad_shape = sorted(k for k in keys & set(want) if tuple(sd[k].shape) != want[k])[:4]
    if keys != set(want) or bad_shape:
        extra, missing = sorted(keys - set(want))[:4], sorted(set(want) - keys)[:4]
        raise ValueError(f"not an MLFN state dict (unexpected keys {extra}, missing keys {missing}, unexpected shapes "
                         f"{bad_shape}); only mlfn with groups 32, channels 64-2048 and embed_dim 1024 is supported")
    w = _np(sd["conv1.weight"])   # [64][3][7][7]
    scale, shift = _bn_fold(sd, "bn1")
    out: List[np.ndarray] = [(w * scale[:, None, None, None]).transpose(2, 3, 1, 0).reshape(147, 64),
                             _np(sd["conv1.bias"]) * scale + shift]
    for i, (cin, cout, _, _, ds) in enumerate(mlfn_blocks()):
        b, mid = f"feature.{i}", cout // 2
        gw = mid // MLFN_GROUPS
        for conv, bn in (("fsm.1", "fsm.2"), ("fsm.4", "fsm.5"), ("fsm.7", "fsm.8")):
            out += list(_pw(sd, f"{b}.{conv}", f"{b}.{bn}"))
        out += list(_pw(sd, b + ".fm_conv1", b + ".fm_bn1"))
        w2 = _np(sd[b + ".fm_conv2.weight"])   # [mid][gw][3][3]
        sc, sh = _bn_fold(sd, b + ".fm_bn2")
        out += [(w2 * sc[:, None, None, None]).transpose(2, 3, 1, 0).reshape(9 * gw, mid), sh]
        out += list(_pw(sd, b + ".fm_conv3", b + ".fm_bn3"))
        if ds:
            out += list(_pw(sd, b + ".downsample.0", b + ".downsample.1"))
    out += list(_pw(sd, "fc_x.0", "fc_x.1"))
    out += list(_pw(sd, "fc_s.0", "fc_s.1"))
    return out


# HACNN (arch 8): HACNN of reid/backbones/hacnn.py (nchannels 128 / 256 / 384, feat_dim 512, learn_region=True).
# Header words 3-7 hold 32, 128, 256, 384 and the 1024-d feature, words 9-10 the 160x64 input.  Every ConvBlock has its
# conv bias and BatchNorm folded; a k x k convolution is stored K-major W[k*k*cin][cout] with k index
# (kh*k + kw)*cin + ci, then b[cout].  In `hacnn_layout` order:
#     conv (stem)                          W[27][32], b[32]
#     per level i = 1..3 (C = 128, 256, 384):
#         inception{i}.0 (InceptionA)      stream1.0, stream1.1, stream2.0, stream2.1, stream3.0, stream3.1, stream4.1
#         inception{i}.1 (InceptionB)      stream1.0, stream1.1, stream2.0, stream2.1, stream2.2, stream3.1
#         ha{i} spatial                    [12]: conv1's 9 taps and bias, conv2's scale and shift (BN folded)
#         ha{i} channel_attn conv1 / conv2 W[C][C/16], b[C/16]; W[C/16][C], b[C]
#         ha{i} soft_attn.conv             W[C][C], b[C]
#         ha{i} hard_attn.fc               W[C][8], b[8]
#     local_conv1..3 (InceptionB)          as above
#     fc_global                            W[384][512], b[512]  (BatchNorm1d folded)
#     fc_local                             W[1536][512], b[512] (BatchNorm1d folded)
def _hacnn_ignored(k: str) -> bool:
    return k.startswith(("classifier_global.", "classifier_local.")) or k.endswith("num_batches_tracked")


def is_hacnn(sd) -> bool:
    return "ha1.hard_attn.fc.weight" in sd


def _conv_block(sd, name) -> List[np.ndarray]:
    w = _np(sd[name + ".conv.weight"])   # [co][ci][k][k]
    scale, shift = _bn_fold(sd, name + ".bn")
    co, ci, k, _ = w.shape
    return [(w * scale[:, None, None, None]).transpose(2, 3, 1, 0).reshape(k * k * ci, co),
            _np(sd[name + ".conv.bias"]) * scale + shift]


def fold_hacnn(sd) -> List[np.ndarray]:
    """HACNN state dict -> arrays of the arch-8 blob.  Only the reference's HACNN with its default nchannels, feat_dim
    and learn_region=True is supported: any key or shape that differs from it, apart from the classifiers and
    `num_batches_tracked`, raises a ValueError naming the keys."""
    from .synthetic import hacnn_layout

    keys = {k for k in sd if not _hacnn_ignored(k)}
    want = {}
    for name, kind, shape in hacnn_layout():
        if kind == "cb":
            want[name + ".conv.weight"], want[name + ".conv.bias"] = shape, shape[:1]
            for p in ("weight", "bias", "running_mean", "running_var"):
                want[f"{name}.bn.{p}"] = shape[:1]
        elif kind == "bn":
            for p in ("weight", "bias", "running_mean", "running_var"):
                want[f"{name}.{p}"] = shape
        else:
            want[name + ".weight"], want[name + ".bias"] = shape, shape[:1]
    bad_shape = sorted(k for k in keys & set(want) if tuple(sd[k].shape) != want[k])[:4]
    if keys != set(want) or bad_shape:
        extra, missing = sorted(keys - set(want))[:4], sorted(set(want) - keys)[:4]
        raise ValueError(f"not a HACNN state dict (unexpected keys {extra}, missing keys {missing}, unexpected shapes "
                         f"{bad_shape}); only HACNN with nchannels 128/256/384, feat_dim 512 and learn_region=True "
                         "is supported")
    out: List[np.ndarray] = []
    spatial = None
    for name, kind, shape in hacnn_layout():
        if name.endswith("spatial_attn.conv1"):
            spatial = _conv_block(sd, name)
        elif name.endswith("spatial_attn.conv2"):
            a, b = _conv_block(sd, name)
            out.append(np.concatenate([spatial[0].ravel(), spatial[1], a.ravel(), b]))
        elif kind == "cb":
            out += _conv_block(sd, name)
        elif kind == "lin":
            w, b = _np(sd[name + ".weight"]), _np(sd[name + ".bias"])
            if name.startswith("fc_"):
                scale, shift = _bn_fold(sd, name[:-1] + "1")
                w, b = w * scale[:, None], b * scale + shift
            out += [w.T.copy(), b]
    return out


# ViT-Nano / ViT-Tiny (arch 9): ViTNano of reid/backbones/vit_nano.py (vit_nano, vit_nano_ain, vit_nano_ain_os,
# vit_tiny) and ViTTinyParts of vit_tiny.py (vit_tiny_parts, vit_tiny_parts3), eval mode.  Every linear weight is stored
# K-major ([in][out]); the arrays are
#     patch     W[768][192] (k = (ky*16 + kx)*3 + ci), b[192]
#     pos       [T][192]  pos_embed, cls_token added to row 0
#     per block norm1: LayerNorm gamma, beta, or (AIN blocks) a = sigmoid(gate) in_norm.weight,
#                      b = (1 - sigmoid(gate)) ln.weight, s = sigmoid(gate) in_norm.bias + (1 - sigmoid(gate)) ln.bias
#               qkv W[192][576] (q | k | v; the q third and its bias scaled by 1/8, exact), b[576]
#               proj W[192][192], b; norm2 gamma, beta; fc1 W[192][768], b; fc2 W[768][192], b
#     norm      gamma[192], beta[192]
#     head      class token:               bottleneck as scale[192], shift[192]
#               class token + proj:        W[192][512] (proj with bottleneck's scale folded), b[512] (its shift)
#               omni-scale:                per scale i: scale_norms[i] gamma, beta; gate W1[192][12], b1[12],
#                                          W2[12][192], b2[192]; bottleneck scale[192], shift[192]
#               class token + P strips:    the class token's W[192][512], b[512], then part_projs[i] with part_bns[i]
#                                          folded, W[192][512], b[512], for each strip
# (depth, AIN blocks, omni-scale, parts, crop h, crop w, patch stride) of each reference model name
VIT_VARIANTS = {
    "vit_nano": (6, 0, False, 0, 256, 128, 16),
    "vit_nano_ain": (6, 3, False, 0, 256, 128, 16),
    "vit_nano_ain_os": (6, 3, True, 0, 256, 128, 16),
    "vit_tiny": (12, 0, False, 0, 384, 128, 12),
    "vit_tiny_parts": (12, 0, False, 2, 384, 128, 12),
    "vit_tiny_parts3": (12, 0, False, 3, 384, 128, 12),
}
VIT_WIDTH, VIT_HEADS, VIT_PROJ = 192, 3, 512
# the reference's ReID model names (core/config.py MODEL_TYPES): a file name resolves to the longest one it contains
REFERENCE_MODEL_TYPES = (
    "resnet50", "resnet101", "mlfn", "hacnn", "mobilenetv2_x1_0", "mobilenetv2_x1_4", "osnet_x1_0", "osnet_x0_75",
    "osnet_x0_5", "osnet_x0_25", "osnet_ibn_x1_0", "osnet_ain_x1_0", "lmbn_ain_n", "lmbn_n", "cspreid_n", "clip",
    *VIT_VARIANTS, "csl_tinyvit_7m", "csl_tinyvit_7m_lmbn", "csl_tinyvit_11m", "csl_tinyvit_11m_lmbn",
    "csl_tinyvit_23m", "csl_tinyvit_23m_lmbn", "csl_tinyvit_small", "csl_tinyvit_normal", "csl_tinyvit_large",
    "csl_tinyvit_lmbn")


def model_name_from_file(name: str):
    """The reference's model name for a weights file name (registry.get_model_name without a checkpoint name)."""
    low = name.lower()
    return next((t for t in sorted(REFERENCE_MODEL_TYPES, key=len, reverse=True) if t in low), None)


def vit_grid(variant):
    """(crop h, crop w, stride, grid h, grid w, tokens) of a variant: PatchEmbed's (size - 16) // stride + 1."""
    _, _, _, _, h, w, stride = VIT_VARIANTS[variant]
    gh, gw = (h - 16) // stride + 1, (w - 16) // stride + 1
    return h, w, stride, gh, gw, 1 + gh * gw


def vit_layout(variant, num_classes=None):
    """{key: shape} of the reference model's state dict for `variant`, without num_batches_tracked; with num_classes,
    the classifiers too (the keys the reference's loader finds but the embedding never reads)."""
    depth, ain, omni, parts, *_ = VIT_VARIANTS[variant]
    d, mlp = VIT_WIDTH, 4 * VIT_WIDTH
    tokens = vit_grid(variant)[5]
    feat = VIT_PROJ if variant.startswith("vit_tiny") else d
    want = {"cls_token": (1, 1, d), "pos_embed": (1, tokens, d), "patch_embed.proj.weight": (d, 3, 16, 16),
            "patch_embed.proj.bias": (d,), "norm.weight": (d,), "norm.bias": (d,)}
    for i in range(depth):
        b = f"blocks.{i}."
        if i < ain:
            want.update({b + "norm1.ln.weight": (d,), b + "norm1.ln.bias": (d,), b + "norm1.in_norm.weight": (d,),
                         b + "norm1.in_norm.bias": (d,), b + "norm1.gate": (d,)})
        else:
            want.update({b + "norm1.weight": (d,), b + "norm1.bias": (d,)})
        want.update({b + "attn.qkv.weight": (3 * d, d), b + "attn.qkv.bias": (3 * d,), b + "attn.proj.weight": (d, d),
                     b + "attn.proj.bias": (d,), b + "norm2.weight": (d,), b + "norm2.bias": (d,),
                     b + "mlp.fc1.weight": (mlp, d), b + "mlp.fc1.bias": (mlp,), b + "mlp.fc2.weight": (d, mlp),
                     b + "mlp.fc2.bias": (d,)})
    if omni:
        mid = d // 16
        want.update({"os_agg.gate.fc.0.weight": (mid, d), "os_agg.gate.fc.0.bias": (mid,),
                     "os_agg.gate.fc.2.weight": (d, mid), "os_agg.gate.fc.2.bias": (d,)})
        for i in range(4):
            want[f"os_agg.scale_norms.{i}.weight"] = want[f"os_agg.scale_norms.{i}.bias"] = (d,)
    if feat != d:
        want["proj.weight"] = (feat, d)
    bns = ["bottleneck"] + [f"part_bns.{i}" for i in range(parts)]
    for bn in bns:
        for p in ("weight", "bias", "running_mean", "running_var"):
            want[f"{bn}.{p}"] = (feat,)
    for i in range(parts):
        want[f"part_projs.{i}.weight"] = (feat, d)
    if num_classes is not None:
        want["classifier.weight"] = (num_classes, feat)
        for i in range(parts):
            want[f"part_classifiers.{i}.weight"] = (num_classes, feat)
    return want


def looks_like_vit(sd) -> bool:
    return "cls_token" in sd and "patch_embed.proj.weight" in sd


def vit_variant_from_keys(sd) -> str:
    """The variant an unnamed state dict's keys suggest (the reference always has a name: file or checkpoint)."""
    tiny = "proj.weight" in sd or "blocks.6.norm1.weight" in sd or "part_projs.0.weight" in sd
    if tiny:
        return "vit_tiny_parts3" if "part_projs.2.weight" in sd else (
            "vit_tiny_parts" if "part_projs.0.weight" in sd else "vit_tiny")
    if "os_agg.gate.fc.0.weight" in sd:
        return "vit_nano_ain_os"
    return "vit_nano_ain" if "blocks.0.norm1.gate" in sd else "vit_nano"


def fold_vit(sd, variant):
    """ViT-Nano / ViT-Tiny state dict -> (header dims, header words 9-15, arrays) of the arch-9 blob for the reference
    model `variant`.  Every tensor of that model (apart from its classifiers) must be present with its shape: a missing
    or mis-shaped key raises a ValueError naming the keys, where the reference would silently run that layer randomly
    initialised.  Keys the model lacks are ignored, as the reference's loader discards them."""
    if variant not in VIT_VARIANTS:
        raise ValueError(f"unknown ViT variant {variant!r}; {', '.join(VIT_VARIANTS)} are supported")
    want = vit_layout(variant)
    missing = sorted(k for k in want if k not in sd)
    bad_shape = sorted(k for k in want if k in sd and tuple(sd[k].shape) != want[k])
    if missing or bad_shape:
        raise ValueError(f"not a {variant} state dict (missing keys {missing[:4]}, unexpected shapes {bad_shape[:4]}); "
                         "the reference would run these layers randomly initialised")
    depth, ain, omni, parts, *_ = VIT_VARIANTS[variant]
    h, w, stride, gh, gw, tokens = vit_grid(variant)
    d = VIT_WIDTH
    tiny = variant.startswith("vit_tiny")
    proj = VIT_PROJ if tiny else 0
    pw = _np(sd["patch_embed.proj.weight"])   # [192][3][16][16]
    pos = _np(sd["pos_embed"])[0].copy()
    pos[0] += _np(sd["cls_token"])[0, 0]
    out: List[np.ndarray] = [pw.transpose(2, 3, 1, 0).reshape(-1, d), _np(sd["patch_embed.proj.bias"]), pos]
    qscale = np.ones(3 * d)
    qscale[:d] = 1.0 / 8.0   # head_dim ** -0.5
    for i in range(depth):
        b = f"blocks.{i}."
        if i < ain:
            g = 1.0 / (1.0 + np.exp(-_np(sd[b + "norm1.gate"])))
            inw, inb = _np(sd[b + "norm1.in_norm.weight"]), _np(sd[b + "norm1.in_norm.bias"])
            lnw, lnb = _np(sd[b + "norm1.ln.weight"]), _np(sd[b + "norm1.ln.bias"])
            out += [g * inw, (1.0 - g) * lnw, g * inb + (1.0 - g) * lnb]
        else:
            out += [_np(sd[b + "norm1.weight"]), _np(sd[b + "norm1.bias"])]
        out += [(_np(sd[b + "attn.qkv.weight"]) * qscale[:, None]).T, _np(sd[b + "attn.qkv.bias"]) * qscale,
                _np(sd[b + "attn.proj.weight"]).T, _np(sd[b + "attn.proj.bias"]),
                _np(sd[b + "norm2.weight"]), _np(sd[b + "norm2.bias"]),
                _np(sd[b + "mlp.fc1.weight"]).T, _np(sd[b + "mlp.fc1.bias"]),
                _np(sd[b + "mlp.fc2.weight"]).T, _np(sd[b + "mlp.fc2.bias"])]
    out += [_np(sd["norm.weight"]), _np(sd["norm.bias"])]
    sc, sh = _bn_fold(sd, "bottleneck")
    if omni:
        for i in range(4):
            out += [_np(sd[f"os_agg.scale_norms.{i}.weight"]), _np(sd[f"os_agg.scale_norms.{i}.bias"])]
        out += [_np(sd["os_agg.gate.fc.0.weight"]).T, _np(sd["os_agg.gate.fc.0.bias"]),
                _np(sd["os_agg.gate.fc.2.weight"]).T, _np(sd["os_agg.gate.fc.2.bias"]), sc, sh]
    elif not proj:
        out += [sc, sh]
    else:
        out += [(_np(sd["proj.weight"]) * sc[:, None]).T, sh]
        for i in range(parts):
            psc, psh = _bn_fold(sd, f"part_bns.{i}")
            out += [(_np(sd[f"part_projs.{i}.weight"]) * psc[:, None]).T, psh]
    pool = 1 if omni else parts
    feat = (1 + parts) * proj if proj else d
    dims = [d, depth, VIT_HEADS, ain, feat]
    return dims, [h, w, gh, gw, stride, pool, proj], out


def resolve_vit(sd, file_name=None, model_name=None):
    """The ViT variant the reference builds for these weights, or None when they are not a ViT-Nano / ViT-Tiny model.
    The name is the checkpoint's `model_name`, else the longest reference model name in the file name; an unnamed
    in-memory state dict falls back to its key set.  Raises ValueError for a `veri` / `vehicleid` file name (the
    reference builds 256x256 crops there, which its positional table does not fit) and for ViT weights under a name
    the reference builds another model for."""
    name = model_name or (model_name_from_file(file_name) if file_name else None)
    if name is None:
        return vit_variant_from_keys(sd) if looks_like_vit(sd) else None
    if name not in VIT_VARIANTS:
        if looks_like_vit(sd) and not name.startswith(("csl_tinyvit", "cspreid")):
            raise ValueError(f"ViT weights under the model name {name!r}: the reference would build {name} and run it "
                             "randomly initialised")
        return None
    if file_name and clip_vehicle_name(file_name):
        raise ValueError(f"ViT weights '{file_name}': the reference runs 256x256 crops for a veri / vehicleid file name, "
                         f"which {name}'s positional table does not fit")
    return name


# CSPReID-n (arch 10): CSPReID_n of reid/backbones/cspreid_n.py.  Header words 3-7 hold the stage widths 128, 256, 384,
# 512 and the 1536-d row, words 9-10 the crop (256x128, or 256x256 for a `veri` / `vehicleid` file name).  Every
# ConvBNSiLU has its BatchNorm folded; a k x k convolution is stored K-major W[k*k*cin][cout] with k index
# (kh*k + kw)*cin + ci, then b[cout].  In `cspreid_layout` order:
#     stem.0, stem.1                       W[27][32], b[32]; W[288][64], b[64]
#     stage{s}.0 (C3k2, mid = out / 2)     cv1 W[in][2 mid], b; per bottleneck: cv1 W[mid][mid/2], b; cv2 W[9 mid/2][mid],
#                                          b; then cv2 W[(2 + n) mid][out], b
#     stage{s}.1 (s = 1..3)                W[9 out][out], b (3x3 stride 2)
#     stage4.1 (SPPF)                      cv1 W[512][256], b; cv2 W[1024][512], b
#     stage4.2 (LightSelfAttention)        fc.0 W[512][64]; fc.2 W[64][512]; spatial depthwise W[9][512] (BN folded),
#                                          b[512]; spatial.3 w[512]
#     head.bn_global / bn_part0 / bn_part1 W[512][512] (BatchNorm1d folded), b[512]
CSPREID_STAGES = ((64, 128, 1), (128, 256, 1), (256, 384, 2), (384, 512, 1))   # C3k2 (in, out, bottlenecks)
CSPREID_FEAT = 1536
CSPREID_HEADS = ("bn_global", "bn_part0", "bn_part1")


def cspreid_layout():
    """[(name, kind, shape)] of CSPReID_n in blob order: kind "cbs" (ConvBNSiLU: `name.conv.weight` of `shape` =
    (cout, cin, k, k) and `name.bn.*`), "lsa" (LightSelfAttention at `name`, shape = (C, hidden)) or "neck" (a BNNeck3
    at `name`, shape = (feat, C))."""
    out = [("stem.0", "cbs", (32, 3, 3, 3)), ("stem.1", "cbs", (64, 32, 3, 3))]
    for s, (cin, cout, n) in enumerate(CSPREID_STAGES, 1):
        mid = cout // 2
        p = f"stage{s}.0"
        out.append((p + ".cv1", "cbs", (2 * mid, cin, 1, 1)))
        for i in range(n):
            out += [(f"{p}.bottlenecks.{i}.cv1", "cbs", (mid // 2, mid, 1, 1)),
                    (f"{p}.bottlenecks.{i}.cv2", "cbs", (mid, mid // 2, 3, 3))]
        out.append((p + ".cv2", "cbs", (cout, (2 + n) * mid, 1, 1)))
        if s < 4:
            out.append((f"stage{s}.1", "cbs", (cout, cout, 3, 3)))
    out += [("stage4.1.cv1", "cbs", (256, 512, 1, 1)), ("stage4.1.cv2", "cbs", (512, 1024, 1, 1)),
            ("stage4.2", "lsa", (512, 64))]
    out += [(f"head.{h}", "neck", (512, 512)) for h in CSPREID_HEADS]
    return out


def cspreid_keys():
    """{key: shape} of CSPReID_n's state dict without num_batches_tracked and the classifiers (the keys the embedding
    reads)."""
    want = {}

    def bn(name, c):
        for p in ("weight", "bias", "running_mean", "running_var"):
            want[f"{name}.{p}"] = (c,)

    for name, kind, shape in cspreid_layout():
        if kind == "cbs":
            want[name + ".conv.weight"] = shape
            bn(name + ".bn", shape[0])
        elif kind == "lsa":
            c, hid = shape
            want.update({name + ".fc.0.weight": (hid, c, 1, 1), name + ".fc.2.weight": (c, hid, 1, 1),
                         name + ".spatial.0.weight": (c, 1, 3, 3), name + ".spatial.3.weight": (1, c, 1, 1)})
            bn(name + ".spatial.1", c)
        else:
            want[name + ".reduction.weight"] = (shape[0], shape[1], 1, 1)
            bn(name + ".bn", shape[0])
    return want


def is_cspreid(sd) -> bool:
    return "stage4.2.spatial.0.weight" in sd or "head.bn_part1.reduction.weight" in sd


def cspreid_input_hw(file_name=None):
    """The reference's crop for cspreid_n weights: 256x256 for a `veri` / `vehicleid` file name, else 256x128
    (base_backend.py:57-64)."""
    return (256, 256) if file_name and clip_vehicle_name(file_name) else (256, 128)


def fold_cspreid(sd) -> List[np.ndarray]:
    """CSPReID_n state dict -> arrays of the arch-10 blob.  Every tensor of the reference model (apart from the
    classifiers) must be present with its shape: a missing or mis-shaped key raises a ValueError naming the keys, where
    the reference's loader would silently run that layer randomly initialised.  Extra keys are ignored, as that loader
    discards them."""
    want = cspreid_keys()
    missing = sorted(k for k in want if k not in sd)
    bad_shape = sorted(k for k in want if k in sd and tuple(sd[k].shape) != want[k])
    if missing or bad_shape:
        raise ValueError(f"not a cspreid_n state dict (missing keys {missing[:4]}, unexpected shapes {bad_shape[:4]}); "
                         "the reference would run these layers randomly initialised")
    out: List[np.ndarray] = []
    for name, kind, shape in cspreid_layout():
        if kind == "cbs":
            w = _np(sd[name + ".conv.weight"])   # [co][ci][k][k]
            scale, shift = _bn_fold(sd, name + ".bn")
            co, ci, k, _ = w.shape
            out += [(w * scale[:, None, None, None]).transpose(2, 3, 1, 0).reshape(k * k * ci, co), shift]
        elif kind == "lsa":
            scale, shift = _bn_fold(sd, name + ".spatial.1")
            dw = _np(sd[name + ".spatial.0.weight"])[:, 0]   # [c][3][3]
            out += [_np(sd[name + ".fc.0.weight"])[:, :, 0, 0].T, _np(sd[name + ".fc.2.weight"])[:, :, 0, 0].T,
                    (dw * scale[:, None, None]).reshape(-1, 9).T, shift, _np(sd[name + ".spatial.3.weight"]).ravel()]
        else:
            scale, shift = _bn_fold(sd, name + ".bn")
            out += [(_np(sd[name + ".reduction.weight"])[:, :, 0, 0] * scale[:, None]).T, shift]
    return out


def _pad4(n: int) -> int:
    return (n + 3) // 4 * 4


def _pad_mat(w: np.ndarray, rows: int, cols: int) -> np.ndarray:
    out = np.zeros((rows, cols))
    out[: w.shape[0], : w.shape[1]] = w
    return out


def _pad_vec(b: np.ndarray, n: int) -> np.ndarray:
    out = np.zeros(n)
    out[: b.shape[0]] = b
    return out


def fold_mobilenetv2(sd):
    """MobileNetV2 (reid/backbones/mobilenetv2.py) -> (stem_c, feat, block table, arrays).  Channel counts such as
    22, 33, 89, 134 are zero-padded to multiples of 4 (padded lanes stay exactly 0 through ReLU6 and feed zero
    weight rows), so the float4 kernels apply unchanged.  Blob (arch 2): header, int32 table [n_blocks][4] =
    (cin, cout, t, stride), then  stem W[27][C0p], b | per block: expand W[cinp][midp], b; dw W[9][midp], b;
    project W[midp][coutp], b | conv9 W[clastp][featp], b."""
    from .synthetic import MOBILENETV2_LAYERS

    stem_c = sd["conv1.conv.weight"].shape[0]
    arrays, table = [], []
    w = _np(sd["conv1.conv.weight"])  # [c0][3][3][3]
    sc, sh = _bn_fold(sd, "conv1.bn")
    w = (w * sc[:, None, None, None]).transpose(2, 3, 1, 0).reshape(27, stem_c)
    arrays += [_pad_mat(w, 27, _pad4(stem_c)), _pad_vec(sh, _pad4(stem_c))]
    stage = 2
    while f"conv{stage}.0.conv1.conv.weight" in sd:
        i = 0
        while f"conv{stage}.{i}.conv1.conv.weight" in sd:
            name = f"conv{stage}.{i}"
            mid, cin = sd[name + ".conv1.conv.weight"].shape[:2]
            cout = sd[name + ".conv3.0.weight"].shape[0]
            stride = MOBILENETV2_LAYERS[stage - 2][3] if i == 0 else 1
            table.append((cin, cout, mid // cin, stride))
            we, be = _pw(sd, name + ".conv1.conv", name + ".conv1.bn")
            arrays += [_pad_mat(we, _pad4(cin), _pad4(mid)), _pad_vec(be, _pad4(mid))]
            sc, sh = _bn_fold(sd, name + ".dwconv2.bn")
            wd = (_np(sd[name + ".dwconv2.conv.weight"])[:, 0] * sc[:, None, None]).reshape(mid, 9).T
            arrays += [_pad_mat(wd, 9, _pad4(mid)), _pad_vec(sh, _pad4(mid))]
            # conv3 is nn.Sequential(Conv2d, BatchNorm2d): keys conv3.0 / conv3.1
            w3 = _np(sd[name + ".conv3.0.weight"])[:, :, 0, 0]
            sc, sh = _bn_fold(sd, name + ".conv3.1")
            arrays += [_pad_mat((w3 * sc[:, None]).T, _pad4(mid), _pad4(cout)), _pad_vec(sh, _pad4(cout))]
            i += 1
        stage += 1
    w9, b9 = _pw(sd, "conv9.conv", "conv9.bn")
    feat = w9.shape[1]
    arrays += [_pad_mat(w9, _pad4(w9.shape[0]), _pad4(feat)), _pad_vec(b9, _pad4(feat))]
    return stem_c, feat, table, arrays


def export_blob(weights, out_path=None) -> Path:
    """`weights`: path to a .pt checkpoint or an in-memory state dict.  Returns the blob path."""
    name = model_name = None
    if isinstance(weights, (str, Path)):
        src = Path(weights)
        if src.suffix == ".b200reid":
            return src
        sd, model_name = _load_checkpoint(src)
        name = src.name
        if out_path is None:
            out_path = src.with_suffix(".b200reid")
    else:
        sd = weights
        if out_path is None:
            raise ValueError("out_path is required when exporting an in-memory state dict")
    table, in_modes, extra = [], [], []
    vit = resolve_vit(sd, name, model_name)
    ref_name = model_name or (model_name_from_file(name) if name else None)
    if vit is not None:
        dims, extra, arrays = fold_vit(sd, vit)
        arch = ARCH_VIT
    elif ref_name == "cspreid_n" or (ref_name is None and is_cspreid(sd)):
        arrays = fold_cspreid(sd)
        arch, dims, extra = ARCH_CSPREID, [128, 256, 384, 512, CSPREID_FEAT], list(cspreid_input_hw(name))
    elif is_cspreid(sd):
        raise ValueError(f"cspreid_n weights under the model name {ref_name!r}: the reference would build {ref_name} "
                         "and run it randomly initialised")
    elif is_clip(sd):
        dims, input_hw, grid, arrays = fold_clip(sd, name)
        arch, extra = ARCH_CLIP, [*input_hw, *grid]
    elif "conv9.conv.weight" in sd:
        stem_c, feat, table, arrays = fold_mobilenetv2(sd)
        arch, dims = ARCH_MOBILENETV2, [stem_c, len(table), 0, 0, feat]
    elif _osnet_in_variant(sd) is not None:
        dims, in_modes, arrays = fold_osnet_in(sd)
        arch = ARCH_OSNET_IN
    elif "conv1.conv.weight" in sd and "conv5.conv.weight" in sd and "fc.0.weight" in sd:
        dims, arrays = fold_osnet(sd)
        arch = ARCH_OSNET
    elif is_lmbn(sd):
        arrays = fold_lmbn_n(sd)
        arch, dims = ARCH_LMBN_N, [64, 256, 384, 512, LMBN_FEAT]
    elif is_resnet(sd):
        blocks, arrays = fold_resnet(sd)
        arch, dims = ARCH_RESNET, blocks + [RESNET_FEAT]
    elif is_mlfn(sd):
        arrays = fold_mlfn(sd)
        arch, dims = ARCH_MLFN, [64, 2048, 32, 16, MLFN_FEAT]
    elif is_hacnn(sd):
        arrays = fold_hacnn(sd)
        arch, dims = ARCH_HACNN, [32, 128, 256, 384, HACNN_FEAT]
    else:
        raise ValueError("only OSNet, OSNet-AIN, OSNet-IBN, MobileNetV2, LMBN_n, ResNet50 / ResNet101, CLIP-ReID "
                         "ViT-B/16, MLFN, HACNN, ViT-Nano / ViT-Tiny and CSPReID-n state dicts are implemented on the "
                         "B200 ReID path")
    # every tensor starts on a 16-byte boundary (the kernels read weights as float4)
    padded = []
    for a in arrays:
        flat = np.asarray(a, dtype=np.float32).ravel()
        padded.append(np.pad(flat, (0, (-flat.size) % 4)))
    payload = np.concatenate(padded)
    header = [MAGIC, VERSION, arch, *dims, int(payload.size)] + [0] * (16 - 9)
    if arch == ARCH_LMBN_N:
        header[9] = LMBN_INPUT_H
    if arch == ARCH_OSNET_IN:
        header[9:16] = in_modes
    if arch == ARCH_CLIP:
        header[9:13] = extra
    if arch == ARCH_HACNN:
        header[9:11] = [160, 64]
    if arch == ARCH_VIT:
        header[9:16] = extra
    if arch == ARCH_CSPREID:
        header[9:11] = extra
    out_path = Path(out_path)
    tmp = out_path.with_suffix(out_path.suffix + ".tmp")
    with open(tmp, "wb") as f:
        f.write(struct.pack("<16i", *header))
        for row in table:
            f.write(struct.pack("<4i", *row))
        f.write(payload.tobytes())
    tmp.replace(out_path)
    return out_path


def read_blob(path):
    raw = Path(path).read_bytes()
    header = struct.unpack("<16i", raw[:64])
    if header[0] != MAGIC or header[1] != VERSION:
        raise ValueError("not a .b200reid blob")
    off = 64
    if header[2] == ARCH_MOBILENETV2:
        off += 16 * header[4]
    payload = np.frombuffer(raw[off:], dtype=np.float32)
    assert payload.size == header[8]
    return header, payload


def read_block_table(path):
    raw = Path(path).read_bytes()
    header = struct.unpack("<16i", raw[:64])
    if header[2] != ARCH_MOBILENETV2:
        return []
    return [struct.unpack("<4i", raw[64 + 16 * i: 80 + 16 * i]) for i in range(header[4])]


def blob_digest(path) -> str:
    return hashlib.sha256(Path(path).read_bytes()).hexdigest()[:16]
