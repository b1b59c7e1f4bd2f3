"""Seeded synthetic inputs for benchmarks and tests: the reference's own throughput-sweep detection
generator and random-init OSNet weights.  Data generators only -- no arithmetic of the tracked path.

`bench_stream` restates /root/reference/tests/performance/benchmark_fps.py:60-94 (`_make_random_dets` +
`_jitter_dets`, seed 42 + n_dets (+ 1000 * stream), fixed random uint8 frame) -- SURVEY.md section 8(d).
`make_osnet_state` builds a state dict with the reference's parameter names (reid/backbones/osnet.py) because the
container has no pretrained checkpoints (SURVEY.md section 8c); BatchNorm statistics are randomised so folding is
exercised, and gains are chosen so activations stay O(1-10) through the network.
"""
from __future__ import annotations

import numpy as np

OSNET_ARCHS = {
    "osnet_x0_25": (16, 64, 96, 128),
    "osnet_x0_5": (32, 128, 192, 256),
    "osnet_x0_75": (48, 192, 288, 384),
    "osnet_x1_0": (64, 256, 384, 512),
}
BRANCH_DEPTHS = (("conv2a", 1), ("conv2b", 2), ("conv2c", 3), ("conv2d", 4))


def bench_image(hw=(720, 1280), seed=0):
    rng = np.random.default_rng(seed)
    return rng.integers(0, 255, size=(hw[0], hw[1], 3), dtype=np.uint8)


def bench_stream(n_dets: int, n_frames: int, hw=(720, 1280), stream: int = 0):
    """Returns (image, [dets_f32 (n,6)] * n_frames) exactly as the reference benchmark would feed them."""
    h, w = hw
    rng = np.random.default_rng(42 + n_dets + 1000 * stream)
    img = rng.integers(0, 255, size=(h, w, 3), dtype=np.uint8)
    cx = rng.uniform(80, w - 80, size=n_dets)
    cy = rng.uniform(80, h - 80, size=n_dets)
    bw = rng.uniform(40, 100, size=n_dets)
    bh = rng.uniform(80, 200, size=n_dets)
    x1 = np.clip(cx - bw / 2, 0, w - 1)
    y1 = np.clip(cy - bh / 2, 0, h - 1)
    x2 = np.clip(cx + bw / 2, 1, w)
    y2 = np.clip(cy + bh / 2, 1, h)
    conf = rng.uniform(0.55, 0.95, size=n_dets)
    cls = np.zeros(n_dets, dtype=np.float32)
    base = np.stack([x1, y1, x2, y2, conf, cls], axis=1).astype(np.float32)
    frames = []
    for _ in range(n_frames):
        out = base.copy()
        dx = rng.normal(0.0, 4.0, size=n_dets).astype(np.float32)
        dy = rng.normal(0.0, 4.0, size=n_dets).astype(np.float32)
        out[:, 0] = np.clip(out[:, 0] + dx, 0, w - 1)
        out[:, 2] = np.clip(out[:, 2] + dx, 1, w)
        out[:, 1] = np.clip(out[:, 1] + dy, 0, h - 1)
        out[:, 3] = np.clip(out[:, 3] + dy, 1, h)
        frames.append(out)
    return img, frames



def _osnet_makers(g, sd):
    """conv / bn / osblock generators writing seeded tensors with the reference's parameter names into `sd`."""
    import torch

    def conv(name, co, ci, k, groups=1, gain=1.0):
        fan_in = (ci // groups) * k * k
        sd[name + ".weight"] = torch.randn(co, ci // groups, k, k, generator=g) * (gain / fan_in) ** 0.5

    def bn(name, c):
        sd[name + ".weight"] = 0.5 + torch.rand(c, generator=g)
        sd[name + ".bias"] = 0.2 * torch.randn(c, generator=g)
        sd[name + ".running_mean"] = 0.2 * torch.randn(c, generator=g)
        sd[name + ".running_var"] = 0.5 + torch.rand(c, generator=g)
        sd[name + ".num_batches_tracked"] = torch.tensor(0)

    def light(name, c):
        conv(name + ".conv1", c, c, 1)
        conv(name + ".conv2", c, c, 3, groups=c)
        bn(name + ".bn", c)

    def osblock(name, cin, cout):
        mid = cout // 4
        conv(name + ".conv1.conv", mid, cin, 1)
        bn(name + ".conv1.bn", mid)
        light(name + ".conv2a", mid)
        for br, depth in BRANCH_DEPTHS[1:]:
            for k in range(depth):
                light(f"{name}.{br}.{k}", mid)
        hid = mid // 16
        conv(name + ".gate.fc1", hid, mid, 1)
        sd[name + ".gate.fc1.bias"] = 0.1 * torch.randn(hid, generator=g)
        conv(name + ".gate.fc2", mid, hid, 1)
        sd[name + ".gate.fc2.bias"] = 0.1 * torch.randn(mid, generator=g)
        conv(name + ".conv3.conv", cout, mid, 1, gain=0.1)
        bn(name + ".conv3.bn", cout)
        if cin != cout:
            conv(name + ".downsample.conv", cout, cin, 1)
            bn(name + ".downsample.bn", cout)

    return conv, bn, osblock


def make_osnet_state(arch: str = "osnet_x0_25", seed: int = 0, feature_dim: int = 512, num_classes: int = 1041):
    import torch

    ch = OSNET_ARCHS[arch]
    g = torch.Generator().manual_seed(seed)
    sd = {}
    conv, bn, osblock = _osnet_makers(g, sd)
    conv("conv1.conv", ch[0], 3, 7)
    bn("conv1.bn", ch[0])
    for s, (cin, cout) in enumerate(((ch[0], ch[1]), (ch[1], ch[2]), (ch[2], ch[3]))):
        stage = f"conv{s + 2}"
        osblock(f"{stage}.0", cin, cout)
        osblock(f"{stage}.1", cout, cout)
        if s < 2:
            conv(f"{stage}.2.0.conv", cout, cout, 1)
            bn(f"{stage}.2.0.bn", cout)
    conv("conv5.conv", ch[3], ch[3], 1)
    bn("conv5.bn", ch[3])
    sd["fc.0.weight"] = 0.05 * torch.randn(feature_dim, ch[3], generator=g)
    sd["fc.0.bias"] = 0.05 * torch.randn(feature_dim, generator=g)
    bn("fc.1", feature_dim)
    sd["classifier.weight"] = 0.01 * torch.randn(num_classes, feature_dim, generator=g)
    sd["classifier.bias"] = torch.zeros(num_classes)
    return sd


def _in_affine(g, sd, name, c):
    """InstanceNorm2d(affine=True) parameters: randomised gamma / beta (some gammas negative) so the affine path and
    the sign handling of the fused ReLU + max pool are exercised."""
    import torch

    sd[name + ".weight"] = (0.5 + torch.rand(c, generator=g)) * torch.where(torch.rand(c, generator=g) < 0.15, -1.0, 1.0)
    sd[name + ".bias"] = 0.2 * torch.randn(c, generator=g)


# reid/backbones/osnet_ain.py: which blocks of conv2 / conv3 / conv4 are OSBlockINin (IN before the residual add)
OSNET_AIN_ININ = ((True, True), (False, True), (True, False))


def _osnet_arch(width: str) -> str:
    """Width name: x0_75, osnet_x0_75 or osnet_ain_x0_75 -> osnet_x0_75."""
    return "osnet_" + width[width.index("x"):]


def make_osnet_ain_state(width: str = "x1_0", seed: int = 0, feature_dim: int = 512, num_classes: int = 4101):
    """Seeded state dict with the parameter names of the reference's osnet_ain_x{1_0,0_75,0_5,0_25}
    (reid/backbones/osnet_ain.py): stem conv + InstanceNorm, blocks `[[INin, INin], [OSBlock, INin], [INin, OSBlock]]`
    whose branches are `conv2.{t}.layers.{i}`, transitions `pool2.0` / `pool3.0`.  `width` is e.g. "x0_75" or
    "osnet_ain_x0_75"."""
    import torch

    ch = OSNET_ARCHS[_osnet_arch(width)]
    g = torch.Generator().manual_seed(seed)
    sd = {}
    conv, bn, _ = _osnet_makers(g, sd)

    def block(name, cin, cout, inin):
        mid = cout // 4
        conv(name + ".conv1.conv", mid, cin, 1)
        bn(name + ".conv1.bn", mid)
        for t in range(4):
            for i in range(t + 1):
                lname = f"{name}.conv2.{t}.layers.{i}"
                conv(lname + ".conv1", mid, mid, 1)
                conv(lname + ".conv2", mid, mid, 3, groups=mid)
                bn(lname + ".bn", mid)
        hid = mid // 16
        conv(name + ".gate.fc1", hid, mid, 1)
        sd[name + ".gate.fc1.bias"] = 0.1 * torch.randn(hid, generator=g)
        conv(name + ".gate.fc2", mid, hid, 1)
        sd[name + ".gate.fc2.bias"] = 0.1 * torch.randn(mid, generator=g)
        conv(name + ".conv3.conv", cout, mid, 1, gain=0.1 if not inin else 1.0)
        if not inin:
            bn(name + ".conv3.bn", cout)
        if cin != cout:
            conv(name + ".downsample.conv", cout, cin, 1)
            bn(name + ".downsample.bn", cout)
        if inin:
            _in_affine(g, sd, name + ".IN", cout)

    conv("conv1.conv", ch[0], 3, 7)
    _in_affine(g, sd, "conv1.bn", ch[0])
    for s, (cin, cout) in enumerate(((ch[0], ch[1]), (ch[1], ch[2]), (ch[2], ch[3]))):
        block(f"conv{s + 2}.0", cin, cout, OSNET_AIN_ININ[s][0])
        block(f"conv{s + 2}.1", cout, cout, OSNET_AIN_ININ[s][1])
        if s < 2:
            conv(f"pool{s + 2}.0.conv", cout, cout, 1)
            bn(f"pool{s + 2}.0.bn", cout)
    conv("conv5.conv", ch[3], ch[3], 1)
    bn("conv5.bn", ch[3])
    sd["fc.0.weight"] = 0.05 * torch.randn(feature_dim, ch[3], generator=g)
    sd["fc.0.bias"] = 0.05 * torch.randn(feature_dim, generator=g)
    bn("fc.1", feature_dim)
    sd["classifier.weight"] = 0.01 * torch.randn(num_classes, feature_dim, generator=g)
    sd["classifier.bias"] = torch.zeros(num_classes)
    return sd


def make_osnet_ibn_state(seed: int = 0, feature_dim: int = 512, num_classes: int = 4101):
    """Seeded state dict with the parameter names of the reference's osnet_ibn_x1_0 (reid/backbones/osnet.py:548,
    `IN=True`): the osnet_x1_0 names, with the stem's `conv1.bn` an InstanceNorm (weight and bias only) and an
    InstanceNorm `IN` after the residual add of conv2.0 and conv2.1."""
    import torch

    sd = make_osnet_state("osnet_x1_0", seed=seed, feature_dim=feature_dim, num_classes=num_classes)
    g = torch.Generator().manual_seed(seed + 7919)
    for k in [k for k in sd if k.startswith("conv1.bn.")]:
        del sd[k]
    _in_affine(g, sd, "conv1.bn", 64)
    for j in range(2):
        _in_affine(g, sd, f"conv2.{j}.IN", 256)
    return sd


LMBN_BRANCHES = ("global_branch", "partial_branch", "channel_branch")


def make_lmbn_n_state(seed: int = 0, num_classes: int = 702):
    """Seeded state dict with the parameter names of the reference's LMBN_n (reid/backbones/lmbn/lmbn_n.py): the
    OSNet_x1_0 trunk up to conv3[0] (`backone`), three branches of conv3[1:] + conv4 + conv5 (nn.Sequential slicing
    keeps the indices: `*_branch.0.1`, `*_branch.0.2.0`), the BatchFeatureErase_Top bottleneck OSBlock, five BNNeck3
    necks, `shared` and two BNNeck.  Every BatchNorm has randomised running statistics so folding is exercised."""
    import torch

    g = torch.Generator().manual_seed(seed)
    sd = {}
    conv, bn, osblock = _osnet_makers(g, sd)
    conv("backone.0.conv", 64, 3, 7)
    bn("backone.0.bn", 64)
    osblock("backone.2.0", 64, 256)
    osblock("backone.2.1", 256, 256)
    conv("backone.2.2.0.conv", 256, 256, 1)
    bn("backone.2.2.0.bn", 256)
    osblock("backone.3", 256, 384)
    for br in LMBN_BRANCHES:
        osblock(f"{br}.0.1", 384, 384)
        conv(f"{br}.0.2.0.conv", 384, 384, 1)
        bn(f"{br}.0.2.0.bn", 384)
        osblock(f"{br}.1.0", 384, 512)
        osblock(f"{br}.1.1", 512, 512)
        conv(f"{br}.2.conv", 512, 512, 1)
        bn(f"{br}.2.bn", 512)
    for i in range(5):
        conv(f"reduction_{i}.reduction", 512, 512, 1)
        bn(f"reduction_{i}.bn", 512)
        sd[f"reduction_{i}.classifier.weight"] = 0.001 * torch.randn(num_classes, 512, generator=g)
    conv("shared.0", 512, 256, 1, gain=2.0)
    bn("shared.1", 512)
    for j in range(2):
        bn(f"reduction_ch_{j}.bn", 512)
        sd[f"reduction_ch_{j}.classifier.weight"] = 0.001 * torch.randn(num_classes, 512, generator=g)
    osblock("batch_drop_block.drop_batch_bottleneck", 512, 512)
    return sd


RESNET_BLOCKS = {50: (3, 4, 6, 3), 101: (3, 4, 23, 3)}   # Bottleneck counts of layer1..4 (resnet.py resnet50 / resnet101)
RESNET_FEAT = 2048


def resnet_layout(depth: int):
    """[(parameter prefix, kind, shape)] of the reference's Bottleneck ResNet (reid/backbones/resnet.py, torchvision
    v1.5: the stride sits on the 3x3), kind "conv" (weight [co][ci][k][k]) or "bn" (BatchNorm2d of `shape[0]` channels),
    in module order.  `classifier` and `fc` are not listed: the embedding is the pooled layer4 map."""
    out = [("conv1", "conv", (64, 3, 7, 7)), ("bn1", "bn", (64,))]
    cin = 64
    for li, n_blocks in enumerate(RESNET_BLOCKS[depth]):
        width = 64 << li
        for j in range(n_blocks):
            name = f"layer{li + 1}.{j}"
            out += [(name + ".conv1", "conv", (width, cin, 1, 1)), (name + ".bn1", "bn", (width,)),
                    (name + ".conv2", "conv", (width, width, 3, 3)), (name + ".bn2", "bn", (width,)),
                    (name + ".conv3", "conv", (4 * width, width, 1, 1)), (name + ".bn3", "bn", (4 * width,))]
            if j == 0:
                out += [(name + ".downsample.0", "conv", (4 * width, cin, 1, 1)), (name + ".downsample.1", "bn", (4 * width,))]
            cin = 4 * width
    return out


def make_resnet_state(depth: int = 50, seed: int = 0, with_fc512: bool = False, num_classes: int = 751):
    """Seeded state dict with the parameter names of the reference's `resnet50` / `resnet101` (loads with strict=True).
    with_fc512 adds the `fc.0` Linear(2048, 512) + `fc.1` BatchNorm1d head and a 512-wide classifier of a
    resnet50_fc512 checkpoint, which the reference drops when it builds plain resnet50 for such a file.  BatchNorm
    statistics are randomised so folding is exercised; conv3 starts small so activations stay O(1-10) through the
    residual stream of resnet101."""
    import torch

    g = torch.Generator().manual_seed(seed)
    sd = {}
    conv, bn, _ = _osnet_makers(g, sd)
    for name, kind, shape in resnet_layout(depth):
        if kind == "bn":
            bn(name, shape[0])
        else:
            conv(name, shape[0], shape[1], shape[2], gain=0.1 if name.endswith("conv3") else 1.0)
    feat = RESNET_FEAT
    if with_fc512:
        feat = 512
        sd["fc.0.weight"] = 0.05 * torch.randn(512, RESNET_FEAT, generator=g)
        sd["fc.0.bias"] = 0.05 * torch.randn(512, generator=g)
        bn("fc.1", 512)
    sd["classifier.weight"] = 0.01 * torch.randn(num_classes, feat, generator=g)
    sd["classifier.bias"] = torch.zeros(num_classes)
    return sd


# MLFN (reid/backbones/mlfn.py, groups 32, channels 64 / 256 / 512 / 1024 / 2048, embed_dim 1024): per stage the
# MLFNBlock count, the output width and the FSM widths; the stride-2 grouped 3x3 sits on the first block of stages 2-4
MLFN_STAGES = ((3, 256, (128, 64)), (4, 512, (256, 128)), (6, 1024, (512, 128)), (3, 2048, (512, 128)))
MLFN_GROUPS = 32
MLFN_FEAT = 1024


def mlfn_blocks():
    """[(cin, cout, stride, (fsm0, fsm1), has_downsample)] of the 16 MLFNBlocks in `feature` order."""
    out, cin = [], 64
    for s, (n, cout, fsm) in enumerate(MLFN_STAGES):
        for j in range(n):
            stride = 2 if (j == 0 and s > 0) else 1
            out.append((cin, cout, stride, fsm, cin != cout or stride > 1))
            cin = cout
    return out


def mlfn_layout():
    """[(parameter prefix, kind, shape)] of the reference's `mlfn` in module order, kind "conv" (weight only), "convb"
    (weight and bias) or "bn" (BatchNorm2d of `shape[0]` channels).  `classifier` is not listed."""
    g = MLFN_GROUPS
    out = [("conv1", "convb", (64, 3, 7, 7)), ("bn1", "bn", (64,))]
    for i, (cin, cout, _, (f0, f1), ds) in enumerate(mlfn_blocks()):
        b, mid = f"feature.{i}", cout // 2
        out += [(b + ".fm_conv1", "conv", (mid, cin, 1, 1)), (b + ".fm_bn1", "bn", (mid,)),
                (b + ".fm_conv2", "conv", (mid, mid // g, 3, 3)), (b + ".fm_bn2", "bn", (mid,)),
                (b + ".fm_conv3", "conv", (cout, mid, 1, 1)), (b + ".fm_bn3", "bn", (cout,)),
                (b + ".fsm.1", "convb", (f0, cin, 1, 1)), (b + ".fsm.2", "bn", (f0,)),
                (b + ".fsm.4", "convb", (f1, f0, 1, 1)), (b + ".fsm.5", "bn", (f1,)),
                (b + ".fsm.7", "convb", (g, f1, 1, 1)), (b + ".fsm.8", "bn", (g,))]
        if ds:
            out += [(b + ".downsample.0", "conv", (cout, cin, 1, 1)), (b + ".downsample.1", "bn", (cout,))]
    out += [("fc_x.0", "conv", (MLFN_FEAT, 2048, 1, 1)), ("fc_x.1", "bn", (MLFN_FEAT,)),
            ("fc_s.0", "conv", (MLFN_FEAT, 16 * g, 1, 1)), ("fc_s.1", "bn", (MLFN_FEAT,))]
    return out


def make_mlfn_state(seed: int = 0, num_classes: int = 751):
    """Seeded state dict with the parameter names of the reference's `mlfn(num_classes)` (loads with strict=True).
    BatchNorm statistics are randomised so folding is exercised, the convolution biases of the stem and the FSM are
    non-zero, and fm_conv3 starts small so the residual stream stays O(1-10) through the 16 blocks."""
    import torch

    g = torch.Generator().manual_seed(seed)
    sd = {}
    conv, bn, _ = _osnet_makers(g, sd)
    for name, kind, shape in mlfn_layout():
        if kind == "bn":
            bn(name, shape[0])
            continue
        groups = MLFN_GROUPS if name.endswith("fm_conv2") else 1
        conv(name, shape[0], shape[1] * groups, shape[2], groups=groups, gain=0.1 if name.endswith("fm_conv3") else 1.0)
        if kind == "convb":
            sd[name + ".bias"] = 0.1 * torch.randn(shape[0], generator=g)
    sd["classifier.weight"] = 0.01 * torch.randn(num_classes, MLFN_FEAT, generator=g)
    sd["classifier.bias"] = torch.zeros(num_classes)
    return sd


# HACNN (reid/backbones/hacnn.py, nchannels 128 / 256 / 384, feat_dim 512, learn_region=True): 160x64 crops
HACNN_CH = (128, 256, 384)
HACNN_FEAT = 512
HACNN_INPUT_HW = (160, 64)
HACNN_HARD_BIAS = (0.0, -0.75, 0.0, -0.25, 0.0, 0.25, 0.0, 0.75)   # HardAttn.init_params


def _inception_a(p, cin, cout):
    mid = cout // 4
    return [(f"{p}.stream{s}.{j}", "cb", (mid, cin if j == 0 else mid, 1 if j == 0 else 3, 1 if j == 0 else 3))
            for s in (1, 2, 3) for j in (0, 1)] + [(f"{p}.stream4.1", "cb", (mid, cin, 1, 1))]


def _inception_b(p, cin, cout):
    mid = cout // 4
    return [(f"{p}.stream1.0", "cb", (mid, cin, 1, 1)), (f"{p}.stream1.1", "cb", (mid, mid, 3, 3)),
            (f"{p}.stream2.0", "cb", (mid, cin, 1, 1)), (f"{p}.stream2.1", "cb", (mid, mid, 3, 3)),
            (f"{p}.stream2.2", "cb", (mid, mid, 3, 3)), (f"{p}.stream3.1", "cb", (2 * mid, cin, 1, 1))]


def hacnn_layout():
    """[(parameter prefix, kind, shape)] of the reference's HACNN in blob order: kind "cb" is a ConvBlock (conv weight
    `shape` and bias, BatchNorm2d), "lin" an nn.Linear (weight `shape`, bias), "bn" a BatchNorm1d of shape[0].  The
    classifiers are not listed."""
    out = [("conv", "cb", (32, 3, 3, 3))]
    cin = 32
    for i, c in enumerate(HACNN_CH, 1):
        out += _inception_a(f"inception{i}.0", cin, c) + _inception_b(f"inception{i}.1", c, c)
        h = f"ha{i}"
        out += [(h + ".soft_attn.spatial_attn.conv1", "cb", (1, 1, 3, 3)),
                (h + ".soft_attn.spatial_attn.conv2", "cb", (1, 1, 1, 1)),
                (h + ".soft_attn.channel_attn.conv1", "cb", (c // 16, c, 1, 1)),
                (h + ".soft_attn.channel_attn.conv2", "cb", (c, c // 16, 1, 1)),
                (h + ".soft_attn.conv", "cb", (c, c, 1, 1)),
                (h + ".hard_attn.fc", "lin", (8, c))]
        cin = c
    cin = 32
    for i, c in enumerate(HACNN_CH, 1):
        out += _inception_b(f"local_conv{i}", cin, c)
        cin = c
    out += [("fc_global.0", "lin", (HACNN_FEAT, HACNN_CH[2])), ("fc_global.1", "bn", (HACNN_FEAT,)),
            ("fc_local.0", "lin", (HACNN_FEAT, 4 * HACNN_CH[2])), ("fc_local.1", "bn", (HACNN_FEAT,))]
    return out


def make_hacnn_state(seed: int = 0, num_classes: int = 751):
    """Seeded state dict with the parameter names of the reference's `HACNN(num_classes)` (loads with strict=True).
    BatchNorm statistics are randomised so folding is exercised, every ConvBlock conv has a non-zero bias, and
    `hard_attn.fc` has a non-zero weight, so the four regions move off centre and partly off the map."""
    import torch

    g = torch.Generator().manual_seed(seed)
    sd = {}
    conv, bn, _ = _osnet_makers(g, sd)
    for name, kind, shape in hacnn_layout():
        if kind == "cb":
            conv(name + ".conv", shape[0], shape[1], shape[2], gain=2.0)
            sd[name + ".conv.bias"] = 0.1 * torch.randn(shape[0], generator=g)
            bn(name + ".bn", shape[0])
        elif kind == "bn":
            bn(name, shape[0])
        elif name.endswith("hard_attn.fc"):
            sd[name + ".weight"] = 2.0 * torch.randn(*shape, generator=g) / shape[1] ** 0.5
            sd[name + ".bias"] = torch.tensor(HACNN_HARD_BIAS) + 0.2 * torch.randn(8, generator=g)
        else:
            sd[name + ".weight"] = torch.randn(*shape, generator=g) / shape[1] ** 0.5
            sd[name + ".bias"] = 0.1 * torch.randn(shape[0], generator=g)
    for name in ("classifier_global", "classifier_local"):
        sd[name + ".weight"] = 0.01 * torch.randn(num_classes, HACNN_FEAT, generator=g)
        sd[name + ".bias"] = torch.zeros(num_classes)
    return sd


def make_cspreid_state(seed: int = 0, num_classes: int = 751):
    """Seeded state dict with the parameter names of the reference's `CSPReID_n(num_classes)` (loads with strict=True).
    Every BatchNorm's gamma, beta and running statistics are randomised, so folding is exercised and no bottleneck's
    residual branch is the identity the reference's zero-gamma initialisation makes of it; the attention's gates are
    spread over (0, 1) rather than saturated."""
    import torch

    from .weights import CSPREID_HEADS, cspreid_layout

    g = torch.Generator().manual_seed(seed)
    sd = {}
    conv, bn, _ = _osnet_makers(g, sd)
    for name, kind, shape in cspreid_layout():
        if kind == "cbs":
            conv(name + ".conv", shape[0], shape[1], shape[2], gain=2.0)
            bn(name + ".bn", shape[0])
        elif kind == "lsa":
            c, hid = shape
            conv(name + ".fc.0", hid, c, 1, gain=0.5)
            conv(name + ".fc.2", c, hid, 1, gain=0.5)
            conv(name + ".spatial.0", c, c, 3, groups=c, gain=2.0)
            bn(name + ".spatial.1", c)
            conv(name + ".spatial.3", 1, c, 1, gain=0.5)
        else:
            conv(name + ".reduction", shape[0], shape[1], 1)
            bn(name + ".bn", shape[0])
    for h in CSPREID_HEADS:
        sd[f"head.{h}.classifier.weight"] = 0.001 * torch.randn(num_classes, 512, generator=g)
    return sd


def make_clip_state(seed: int = 0, vehicle: bool = False, num_classes: int = 751, extras: bool = True):
    """Seeded state dict with the key set of the reference's CLIP-ReID `build_transformer` (ViT-B/16: image_encoder.*,
    bottleneck.*, bottleneck_proj.*, classifier.*, classifier_proj.*); vehicle=True gives the 257-row positional table
    of 256x256 crops (clip_veri / clip_vehicleid), otherwise 129 rows (256x128).  extras adds a few keys of CLIP-ReID
    training checkpoints that the reference's loader discards (prompt_learner.*, text_encoder.*).
    Not trivial on purpose: BatchNorm statistics and LayerNorm gammas / betas are randomised, and in_proj is scaled so
    that q.k / 8 has a spread of a few units and attention rows are far from uniform; c_proj and out_proj start small
    so the residual stream stays O(1) through the 12 blocks."""
    import torch

    g = torch.Generator().manual_seed(seed)
    d, tokens = 768, (257 if vehicle else 129)
    e = "image_encoder."

    def randn(*shape, std=1.0):
        return torch.randn(*shape, generator=g) * std

    def ln(name):
        sd[name + ".weight"] = 0.5 + torch.rand(d, generator=g)
        sd[name + ".bias"] = randn(d, std=0.1)

    def bn(name, c):
        sd[name + ".weight"] = 0.5 + torch.rand(c, generator=g)
        sd[name + ".bias"] = randn(c, std=0.1)
        sd[name + ".running_mean"] = randn(c, std=0.1)
        sd[name + ".running_var"] = 0.5 + torch.rand(c, generator=g)
        sd[name + ".num_batches_tracked"] = torch.tensor(0)

    sd = {"classifier.weight": randn(num_classes, d, std=0.001)}
    sd["classifier_proj.weight"] = randn(num_classes, 512, std=0.001)
    sd[e + "class_embedding"] = randn(d, std=0.1)
    sd[e + "positional_embedding"] = randn(tokens, d, std=0.1)
    sd[e + "proj"] = randn(d, 512, std=d ** -0.5)
    sd[e + "conv1.weight"] = randn(d, 3, 16, 16, std=0.02)
    ln(e + "ln_pre")
    for i in range(12):
        b = f"{e}transformer.resblocks.{i}."
        sd[b + "attn.in_proj_weight"] = randn(3 * d, d, std=0.06)
        sd[b + "attn.in_proj_bias"] = randn(3 * d, std=0.05)
        sd[b + "attn.out_proj.weight"] = randn(d, d, std=0.02)
        sd[b + "attn.out_proj.bias"] = randn(d, std=0.02)
        ln(b + "ln_1")
        sd[b + "mlp.c_fc.weight"] = randn(4 * d, d, std=0.04)
        sd[b + "mlp.c_fc.bias"] = randn(4 * d, std=0.05)
        sd[b + "mlp.c_proj.weight"] = randn(d, 4 * d, std=0.01)
        sd[b + "mlp.c_proj.bias"] = randn(d, std=0.02)
        ln(b + "ln_2")
    ln(e + "ln_post")
    bn("bottleneck", d)
    bn("bottleneck_proj", 512)
    if extras:
        sd["prompt_learner.cls_ctx"] = randn(num_classes, 4, 512, std=0.02)
        sd["text_encoder.positional_embedding"] = randn(77, 512, std=0.01)
    return sd


def make_vit_state(variant: str = "vit_tiny", seed: int = 0, num_classes: int = 751):
    """Seeded state dict with the key set of the reference's ViT-Nano / ViT-Tiny model `variant` (vit_nano.py ViTNano,
    vit_tiny.py ViTTinyParts), classifiers and num_batches_tracked included.
    Not trivial on purpose: BatchNorm statistics, LayerNorm / InstanceNorm affines and the AIN gates (|gate| >= 1, far
    from sigmoid's midpoint) are randomised, qkv is scaled so that q.k / 8 has a spread of a few units and attention
    rows are far from uniform, and proj / fc2 start small so the residual stream stays O(1) through the blocks."""
    import torch

    from .weights import vit_layout

    g = torch.Generator().manual_seed(seed)

    def randn(*shape, std=1.0):
        return torch.randn(*shape, generator=g) * std

    sd = {}
    for k, shape in vit_layout(variant, num_classes=num_classes).items():
        name = k.rsplit(".", 1)[-1]
        if k.endswith("norm1.gate"):
            sd[k] = torch.sign(randn(*shape)) * (1.0 + 2.0 * torch.rand(*shape, generator=g))
        elif name == "running_var":
            sd[k] = 0.5 + torch.rand(*shape, generator=g)
        elif name == "running_mean":
            sd[k] = randn(*shape, std=0.1)
        elif name == "weight" and len(shape) == 1:   # LayerNorm / InstanceNorm / BatchNorm scale
            sd[k] = 0.5 + torch.rand(*shape, generator=g)
        elif name == "bias" and len(shape) == 1:
            sd[k] = randn(*shape, std=0.1 if "norm" in k or "bn" in k or "bottleneck" in k else 0.05)
        elif k in ("cls_token", "pos_embed"):
            sd[k] = randn(*shape, std=0.1)
        elif k == "patch_embed.proj.weight":
            sd[k] = randn(*shape, std=0.04)
        elif k.endswith("attn.qkv.weight"):
            sd[k] = randn(*shape, std=0.12)
        elif k.endswith(("attn.proj.weight", "mlp.fc2.weight")):
            sd[k] = randn(*shape, std=0.03)
        elif "classifier" in k:
            sd[k] = randn(*shape, std=0.001)
        else:   # mlp.fc1, proj, part_projs, the omni-scale gate
            sd[k] = randn(*shape, std=shape[-1] ** -0.5)
    for k in [k for k in sd if k.endswith("running_var")]:
        sd[k[: -len("running_var")] + "num_batches_tracked"] = torch.tensor(0)
    return sd


MOBILENETV2_LAYERS = ((1, 16, 1, 1), (6, 24, 2, 2), (6, 32, 3, 2), (6, 64, 4, 2), (6, 96, 3, 1), (6, 160, 3, 2),
                      (6, 320, 1, 1))  # (expansion t, base channels c, repeats n, first stride s), mobilenetv2.py:91-99


def mobilenetv2_blocks(width_mult: float = 1.4):
    """[(cin, cout, t, stride)] for every Bottleneck, plus stem channels and feature dim (mobilenetv2.py:86-102)."""
    cin = int(32 * width_mult)
    stem = cin
    blocks = []
    for t, c, n, s in MOBILENETV2_LAYERS:
        cout = int(c * width_mult)
        for i in range(n):
            blocks.append((cin, cout, t, s if i == 0 else 1))
            cin = cout
    feat = int(1280 * width_mult) if width_mult > 1 else 1280
    return stem, blocks, feat


def make_mobilenetv2_state(width_mult: float = 1.4, seed: int = 0, num_classes: int = 1041):
    """Seeded state dict with the reference's MobileNetV2 parameter names (reid/backbones/mobilenetv2.py)."""
    import torch

    g = torch.Generator().manual_seed(seed)
    sd = {}

    def conv(name, co, ci, k, groups=1, gain=1.0):
        fan_in = (ci // groups) * k * k
        sd[name + ".weight"] = torch.randn(co, ci // groups, k, k, generator=g) * (gain / fan_in) ** 0.5

    def bn(name, c):
        sd[name + ".weight"] = 0.5 + torch.rand(c, generator=g)
        sd[name + ".bias"] = 0.2 * torch.randn(c, generator=g)
        sd[name + ".running_mean"] = 0.2 * torch.randn(c, generator=g)
        sd[name + ".running_var"] = 0.5 + torch.rand(c, generator=g)
        sd[name + ".num_batches_tracked"] = torch.tensor(0)

    stem, blocks, feat = mobilenetv2_blocks(width_mult)
    conv("conv1.conv", stem, 3, 3, gain=2.0)
    bn("conv1.bn", stem)
    stage, idx, prev = 2, 0, None
    layer_of = []
    for t, c, n, s in MOBILENETV2_LAYERS:
        for i in range(n):
            layer_of.append((stage, i))
        stage += 1
    for (cin, cout, t, stride), (st, i) in zip(blocks, layer_of):
        name = f"conv{st}.{i}"
        mid = cin * t
        conv(name + ".conv1.conv", mid, cin, 1, gain=2.0)
        bn(name + ".conv1.bn", mid)
        conv(name + ".dwconv2.conv", mid, mid, 3, groups=mid, gain=2.0)
        bn(name + ".dwconv2.bn", mid)
        conv(name + ".conv3.0", cout, mid, 1, gain=0.5)
        bn(name + ".conv3.1", cout)
    conv("conv9.conv", feat, blocks[-1][1], 1, gain=2.0)
    bn("conv9.bn", feat)
    sd["classifier.weight"] = 0.01 * torch.randn(num_classes, feat, generator=g)
    sd["classifier.bias"] = torch.zeros(num_classes)
    return sd


def cohort_stream(n_objects=2048, cohorts=4, frames=10, hw=(1080, 1920), seed=3, dim=512, conf_lo=0.4):
    """BASELINE config 3 generator (SURVEY 8d): `n_objects` fixed objects in `cohorts` cohorts, cohort f mod cohorts is
    visible on frame f (every track is re-observed every `cohorts` frames < max_age) -> ~n_objects live tracks and
    n_objects / cohorts detections per frame.  Returns (dets per frame, unit appearance rows per frame)."""
    rng = np.random.default_rng(seed)
    h, w = hw
    cx, cy = rng.uniform(40, w - 40, n_objects), rng.uniform(60, h - 60, n_objects)
    bw, bh = rng.uniform(20, 50, n_objects), rng.uniform(40, 100, n_objects)
    conf = rng.uniform(conf_lo, 0.95, n_objects)   # conf_lo above the tracker's det_thresh: every object is tracked
    proto = np.abs(rng.normal(size=(n_objects, dim))).astype(np.float32)
    dets, embs = [], []
    for f in range(frames):
        idx = np.arange(f % cohorts, n_objects, cohorts)
        jx, jy = rng.normal(0, 2.0, idx.size), rng.normal(0, 2.0, idx.size)
        d = np.stack([cx[idx] + jx - bw[idx] / 2, cy[idx] + jy - bh[idx] / 2, cx[idx] + jx + bw[idx] / 2,
                      cy[idx] + jy + bh[idx] / 2, conf[idx], np.zeros(idx.size)], 1).astype(np.float32)
        e = np.maximum(proto[idx] + 0.3 * rng.normal(size=(idx.size, dim)).astype(np.float32), 0)
        dets.append(d)
        embs.append((e / np.linalg.norm(e, axis=1, keepdims=True)).astype(np.float32))
    return dets, embs


def camera_pan_sequence(n_frames: int = 16, hw=(360, 640), n_objects: int = 24, seed: int = 5, max_step: float = 4.0,
                        dim: int = 0):
    """Moving-camera test input (SURVEY 8f-3): a smooth textured canvas seen through a window that pans by a few whole
    pixels per frame (plus per-frame sensor noise), and detections of objects that stand still on the canvas -- so they
    move in the image by exactly the camera motion.  Pure numpy, seeded.  Returns (frames [H,W,3] uint8 BGR, dets (n,6)
    float32 per frame, window offsets (n_frames, 2) int, embeddings per frame or None)."""
    h, w = hw
    rng = np.random.default_rng(seed)
    margin = int(max_step * n_frames) + 8
    H, W = h + 2 * margin, w + 2 * margin
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    canvas = np.zeros((H, W, 3), np.float32)
    def smooth_field(cell):   # random grid of `cell`-pixel cells, bilinearly interpolated: smooth at the 0.15 scale
        gh, gw = H // cell + 3, W // cell + 3
        g = rng.random((gh, gw)).astype(np.float32)
        fy, fx = yy / cell, xx / cell
        y0, x0 = fy.astype(np.int64), fx.astype(np.int64)
        ay, ax = fy - y0, fx - x0
        return (g[y0, x0] * (1 - ay) * (1 - ax) + g[y0, x0 + 1] * (1 - ay) * ax
                + g[y0 + 1, x0] * ay * (1 - ax) + g[y0 + 1, x0 + 1] * ay * ax)

    for c in range(3):
        canvas[..., c] = smooth_field(56) + 0.5 * smooth_field(28) + 0.08 * rng.random((H, W)).astype(np.float32)
    canvas -= canvas.min()
    canvas = canvas / canvas.max() * 215.0 + 20.0
    ox, oy = float(margin), float(margin)
    offs, frames, dets, embs = [], [], [], []
    cx = rng.uniform(margin + 40, margin + w - 40, n_objects)
    cy = rng.uniform(margin + 40, margin + h - 40, n_objects)
    bw = rng.uniform(18, 46, n_objects)
    bh = rng.uniform(36, 90, n_objects)
    protos = np.abs(rng.normal(size=(n_objects, max(dim, 1)))).astype(np.float32)
    vx, vy = rng.uniform(-max_step, max_step, 2)
    for f in range(n_frames):
        if f % 5 == 0:
            vx, vy = rng.uniform(-max_step, max_step, 2)
        ox = float(np.clip(ox + vx, 2, 2 * margin - 2))
        oy = float(np.clip(oy + vy, 2, 2 * margin - 2))
        ix, iy = int(round(ox)), int(round(oy))
        offs.append((ix, iy))
        win = canvas[iy:iy + h, ix:ix + w] + rng.normal(0.0, 1.5, (h, w, 3)).astype(np.float32)
        frames.append(np.clip(np.rint(win), 0, 255).astype(np.uint8))
        keep = rng.random(n_objects) > 0.1
        x1 = cx - bw / 2 - ix + rng.normal(0, 0.4, n_objects)
        y1 = cy - bh / 2 - iy + rng.normal(0, 0.4, n_objects)
        d = np.stack([x1, y1, x1 + bw, y1 + bh, rng.uniform(0.55, 0.95, n_objects), np.zeros(n_objects)], 1)
        vis = keep & (d[:, 0] > 0) & (d[:, 1] > 0) & (d[:, 2] < w) & (d[:, 3] < h)
        dets.append(d[vis].astype(np.float32))
        if dim:
            e = np.maximum(protos[vis] + 0.3 * rng.normal(size=(int(vis.sum()), dim)).astype(np.float32), 0.0)
            embs.append((e / np.linalg.norm(e, axis=1, keepdims=True)).astype(np.float32))
    return frames, dets, np.asarray(offs), (embs if dim else None)


def camera_similarity_sequence(n_frames: int = 12, hw=(360, 640), n_objects: int = 24, seed: int = 5,
                               max_step: float = 4.0, max_rot_deg: float = 1.0, max_zoom: float = 0.01):
    """Moving-camera input for the partial-affine (similarity) estimators: a smooth textured canvas, like
    `camera_pan_sequence`'s, seen through a window that per frame pans by up to `max_step` pixels (sub-pixel), rotates by
    up to `max_rot_deg` degrees and zooms by up to `max_zoom`, sampled bilinearly, plus sensor noise.  Detections are
    the boxes of objects that stand still on the canvas, carried into the image by the window's similarity.  Pure numpy,
    seeded.  Returns (frames [H,W,3] uint8 BGR, dets (n,6) float32 per frame, windows (n_frames, 4) float64 =
    (centre x, centre y, angle rad, zoom) of each frame's window on the canvas)."""
    h, w = hw
    rng = np.random.default_rng(seed)
    margin = int(max_step * n_frames + 0.05 * max(h, w) * (1 + max_rot_deg * n_frames / 10.0)) + 16
    H, W = h + 2 * margin, w + 2 * margin
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    canvas = np.zeros((H, W, 3), np.float32)

    def smooth_field(cell):
        gh, gw = H // cell + 3, W // cell + 3
        g = rng.random((gh, gw)).astype(np.float32)
        fy, fx = yy / cell, xx / cell
        y0, x0 = fy.astype(np.int64), fx.astype(np.int64)
        ay, ax = fy - y0, fx - x0
        return (g[y0, x0] * (1 - ay) * (1 - ax) + g[y0, x0 + 1] * (1 - ay) * ax
                + g[y0 + 1, x0] * ay * (1 - ax) + g[y0 + 1, x0 + 1] * ay * ax)

    for c in range(3):
        canvas[..., c] = smooth_field(56) + 0.5 * smooth_field(28) + 0.08 * rng.random((H, W)).astype(np.float32)
    canvas -= canvas.min()
    canvas = canvas / canvas.max() * 215.0 + 20.0
    cx = rng.uniform(margin + 40, margin + w - 40, n_objects)
    cy = rng.uniform(margin + 40, margin + h - 40, n_objects)
    bw = rng.uniform(18, 46, n_objects)
    bh = rng.uniform(36, 90, n_objects)
    px, py, ang, zoom = W / 2.0, H / 2.0, 0.0, 1.0
    gy, gx = np.mgrid[0:h, 0:w].astype(np.float64)
    gx -= (w - 1) / 2.0
    gy -= (h - 1) / 2.0
    frames, dets, wins = [], [], []
    for f in range(n_frames):
        if f:
            px += rng.uniform(-max_step, max_step)
            py += rng.uniform(-max_step, max_step)
            ang += np.deg2rad(rng.uniform(-max_rot_deg, max_rot_deg))
            zoom *= 1.0 + rng.uniform(-max_zoom, max_zoom)
        wins.append((px, py, ang, zoom))
        ca, sa = np.cos(ang) / zoom, np.sin(ang) / zoom   # image pixel -> canvas point
        sx = px + ca * gx - sa * gy
        sy = py + sa * gx + ca * gy
        x0 = np.clip(np.floor(sx).astype(np.int64), 0, W - 2)
        y0 = np.clip(np.floor(sy).astype(np.int64), 0, H - 2)
        ax = (sx - x0)[..., None]
        ay = (sy - y0)[..., None]
        win = (canvas[y0, x0] * (1 - ay) * (1 - ax) + canvas[y0, x0 + 1] * (1 - ay) * ax
               + canvas[y0 + 1, x0] * ay * (1 - ax) + canvas[y0 + 1, x0 + 1] * ay * ax)
        win = win + rng.normal(0.0, 1.5, (h, w, 3))
        frames.append(np.clip(np.rint(win), 0, 255).astype(np.uint8))
        # canvas point -> image pixel (inverse similarity) for the object centres
        dx, dy = cx - px, cy - py
        ix = (np.cos(ang) * dx + np.sin(ang) * dy) * zoom + (w - 1) / 2.0
        iy = (-np.sin(ang) * dx + np.cos(ang) * dy) * zoom + (h - 1) / 2.0
        x1, y1 = ix - bw * zoom / 2, iy - bh * zoom / 2
        d = np.stack([x1, y1, x1 + bw * zoom, y1 + bh * zoom, rng.uniform(0.55, 0.95, n_objects),
                      np.zeros(n_objects)], 1)
        vis = (rng.random(n_objects) > 0.1) & (d[:, 0] > 0) & (d[:, 1] > 0) & (d[:, 2] < w) & (d[:, 3] < h)
        dets.append(d[vis].astype(np.float32))
    return frames, dets, np.asarray(wins)
