"""Walk an arch-4 (OSNet-AIN / OSNet-IBN) `.b200reid` blob exactly as csrc/reid_model.cu does and evaluate the folded
network with torch ops (NHWC, float32).  Test infrastructure: validates weights.fold_osnet_in against oracle.osnet_in
without a GPU, and documents where each instance norm sits."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from boxmot_b200.weights import ARCH_OSNET_IN, IN_AFTER_RESIDUAL, IN_BEFORE_RESIDUAL, read_blob
from tests.blobsim import LIGHTS, _Cursor, _dw3, _pw


def _inorm(x, gamma, beta):
    """Instance norm of an NHWC map: statistics per crop and channel over H x W (float64), then the affine."""
    xd = x.double()
    mean = xd.mean(dim=(1, 2), keepdim=True)
    var = ((xd - mean) ** 2).mean(dim=(1, 2), keepdim=True)
    return ((xd - mean) / torch.sqrt(var + 1e-5)).float() * gamma + beta


def _block(cur, x, cin, cout, mode):
    mid, hid = cout // 4, cout // 64
    x1 = _pw(x, cur.take(cin, mid), cur.take(mid), True)
    branches = []
    for depth in LIGHTS:
        y = x1
        for _ in range(depth):
            wpw, wdw, bb = cur.take(mid, mid), cur.take(9, mid), cur.take(mid)
            y = _dw3(y @ wpw, wdw, bb)
        branches.append(y)
    w1, b1, w2, b2 = cur.take(mid, hid), cur.take(hid), cur.take(hid, mid), cur.take(mid)
    x2 = 0
    for y in branches:
        g = torch.sigmoid(F.relu(y.mean(dim=(1, 2)) @ w1 + b1) @ w2 + b2)
        x2 = x2 + y * g[:, None, None, :]
    if mode == IN_BEFORE_RESIDUAL:   # conv3 (zero bias) -> IN, downsample on its own, then add and ReLU
        x3 = x2 @ cur.take(mid, cout) + cur.take(cout)
        ident = x @ cur.take(cin, cout) + cur.take(cout) if cin != cout else x
        return F.relu(_inorm(x3, cur.take(cout), cur.take(cout)) + ident)
    if cin != cout:
        z = torch.cat([x2, x], dim=-1) @ cur.take(mid + cin, cout) + cur.take(cout)
    else:
        z = x2 @ cur.take(mid, cout) + cur.take(cout) + x
    if mode == IN_AFTER_RESIDUAL:
        return F.relu(_inorm(z, cur.take(cout), cur.take(cout)))
    return F.relu(z)


@torch.no_grad()
def blob_forward_osnet_in(blob_path, x_nhwc: torch.Tensor, return_stages=False):
    """Arch-4 blob walk: x_nhwc (N,256,128,3) -> (N, feat) un-normalised embedding; NHWC taps named as in
    oracle.osnet_in.osnet_ain_forward."""
    header, payload = read_blob(blob_path)
    assert header[2] == ARCH_OSNET_IN
    c, feat, stem_in, modes = list(header[3:7]), header[7], header[9], header[10:16]
    cur = _Cursor(payload)
    st = {}
    w = cur.take(147, c[0])
    wt = w.view(7, 7, 3, c[0]).permute(3, 2, 0, 1).contiguous()
    x = F.conv2d(x_nhwc.permute(0, 3, 1, 2), wt, None, stride=2, padding=3).permute(0, 2, 3, 1)
    x = _inorm(x, cur.take(c[0]), cur.take(c[0])) if stem_in else x + cur.take(c[0])
    x = st["stem"] = F.relu(x).contiguous()
    x = F.max_pool2d(x.permute(0, 3, 1, 2), 3, stride=2, padding=1).permute(0, 2, 3, 1).contiguous()
    st["pool"] = x
    for s in range(3):
        for j in range(2):
            x = _block(cur, x, c[s] if j == 0 else c[s + 1], c[s + 1], modes[s * 2 + j])
            st[f"conv{s + 2}.{j}"] = x
        if s < 2:
            x = _pw(x, cur.take(c[s + 1], c[s + 1]), cur.take(c[s + 1]), True)
            n, h, wd, ch = x.shape
            x = st[f"conv{s + 2}.2"] = x.view(n, h // 2, 2, wd // 2, 2, ch).mean(dim=(2, 4))
    x = st["conv5"] = _pw(x, cur.take(c[3], c[3]), cur.take(c[3]), True)
    v = F.relu(x.mean(dim=(1, 2)) @ cur.take(c[3], feat) + cur.take(feat))
    assert cur.o == payload.size
    return (v, st) if return_stages else v
