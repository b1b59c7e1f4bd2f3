"""Walk an arch-3 (LMBN_n) `.b200reid` blob exactly as csrc/reid_model.cu does and evaluate the folded network with
torch ops (NHWC, float32).  Test infrastructure: validates weights.fold_lmbn_n against oracle.lmbn without a GPU."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from boxmot_b200.weights import read_blob
from tests.blobsim import LIGHTS, _Cursor, _dw3, _pw


def _osblock(cur, x, cin, cout):
    """One OSBlock of the blob walk (NHWC): conv1, the four LightConv3x3 branches, the shared gate, conv3 (+ downsample)."""
    mid, hid = cout // 4, cout // 64
    x1 = _pw(x, cur.take(cin, mid), cur.take(mid), True)
    x2 = 0
    branches = []
    for depth in LIGHTS:
        y = x1
        for _ in range(depth):
            wpw, wdw, bb = cur.take(mid, mid), cur.take(9, mid), cur.take(mid)
            y = _dw3(y @ wpw, wdw, bb)
        branches.append(y)
    w1, b1, w2, b2 = cur.take(mid, hid), cur.take(hid), cur.take(hid, mid), cur.take(mid)
    for y in branches:
        g = torch.sigmoid(F.relu(y.mean(dim=(1, 2)) @ w1 + b1) @ w2 + b2)
        x2 = x2 + y * g[:, None, None, :]
    if cin != cout:
        return F.relu(torch.cat([x2, x], dim=-1) @ cur.take(mid + cin, cout) + cur.take(cout))
    return F.relu(x2 @ cur.take(mid, cout) + cur.take(cout) + x)


def _transition(cur, x, c):
    x = _pw(x, cur.take(c, c), cur.take(c), True)
    n, h, wd, ch = x.shape
    return x.view(n, h // 2, 2, wd // 2, 2, ch).mean(dim=(2, 4))


LMBN_BRANCHES = ("global_branch", "partial_branch", "channel_branch")


@torch.no_grad()
def blob_forward_lmbn(blob_path, x_nhwc: torch.Tensor, return_stages=False):
    """Arch-3 (LMBN_n) blob walk: x_nhwc (N,384,128,3) -> (N, 3584) un-normalised, interleaved embedding.  Stage taps are
    NHWC and named as in oracle.reid.lmbn_n_forward."""
    header, payload = read_blob(blob_path)
    assert header[2] == 3 and header[9] == x_nhwc.shape[1]
    cur = _Cursor(payload)
    st = {}
    w, b = cur.take(147, 64), cur.take(64)
    x = F.relu(F.conv2d(x_nhwc.permute(0, 3, 1, 2), w.view(7, 7, 3, 64).permute(3, 2, 0, 1).contiguous(), b, stride=2,
                        padding=3))
    st["stem"] = x.permute(0, 2, 3, 1).contiguous()
    x = F.max_pool2d(x, 3, stride=2, padding=1).permute(0, 2, 3, 1).contiguous()
    st["pool"] = x
    x = st["backone.2.0"] = _osblock(cur, x, 64, 256)
    x = st["backone.2.1"] = _osblock(cur, x, 256, 256)
    x = st["backone.2.2"] = _transition(cur, x, 256)
    trunk = st["trunk"] = _osblock(cur, x, 256, 384)
    outs = {}
    for br in LMBN_BRANCHES:
        y = st[f"{br}.0.1"] = _osblock(cur, trunk, 384, 384)
        y = st[f"{br}.0.2"] = _transition(cur, y, 384)
        y = st[f"{br}.1.0"] = _osblock(cur, y, 384, 512)
        y = st[f"{br}.1.1"] = _osblock(cur, y, 512, 512)
        outs[br] = st[f"{br}.2"] = _pw(y, cur.take(512, 512), cur.take(512), True)
    glo = st["bottleneck"] = _osblock(cur, outs["global_branch"], 512, 512)
    par, cha = outs["partial_branch"], outs["channel_branch"]
    h = par.shape[1]
    pooled = [glo.mean(dim=(1, 2)), glo.amax(dim=(1, 2)), par.amax(dim=(1, 2)), par[:, : h // 2].mean(dim=(1, 2)),
              par[:, h // 2:].mean(dim=(1, 2))]
    feats = [p @ cur.take(512, 512) + cur.take(512) for p in pooled]
    wsh, bsh = cur.take(256, 512), cur.take(512)
    c = cha.mean(dim=(1, 2))
    hs = [F.relu(c[:, :256] @ wsh + bsh), F.relu(c[:, 256:] @ wsh + bsh)]
    for hj in hs:
        s, t = cur.take(512), cur.take(512)
        feats.append(hj * s + t)
    assert cur.o == payload.size
    v = torch.stack(feats, dim=2).flatten(1, 2)
    return (v, st) if return_stages else v
