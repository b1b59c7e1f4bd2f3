"""HACNN on the host: the functional oracle (oracle/hacnn.py) against the reference class's embeddings (a strict load and
a hacnn_market1501.pt checkpoint), 160x64 crop staging against the reference's crops, the synthetic state dict against
the reference class's keys and shapes, the arch-8 blob (weights.fold_hacnn) walked in float64 against the oracle, and
the refusal of incomplete or differently shaped state dicts."""
import hashlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import hacnn as oha
from tests.common import GOLDEN

CASES = ("strict", "checkpoint")


def _golden():
    z = np.load(GOLDEN / "reid_hacnn_reference.npz")
    img = np.random.default_rng(int(z["image_seed"])).integers(0, 255, size=(540, 960, 3), dtype=np.uint8)
    return z, img


def _case_state(z, case):
    from boxmot_b200.synthetic import make_hacnn_state

    return make_hacnn_state(seed=int(z[f"{case}_seed"]), num_classes=int(z["num_classes"]))


@pytest.mark.parametrize("mode", ["resize", "resize_pad"])
def test_hacnn_crops_match_reference_golden(mode):
    z, img = _golden()
    crops = oha.get_crops(z["boxes"], img, mode).numpy()
    assert crops.shape[1:] == (3, 160, 64)
    assert hashlib.sha256(np.ascontiguousarray(crops).tobytes()).hexdigest() == str(z[f"crops_sha256_{mode}"])


@pytest.mark.parametrize("mode", ["resize", "resize_pad"])
@pytest.mark.parametrize("case", CASES)
def test_hacnn_oracle_matches_reference_class(case, mode):
    z, img = _golden()
    feats = oha.get_features(_case_state(z, case), z["boxes"], img, mode)
    assert feats.shape == (len(z["boxes"]), 1024)
    np.testing.assert_allclose(feats, z[f"{case}_features_{mode}"], rtol=0, atol=1e-5)   # float32 on both sides


def _bilinear_zero(x, iy, ix):
    """x (N,C,H,W) sampled at per-row iy (N,h) and per-column ix (N,w) with zero padding (grid_sample's taps)."""
    n, c, H, W = x.shape
    y0, x0 = torch.floor(iy), torch.floor(ix)
    out = 0
    for dy in (0, 1):
        for dx in (0, 1):
            yy, xx = y0 + dy, x0 + dx
            wy = (1 - (iy - y0)) if dy == 0 else (iy - y0)
            wx = (1 - (ix - x0)) if dx == 0 else (ix - x0)
            ok = ((yy >= 0) & (yy < H))[:, :, None] & ((xx >= 0) & (xx < W))[:, None, :]
            yi, xi = yy.clamp(0, H - 1).long(), xx.clamp(0, W - 1).long()
            v = x[torch.arange(n)[:, None, None], :, yi[:, :, None], xi[:, None, :]].permute(0, 3, 1, 2)
            out = out + v * (wy[:, :, None] * wx[:, None, :] * ok)[:, None]
    return out


def test_stn_source_coordinates_equal_grid_sample():
    """The closed form the STN kernel uses: ix = j + tx W / 2, iy = ((0.25 y_k + ty + 1) H - 1) / 2."""
    g = torch.Generator().manual_seed(3)
    x = torch.randn(3, 5, 20, 8, generator=g, dtype=torch.float64)
    th = torch.tensor([[0.6, -0.9], [-0.7, 0.95], [0.1, 0.2]], dtype=torch.float64)
    H, W = x.shape[2:]
    ix = torch.arange(W, dtype=torch.float64)[None] + th[:, :1] * W / 2
    yk = (2 * torch.arange(H, dtype=torch.float64) + 1) / H - 1
    iy = ((0.25 * yk[None] + th[:, 1:] + 1) * H - 1) / 2
    assert float((_bilinear_zero(x, iy, ix) - oha.stn(x, th)).abs().max()) < 1e-12


def blob_forward_hacnn(blob, x):
    """Float64 walk of an arch-8 blob (the order csrc/reid_model.cu reads it) on NCHW x: (v, theta (N, 3, 8))."""
    from boxmot_b200.weights import read_blob

    _, payload = read_blob(blob)
    p = torch.from_numpy(payload.astype(np.float64))
    o = 0

    def take(*shape):
        nonlocal o
        n = int(np.prod(shape))
        t = p[o:o + n].reshape(shape)
        o += (n + 3) // 4 * 4
        return t

    def cb(x, co, k=1, stride=1):
        w = take(k * k * x.shape[1], co).reshape(k, k, x.shape[1], co).permute(3, 2, 0, 1)
        return F.relu(F.conv2d(x, w, take(co), stride=stride, padding=k // 2))

    def inc_a(x, c):
        mid = c // 4
        s = [cb(cb(x, mid), mid, 3) for _ in range(3)]
        return torch.cat(s + [cb(F.avg_pool2d(x, 3, 1, 1), mid)], 1)

    def inc_b(x, c):
        mid = c // 4
        s1 = cb(cb(x, mid), mid, 3, 2)
        s2 = cb(cb(cb(x, mid), mid, 3), mid, 3, 2)
        return torch.cat([s1, s2, cb(F.max_pool2d(x, 3, 2, 1), 2 * mid)], 1)

    x = cb(x.double(), 32, 3, 2)
    outs, xs, thetas = [x], [], []
    for c in (128, 256, 384):
        xi = inc_b(inc_a(outs[-1], c), c)
        sp = take(12)
        m = F.conv2d(xi.mean(1, keepdim=True), sp[:9].view(1, 1, 3, 3), sp[9:10], stride=2, padding=1)
        m = F.interpolate(F.relu(m), scale_factor=2, mode="bilinear", align_corners=True)
        s = F.relu(sp[10] * m + sp[11])
        g = xi.mean(dim=(2, 3))
        ch = F.relu(g @ take(c, c // 16) + take(c // 16))
        ch = F.relu(ch @ take(c // 16, c) + take(c))
        v = ch @ take(c, c)
        attn = torch.sigmoid(F.relu(s * v[:, :, None, None] + take(c)[None, :, None, None]))
        thetas.append(torch.tanh(g @ take(c, 8) + take(8)))
        xs.append(xi)
        outs.append(xi * attn)
    local = 0
    for i, c in enumerate((128, 256, 384)):   # the four regions as one batch [region][crop]: each layer is read once
        th = thetas[i].view(-1, 4, 2)
        t = torch.cat([oha.stn(outs[i], th[:, r]) for r in range(4)])
        local = inc_b(F.interpolate(t, oha.LOCAL_HW[i], mode="bilinear", align_corners=True) + local, c)
    xg = F.relu(outs[3].mean(dim=(2, 3)) @ take(384, 512) + take(512))
    xl = torch.cat(local.mean(dim=(2, 3)).chunk(4), 1)
    xl = F.relu(xl @ take(1536, 512) + take(512))
    assert o == payload.size
    return torch.cat([xg, xl], 1), torch.stack(thetas, 1)


def test_hacnn_folded_blob_equals_oracle(tmp_path):
    from boxmot_b200.weights import ARCH_HACNN, export_blob, read_blob

    z, _ = _golden()
    sd = _case_state(z, "strict")
    blob = export_blob(sd, tmp_path / "hacnn.b200reid")
    header, _ = read_blob(blob)
    assert header[2] == ARCH_HACNN and header[3:8] == (32, 128, 256, 384, 1024) and header[9:11] == (160, 64)
    x = torch.randn(2, 3, 160, 64, generator=torch.Generator().manual_seed(1))
    want, st = oha.hacnn_forward({k: v.double() for k, v in sd.items()}, x.double(), return_stages=True)
    got, theta = blob_forward_hacnn(blob, x)
    assert float((theta - st["theta"]).abs().max()) < 1e-6
    assert float((got - want).abs().max()) < 1e-6 * max(1.0, float(want.abs().max()))   # float32 weights
    # the regions move off centre, and some leave the map (|tx| > 0.5 or |ty| > 0.75 puts a region partly outside)
    tx, ty = st["theta"][..., 0::2], st["theta"][..., 1::2]
    assert float(tx.abs().max()) > 0.3 and bool(((tx.abs() > 0.5) | (ty.abs() > 0.75)).any())


def test_hacnn_checkpoint_roundtrip(tmp_path):
    """A checkpoint saved like the released hacnn_market1501.pt (`state_dict`, `module.` prefixes, classifiers
    included) converts to the same blob as the bare state dict."""
    from boxmot_b200.synthetic import make_hacnn_state
    from boxmot_b200.weights import export_blob, read_blob

    sd = make_hacnn_state(seed=4)
    pt = tmp_path / "hacnn_market1501.pt"
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, pt)
    blob = export_blob(pt)
    plain = export_blob({k: v for k, v in sd.items() if not k.startswith("classifier_")}, tmp_path / "p.b200reid")
    assert blob.read_bytes() == plain.read_bytes()
    header, payload = read_blob(blob)
    assert header[7] == 1024 and payload.size == header[8]


def test_hacnn_variants_are_refused(tmp_path):
    from boxmot_b200.synthetic import make_hacnn_state
    from boxmot_b200.weights import export_blob

    sd = make_hacnn_state(seed=1)
    missing = dict(sd)
    missing.pop("inception2.1.stream2.2.bn.running_var")
    with pytest.raises(ValueError, match="inception2.1.stream2.2.bn.running_var"):
        export_blob(missing, tmp_path / "missing.b200reid")
    no_region = {k: v for k, v in sd.items() if not k.startswith(("local_conv", "fc_local", "classifier_local"))}
    with pytest.raises(ValueError, match="missing keys .'fc_local"):
        export_blob(no_region, tmp_path / "noregion.b200reid")


@pytest.mark.parametrize("kw", [{"nchannels": [64, 128, 256]}, {"feat_dim": 256}, {"learn_region": False}])
def test_reference_hacnn_variants_are_refused(tmp_path, kw):
    refharness = pytest.importorskip("tests.golden.refharness")
    if not refharness.reference_available():
        pytest.skip("reference tree not present")
    refharness.install_reference()
    from boxmot.reid.backbones.hacnn import HACNN

    from boxmot_b200.weights import export_blob

    m = HACNN(10, **kw)
    with pytest.raises(ValueError, match="not a HACNN state dict"):
        export_blob(m.state_dict(), tmp_path / "variant.b200reid")


def test_reference_hacnn_state_dict_keys_match_synthetic():
    refharness = pytest.importorskip("tests.golden.refharness")
    if not refharness.reference_available():
        pytest.skip("reference tree not present")
    refharness.install_reference()
    from boxmot.reid.backbones.hacnn import HACNN

    from boxmot_b200.synthetic import make_hacnn_state

    ref = HACNN(751).state_dict()
    syn = make_hacnn_state(seed=0)
    assert len(ref) == 535
    assert sorted(ref) == sorted(syn)
    assert all(tuple(ref[k].shape) == tuple(syn[k].shape) for k in ref)
