"""MLFN on the host: the functional oracle (oracle/mlfn.py) against the reference class's embeddings (a strict load and
an mlfn_market1501.pt checkpoint), crop staging against the reference's crops, the synthetic state dict against the
reference class's keys and shapes, the arch-7 blob (weights.fold_mlfn) walked in float64 against the oracle, and the
refusal of incomplete or differently shaped state dicts."""
import hashlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import mlfn as oml
from oracle.reid import get_crops
from tests.common import GOLDEN

CASES = ("strict", "checkpoint")


def _golden():
    z = np.load(GOLDEN / "reid_mlfn_reference.npz")
    img = np.random.default_rng(int(z["image_seed"])).integers(0, 255, size=(540, 960, 3), dtype=np.uint8)
    return z, img


def _case_state(z, case):
    from boxmot_b200.synthetic import make_mlfn_state

    return make_mlfn_state(seed=int(z[f"{case}_seed"]), num_classes=int(z["num_classes"]))


@pytest.mark.parametrize("mode", ["resize", "resize_pad"])
def test_mlfn_crops_match_reference_golden(mode):
    z, img = _golden()
    crops = get_crops(z["boxes"], img, mode).numpy()
    assert hashlib.sha256(np.ascontiguousarray(crops).tobytes()).hexdigest() == str(z[f"crops_sha256_{mode}"])


@pytest.mark.parametrize("mode", ["resize", "resize_pad"])
@pytest.mark.parametrize("case", CASES)
def test_mlfn_oracle_matches_reference_class(case, mode):
    z, img = _golden()
    feats = oml.get_features(_case_state(z, case), z["boxes"], img, mode)
    assert feats.shape == (len(z["boxes"]), 1024)
    np.testing.assert_allclose(feats, z[f"{case}_features_{mode}"], rtol=0, atol=2e-6)


def blob_forward_mlfn(blob, x):
    """Float64 walk of an arch-7 blob (the order csrc/reid_model.cu reads it) on NCHW x: (v, s_hat)."""
    from boxmot_b200.synthetic import mlfn_blocks
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

    def pw(x, ci, co, stride=1):   # K-major [ci][co] 1x1 convolution + bias
        w = take(ci, co)
        return F.conv2d(x[:, :, ::stride, ::stride], w.t()[:, :, None, None]) + take(co).view(1, -1, 1, 1)

    x = x.double()
    w = take(147, 64).reshape(7, 7, 3, 64).permute(3, 2, 0, 1)
    x = F.max_pool2d(F.relu(F.conv2d(x, w, stride=2, padding=3) + take(64).view(1, -1, 1, 1)), 3, 2, 1)
    gates = []
    for cin, cout, stride, (f0, f1), ds in mlfn_blocks():
        mid, gw = cout // 2, cout // 64
        s = x.mean(dim=(2, 3), keepdim=True)
        s = torch.sigmoid(pw(F.relu(pw(F.relu(pw(s, cin, f0)), f0, f1)), f1, 32))
        gates.append(s.flatten(1))
        y = F.relu(pw(x, cin, mid))
        w2 = take(9, gw, mid).reshape(3, 3, gw, mid).permute(3, 2, 0, 1)   # [mid][gw][3][3]
        y = F.relu(F.conv2d(y, w2, stride=stride, padding=1, groups=32) + take(mid).view(1, -1, 1, 1))
        y = y * s.flatten(1).repeat_interleave(gw, dim=1)[:, :, None, None]
        y = F.relu(pw(y, mid, cout))
        x = F.relu((pw(x, cin, cout, stride) if ds else x) + y)
    s_hat = torch.cat(gates, 1)
    xv = F.relu(pw(x.mean(dim=(2, 3), keepdim=True), 2048, 1024))
    sv = F.relu(pw(s_hat[:, :, None, None], 512, 1024))
    assert o == payload.size
    return ((xv + sv) * 0.5).flatten(1), s_hat


def test_mlfn_folded_blob_equals_oracle(tmp_path):
    from boxmot_b200.weights import ARCH_MLFN, export_blob, read_blob

    z, _ = _golden()
    sd = _case_state(z, "strict")
    blob = export_blob(sd, tmp_path / "mlfn.b200reid")
    header, _ = read_blob(blob)
    assert header[2] == ARCH_MLFN and header[3:8] == (64, 2048, 32, 16, 1024)
    x = torch.randn(2, 3, 256, 128, generator=torch.Generator().manual_seed(1))
    want, st = oml.mlfn_forward({k: v.double() for k, v in sd.items()}, x.double(), return_stages=True)
    got, s_hat = blob_forward_mlfn(blob, x)
    assert float((s_hat - st["s_hat"]).abs().max()) < 1e-6
    assert float((got - want).abs().max()) < 1e-6 * max(1.0, float(want.abs().max()))   # float32 weights
    # the gates are not saturated: the FSM path is exercised
    assert 0.05 < float(st["s_hat"].mean()) < 0.95 and float(st["s_hat"].std()) > 0.05


def test_mlfn_checkpoint_roundtrip(tmp_path):
    """A checkpoint saved like the released mlfn_market1501.pt (`state_dict`, `module.` prefixes, classifier
    included) converts to the same blob as the bare state dict."""
    from boxmot_b200.synthetic import make_mlfn_state
    from boxmot_b200.weights import export_blob, read_blob

    sd = make_mlfn_state(seed=4)
    pt = tmp_path / "mlfn_market1501.pt"
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, pt)
    blob = export_blob(pt)
    plain = export_blob({k: v for k, v in sd.items() if not k.startswith("classifier.")}, tmp_path / "p.b200reid")
    assert blob.read_bytes() == plain.read_bytes()
    header, payload = read_blob(blob)
    assert header[7] == 1024 and payload.size == header[8]


def test_mlfn_variants_are_refused(tmp_path):
    from boxmot_b200.synthetic import make_mlfn_state
    from boxmot_b200.weights import export_blob

    sd = make_mlfn_state(seed=1)
    missing = dict(sd)
    missing.pop("feature.5.fm_bn2.running_var")
    with pytest.raises(ValueError, match="feature.5.fm_bn2.running_var"):
        export_blob(missing, tmp_path / "missing.b200reid")
    short = {k: v for k, v in sd.items() if not k.startswith("feature.15.")}   # a truncated `feature` list
    with pytest.raises(ValueError, match="feature.15"):
        export_blob(short, tmp_path / "short.b200reid")


@pytest.mark.parametrize("kw", [{"groups": 16}, {"embed_dim": 512}])
def test_reference_mlfn_variants_are_refused(tmp_path, kw):
    refharness = pytest.importorskip("tests.golden.refharness")
    if not refharness.reference_available():
        pytest.skip("reference tree not present")
    refharness.install_reference()
    from boxmot.reid.backbones import mlfn as ref_mlfn

    from boxmot_b200.weights import export_blob

    m = ref_mlfn.mlfn(num_classes=10, pretrained=False, **kw)
    with pytest.raises(ValueError, match="not an MLFN state dict"):
        export_blob(m.state_dict(), tmp_path / "variant.b200reid")


def test_reference_mlfn_state_dict_keys_match_synthetic():
    refharness = pytest.importorskip("tests.golden.refharness")
    if not refharness.reference_available():
        pytest.skip("reference tree not present")
    refharness.install_reference()
    from boxmot.reid.backbones import mlfn as ref_mlfn

    from boxmot_b200.synthetic import make_mlfn_state

    ref = ref_mlfn.mlfn(num_classes=751, pretrained=False).state_dict()
    syn = make_mlfn_state(seed=0)
    assert len(ref) == 669
    assert sorted(ref) == sorted(syn)
    assert all(tuple(ref[k].shape) == tuple(syn[k].shape) for k in ref)
