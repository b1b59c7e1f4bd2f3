"""ViT-Nano / ViT-Tiny on the host: the functional oracle (tests/vit_oracle.py) against the reference's embeddings of
all six variants (trainer-format checkpoints loaded by the reference's own loader), crop staging at 256x128 and 384x128
against the reference's crops, the arch-9 blob (weights.fold_vit) walked in float64 against the oracle, the checkpoint
round trip with the reference's name resolution (checkpoint `model_name` before the file name), the refusals, and the
properties of the synthetic weights that make the tests meaningful (non-uniform attention, AIN gates off 0.5)."""
import hashlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from boxmot_b200.weights import VIT_VARIANTS
from tests import vit_oracle as ov
from tests.common import GOLDEN

VARIANTS = tuple(VIT_VARIANTS)


def _golden():
    z = np.load(GOLDEN / "reid_vit_reference.npz")
    img = np.random.default_rng(int(z["image_seed"])).integers(0, 255, size=(540, 960, 3), dtype=np.uint8)
    return z, img


def _state(z, variant):
    from boxmot_b200.synthetic import make_vit_state

    return make_vit_state(variant, int(z[f"{variant}_seed"]), num_classes=int(z["num_classes"]))


@pytest.mark.parametrize("mode", ["resize", "resize_pad"])
@pytest.mark.parametrize("variant", ["vit_nano", "vit_tiny"])
def test_vit_crops_match_reference_golden(variant, mode):
    z, img = _golden()
    hw = ov.input_hw(variant)
    crops = ov.get_crops(z["boxes"], img, mode, hw).numpy()
    assert crops.shape == (len(z["boxes"]), 3, *hw)
    assert hashlib.sha256(np.ascontiguousarray(crops).tobytes()).hexdigest() == str(z[f"{variant}_crops_sha256_{mode}"])


@pytest.mark.parametrize("mode", ["resize", "resize_pad"])
@pytest.mark.parametrize("variant", VARIANTS)
def test_vit_oracle_matches_reference(variant, mode):
    """The reference runs in float32, the oracle in float64: on these weights the two differ by at most 7.9e-7 on
    L2-normalised rows whose largest entry is 0.11-0.37, so 2e-6 leaves a margin of 2.5."""
    z, img = _golden()
    feats = ov.get_features(_state(z, variant), variant, z["boxes"], img, mode)
    want = z[f"{variant}_features_{mode}"]
    assert feats.shape == want.shape
    np.testing.assert_allclose(feats, want, rtol=0, atol=2e-6)


def blob_forward_vit(blob, x):
    """Float64 walk of an arch-9 blob (the order csrc/reid_model.cu reads it) on NCHW x: the un-normalised row."""
    from boxmot_b200.weights import read_blob

    header, payload = read_blob(blob)
    p = torch.from_numpy(payload.astype(np.float64))
    o = 0

    def take(*shape):
        nonlocal o
        n = int(np.prod(shape))
        t = p[o:o + n].reshape(shape)
        o += (n + 3) // 4 * 4
        return t

    d, depth, heads, n_ain, feat = header[3:8]
    _, _, gh, gw, stride, pool, proj = header[9:16]
    T = 1 + gh * gw
    x = x.double()
    n = x.shape[0]
    patches = F.unfold(x.permute(0, 2, 3, 1).permute(0, 3, 1, 2), 16, stride=stride)   # (n, 3*256, P), k = ci*256 + tap
    patches = patches.reshape(n, 3, 256, gh * gw).permute(0, 3, 2, 1).reshape(n, gh * gw, 768)   # k = tap*3 + ci
    w, b = take(768, d), take(d)
    h = torch.cat([torch.zeros(n, 1, d, dtype=torch.float64), patches @ w + b], 1) + take(T, d)
    ln = lambda t: F.layer_norm(t, (d,), eps=1e-5)   # noqa: E731
    for i in range(depth):
        if i < n_ain:
            a, c, s = take(d), take(d), take(d)
            xin = F.instance_norm(h.transpose(1, 2), eps=1e-5).transpose(1, 2)
            y = a * xin + c * ln(h) + s
        else:
            y = ln(h) * take(d) + take(d)
        qkv = y @ take(d, 3 * d) + take(3 * d)
        q, k, v = (z.reshape(n, T, heads, 64).transpose(1, 2) for z in qkv.split(d, -1))
        att = (torch.softmax(q @ k.transpose(-1, -2), -1) @ v).transpose(1, 2).reshape(n, T, d)   # q pre-scaled
        h = h + att @ take(d, d) + take(d)
        y = ln(h) * take(d) + take(d)
        m = F.gelu(y @ take(d, 4 * d) + take(4 * d))
        h = h + m @ take(4 * d, d) + take(d)
    h = ln(h) * take(d) + take(d)
    if pool == 1:
        pm = h[:, 1:].mean(1)
        gs = [(take(d), take(d)) for _ in range(4)]
        w1, b1, w2, b2 = take(d, 12), take(12), take(12, d), take(d)
        f = 0
        for g, bb in gs:
            qv = ln(pm) * g + bb
            f = f + torch.sigmoid(torch.relu(qv @ w1 + b1) @ w2 + b2) * qv
        row = f * take(d) + take(d)
    elif not proj:
        row = h[:, 0] * take(d) + take(d)
    else:
        vecs = [h[:, 0]]
        sp = h[:, 1:].reshape(n, gh, gw, d)
        for i in range(pool):
            r0 = i * (gh // pool)
            r1 = gh if i == pool - 1 else r0 + gh // pool
            vecs.append(sp[:, r0:r1].mean((1, 2)))
        row = torch.cat([v @ take(d, proj) + take(proj) for v in vecs], 1)
    assert o == payload.size and row.shape[1] == feat
    return row


@pytest.mark.parametrize("variant", VARIANTS)
def test_vit_folded_blob_equals_oracle(tmp_path, variant):
    from boxmot_b200.synthetic import make_vit_state
    from boxmot_b200.weights import ARCH_VIT, export_blob, read_blob, vit_grid

    sd = make_vit_state(variant, 3)
    blob = export_blob(sd, tmp_path / f"{variant}.b200reid")
    header, _ = read_blob(blob)
    h, w, stride, gh, gw, _ = vit_grid(variant)
    depth, n_ain, omni, parts, *_ = VIT_VARIANTS[variant]
    tiny = variant.startswith("vit_tiny")
    feat = (1 + parts) * 512 if tiny else 192
    assert header[2] == ARCH_VIT and header[3:8] == (192, depth, 3, n_ain, feat)
    assert header[9:16] == (h, w, gh, gw, stride, 1 if omni else parts, 512 if tiny else 0)
    x = torch.randn(2, 3, h, w, generator=torch.Generator().manual_seed(1))
    want = ov.vit_forward(ov.double_state(sd), variant, x.double())
    got = blob_forward_vit(blob, x)
    assert float((got - want).abs().max()) < 1e-5 * max(1.0, float(want.abs().max()))   # float32 weights


def _save(path, sd, model_name=None, prefix=True):
    ckpt = {"state_dict": {("module." + k if prefix else k): v for k, v in sd.items()}}
    if model_name:
        ckpt["model_name"] = model_name
    torch.save(ckpt, path)


@pytest.mark.parametrize("variant", VARIANTS)
def test_vit_checkpoint_roundtrip(tmp_path, variant):
    """A trainer-format checkpoint (`state_dict` with `module.` prefixes, classifiers, `model_name`) gives the blob of
    the bare state dict; the checkpoint's model_name decides the variant whatever the file name says."""
    from boxmot_b200.synthetic import make_vit_state
    from boxmot_b200.weights import export_blob, read_blob

    sd = make_vit_state(variant, 4)
    bare = {k: v for k, v in sd.items() if "classifier" not in k and "num_batches" not in k}
    plain = export_blob(bare, tmp_path / "bare.b200reid")
    pt = tmp_path / f"{variant}_market1501.pt"
    _save(pt, sd, model_name=variant)
    assert export_blob(pt).read_bytes() == plain.read_bytes()
    named = tmp_path / "reid_weights.pt"   # no model type in the file name: the checkpoint's name decides
    _save(named, sd, model_name=variant)
    assert export_blob(named).read_bytes() == plain.read_bytes()
    by_file = tmp_path / f"my_{variant}_msmt17.pt"   # no model_name: the longest model type in the file name
    _save(by_file, sd, prefix=False)
    assert export_blob(by_file).read_bytes() == plain.read_bytes()
    header, payload = read_blob(plain)
    assert payload.size == header[8]


def test_vit_model_name_takes_precedence_over_the_file_name(tmp_path):
    """vit_tiny_parts3 weights hold every vit_tiny tensor: saved with model_name "vit_tiny" under a parts3 file name,
    the reference builds vit_tiny and discards the part heads, and so does the export."""
    from boxmot_b200.synthetic import make_vit_state
    from boxmot_b200.weights import export_blob, read_blob

    sd = make_vit_state("vit_tiny_parts3", 5)
    pt = tmp_path / "vit_tiny_parts3_market1501.pt"
    _save(pt, sd, model_name="vit_tiny")
    header, _ = read_blob(export_blob(pt))
    assert header[7] == 512 and header[14] == 0
    _save(pt, sd)
    header, _ = read_blob(export_blob(pt))
    assert header[7] == 2048 and header[14] == 3


def test_vit_missing_or_misshaped_tensors_are_refused(tmp_path):
    from boxmot_b200.synthetic import make_vit_state
    from boxmot_b200.weights import export_blob

    sd = make_vit_state("vit_tiny_parts", 1)
    missing = dict(sd)
    missing.pop("blocks.7.mlp.fc1.bias")
    with pytest.raises(ValueError, match="blocks.7.mlp.fc1.bias"):
        export_blob(missing, tmp_path / "missing.b200reid")
    pt = tmp_path / "vit_tiny_parts3_market1501.pt"   # a 2-part checkpoint under a 3-part name
    _save(pt, sd)
    with pytest.raises(ValueError, match="part_bns.2"):
        export_blob(pt)
    wide = dict(sd)
    wide["pos_embed"] = torch.zeros(1, 129, 192)   # a 256x128 table under a vit_tiny model
    with pytest.raises(ValueError, match="pos_embed"):
        export_blob(wide, tmp_path / "wide.b200reid")
    nano = make_vit_state("vit_nano_ain", 2)
    pt = tmp_path / "vit_nano_ain_os_duke.pt"   # no omni-scale head in the file
    _save(pt, nano)
    with pytest.raises(ValueError, match="os_agg"):
        export_blob(pt)


@pytest.mark.parametrize("fname", ["vit_tiny_veri.pt", "vit_nano_vehicleid.pt"])
def test_vit_vehicle_file_names_are_refused(tmp_path, fname):
    """The reference builds 256x256 crops for a veri / vehicleid file name, which no ViT positional table fits."""
    from boxmot_b200.synthetic import make_vit_state
    from boxmot_b200.weights import export_blob

    pt = tmp_path / fname
    _save(pt, make_vit_state(fname.rsplit("_", 1)[0], 0))
    with pytest.raises(ValueError, match="256x256"):
        export_blob(pt)


@pytest.mark.parametrize("name", ["osnet_x0_25_market1501.pt", "csl_tinyvit_7m_market1501.pt"])
def test_vit_weights_under_another_model_name_are_refused(tmp_path, name):
    from boxmot_b200.synthetic import make_vit_state
    from boxmot_b200.weights import export_blob

    pt = tmp_path / name
    _save(pt, make_vit_state("vit_nano", 0))
    with pytest.raises(ValueError):
        export_blob(pt)


@pytest.mark.parametrize("variant", ["vit_nano_ain_os", "vit_tiny_parts3"])
def test_synthetic_vit_attention_is_not_uniform(variant):
    """Uniform attention (every probability 1/T) would make the attention kernel's softmax and P.V untestable: the
    synthetic qkv puts the largest probability of every row well above 1/T."""
    from boxmot_b200.synthetic import make_vit_state

    sd = ov.double_state(make_vit_state(variant, 3))
    h, w = ov.input_hw(variant)
    x = torch.rand(2, 3, h, w, generator=torch.Generator().manual_seed(2)).double() * 2 - 1
    T = 1 + ((h - 16) // VIT_VARIANTS[variant][6] + 1) * ((w - 16) // VIT_VARIANTS[variant][6] + 1)
    for block in (0, VIT_VARIANTS[variant][0] - 1):
        rm = ov.attention_row_max(sd, variant, x, block)
        assert float(rm.mean()) > 10.0 / T and float(rm.min()) > 3.0 / T


def test_synthetic_vit_ain_gates_are_far_from_one_half():
    from boxmot_b200.synthetic import make_vit_state

    sd = make_vit_state("vit_nano_ain", 0)
    for i in range(3):
        g = torch.sigmoid(sd[f"blocks.{i}.norm1.gate"])
        assert float((g - 0.5).abs().min()) > 0.2
