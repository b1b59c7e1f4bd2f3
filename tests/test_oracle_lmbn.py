"""LMBN_n on the host: the functional oracle (oracle/lmbn.py) against the reference class's embeddings, 384x128 crop
staging against the reference's crops, the arch-3 blob (weights.fold_lmbn_n) walked by tests/blobsim_lmbn.py against the
oracle, checkpoint round trip, refusal of other LMBN variants, and the other architectures' blobs unchanged."""
import hashlib

import numpy as np
import pytest
import torch

from oracle import lmbn as olm
from tests.common import GOLDEN


def _golden():
    z = np.load(GOLDEN / "reid_lmbn_n_reference.npz")
    img = np.random.default_rng(int(z["image_seed"])).integers(0, 255, size=(540, 960, 3), dtype=np.uint8)
    return z, img


@pytest.mark.parametrize("mode", ["resize", "resize_pad"])
def test_lmbn_crops_match_reference_golden(mode):
    z, img = _golden()
    crops = olm.get_crops_hw(z["boxes"], img, mode, olm.LMBN_INPUT_HW).numpy()
    assert crops.shape == (len(z["boxes"]), 3, 384, 128)
    assert hashlib.sha256(np.ascontiguousarray(crops).tobytes()).hexdigest() == str(z[f"crops_sha256_{mode}"])


@pytest.mark.parametrize("mode", ["resize", "resize_pad"])
def test_lmbn_oracle_matches_reference_class(mode):
    from boxmot_b200.synthetic import make_lmbn_n_state

    z, img = _golden()
    sd = make_lmbn_n_state(seed=int(z["weight_seed"]), num_classes=int(z["num_classes"]))
    feats = olm.get_features_any(sd, z["boxes"], img, mode)
    assert feats.shape == (len(z["boxes"]), 3584)
    np.testing.assert_allclose(feats, z[f"features_{mode}"], rtol=0, atol=2e-6)
    assert abs(np.linalg.norm(feats, axis=1) - 1).max() < 1e-6


def test_lmbn_folded_blob_equals_oracle(tmp_path):
    from boxmot_b200.synthetic import make_lmbn_n_state
    from boxmot_b200.weights import export_blob, read_blob
    from tests.blobsim_lmbn import blob_forward_lmbn

    sd = make_lmbn_n_state(seed=3)
    blob = export_blob(sd, tmp_path / "lmbn_n.b200reid")
    header, _ = read_blob(blob)
    assert header[2] == 3 and header[3:8] == (64, 256, 384, 512, 3584) and header[9] == 384
    x = torch.randn(2, 3, 384, 128)
    want, st_w = olm.lmbn_n_forward(sd, x, return_stages=True)
    got, st_g = blob_forward_lmbn(blob, x.permute(0, 2, 3, 1).contiguous(), return_stages=True)
    assert sorted(st_g) == sorted(st_w)
    for k in st_w:
        w = st_w[k].permute(0, 2, 3, 1).numpy()
        assert np.abs(st_g[k].numpy() - w).max() < 2e-5 * max(1.0, float(np.abs(w).max())), k
    scale = float(want.abs().max())
    assert float((got - want).abs().max()) < 2e-6 * max(scale, 1.0)


def test_lmbn_pt_roundtrip(tmp_path):
    from boxmot_b200.synthetic import make_lmbn_n_state
    from boxmot_b200.weights import export_blob, read_blob

    sd = make_lmbn_n_state(seed=4)
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, tmp_path / "lmbn_n_duke.pt")
    blob = export_blob(tmp_path / "lmbn_n_duke.pt")
    header, payload = read_blob(blob)
    assert header[3:8] == (64, 256, 384, 512, 3584) and payload.size == header[8]


def test_other_lmbn_variants_are_refused(tmp_path):
    """lmbn_ain_n replaces BatchNorm by instance norms in parts of the network: its state dict must be refused, never
    misread as LMBN_n."""
    from boxmot_b200.synthetic import make_lmbn_n_state
    from boxmot_b200.weights import export_blob

    sd = make_lmbn_n_state(seed=1)
    ain = dict(sd)
    for k in [k for k in sd if k.startswith("backone.2.0.conv1.bn.")]:   # an IBN-style layer: instance-norm affine only
        ain[k.replace("conv1.bn.", "conv1.IN.")] = ain.pop(k)
    with pytest.raises(ValueError):
        export_blob(ain, tmp_path / "ain.b200reid")
    missing = dict(sd)
    missing.pop("shared.1.running_var")
    with pytest.raises(ValueError):
        export_blob(missing, tmp_path / "missing.b200reid")


def test_lmbn_ain_n_reference_state_dict_is_refused(tmp_path):
    """The reference's own LMBN_ain_n class, built without downloads, yields a state dict export_blob refuses."""
    refharness = pytest.importorskip("tests.golden.refharness")
    if not refharness.reference_available():
        pytest.skip("reference tree not present")
    refharness.install_reference()
    from boxmot.reid.backbones.lmbn.lmbn_ain_n import LMBN_ain_n

    from boxmot_b200.weights import export_blob

    m = LMBN_ain_n(num_classes=702, loss="softmax", pretrained=False, use_gpu=False)
    with pytest.raises(ValueError):
        export_blob(m.state_dict(), tmp_path / "lmbn_ain_n.b200reid")


# sha256 of blobs exported at the parent of the LMBN_n change: adding arch 3 leaves the other layouts byte-identical
BLOB_SHA256 = {
    "osnet_x0_25": "28bdec0ba171455dd946e0f6f13634d8a1cb08c1d51505cbcf8a1adff35b5b42",
    "osnet_x1_0": "05c009cd1dcd1a2d97261ac5152d4e46bbc323f0a1a7c2818a55f9d5a28272c2",
    "mobilenetv2_x1_4": "c4a6ed20fc466ad815b5b33123c16a7b74924dc0ad4cb7cd8a830700127dd642",
}


@pytest.mark.parametrize("arch", sorted(BLOB_SHA256))
def test_existing_blob_layouts_unchanged(arch, tmp_path):
    from boxmot_b200.synthetic import make_mobilenetv2_state, make_osnet_state
    from boxmot_b200.weights import export_blob

    seed = {"osnet_x0_25": 21, "osnet_x1_0": 22, "mobilenetv2_x1_4": 23}[arch]
    sd = make_mobilenetv2_state(1.4, seed=seed) if arch.startswith("mobilenet") else make_osnet_state(arch, seed=seed)
    blob = export_blob(sd, tmp_path / f"{arch}.b200reid")
    assert hashlib.sha256(blob.read_bytes()).hexdigest() == BLOB_SHA256[arch]
