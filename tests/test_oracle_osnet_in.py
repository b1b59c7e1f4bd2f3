"""OSNet-AIN / OSNet-IBN on the host: the functional oracle (oracle/osnet_in.py) against the reference classes'
embeddings, the arch-4 blob (weights.fold_osnet_in) walked by tests/blobsim_osnet_in.py against the oracle at every tap,
export of the reference classes' own state dicts, checkpoint round trip, and refusal of near-miss state dicts."""
import numpy as np
import pytest
import torch

from oracle import osnet_in as oin
from tests.common import GOLDEN

GOLDEN_MODELS = ("osnet_ain_x1_0", "osnet_ain_x0_25", "osnet_ibn_x1_0")


def _state(name, seed, **kw):
    from boxmot_b200.synthetic import make_osnet_ain_state, make_osnet_ibn_state

    return make_osnet_ibn_state(seed=seed, **kw) if name == "osnet_ibn_x1_0" else make_osnet_ain_state(name, seed, **kw)


@pytest.mark.parametrize("mode", ["resize", "resize_pad"])
@pytest.mark.parametrize("name", GOLDEN_MODELS)
def test_osnet_in_oracle_matches_reference_class(name, mode):
    z = np.load(GOLDEN / "reid_osnet_in_reference.npz")
    img = np.random.default_rng(int(z["image_seed"])).integers(0, 255, size=(540, 960, 3), dtype=np.uint8)
    sd = _state(name, int(z[f"weight_seed_{name}"]), num_classes=int(z["num_classes"]))
    feats = oin.get_features(sd, z["boxes"], img, mode)
    assert feats.shape == (len(z["boxes"]), 512)
    np.testing.assert_allclose(feats, z[f"{name}_{mode}"], rtol=0, atol=2e-6)
    assert abs(np.linalg.norm(feats, axis=1) - 1).max() < 1e-6


@pytest.mark.parametrize("name", ["osnet_ain_x1_0", "osnet_ain_x0_75", "osnet_ain_x0_25", "osnet_ibn_x1_0"])
def test_osnet_in_folded_blob_equals_oracle(name, tmp_path):
    """Both IN placements, and x0_75 whose mid channels (48, 72, 96) are not all multiples of 16."""
    from boxmot_b200.weights import ARCH_OSNET_IN, export_blob, read_blob
    from tests.blobsim_osnet_in import blob_forward_osnet_in

    sd = _state(name, 3)
    blob = export_blob(sd, tmp_path / f"{name}.b200reid")
    header, _ = read_blob(blob)
    assert header[2] == ARCH_OSNET_IN and header[7] == 512 and header[9] == 1
    want_modes = (1, 1, 0, 1, 1, 0) if "ain" in name else (2, 2, 0, 0, 0, 0)
    assert tuple(header[10:16]) == want_modes
    x = torch.randn(2, 3, 256, 128)
    x[1] = x[1, :, :1, :1]   # a constant crop, like the blank crop of a box outside the frame
    want, st_w = oin.osnet_in_forward(sd, x, return_stages=True)
    got, st_g = blob_forward_osnet_in(blob, x.permute(0, 2, 3, 1).contiguous(), return_stages=True)
    assert sorted(st_g) == sorted(st_w)
    for k in st_w:
        w = st_w[k].permute(0, 2, 3, 1).numpy()
        assert np.abs(st_g[k].numpy() - w).max() < 2e-5 * max(1.0, float(np.abs(w).max())), k
    scale = float(want.abs().max())
    assert float((got - want).abs().max()) < 2e-6 * max(scale, 1.0)


def test_osnet_in_pt_roundtrip(tmp_path):
    from boxmot_b200.weights import export_blob, read_blob

    sd = _state("osnet_ain_x1_0", 4)
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, tmp_path / "osnet_ain_x1_0_msmt17.pt")
    blob = export_blob(tmp_path / "osnet_ain_x1_0_msmt17.pt")
    header, payload = read_blob(blob)
    assert header[2] == 4 and header[3:8] == (64, 256, 384, 512, 512) and payload.size == header[8]
    assert blob.read_bytes() == export_blob(sd, tmp_path / "direct.b200reid").read_bytes()


def test_near_miss_state_dicts_are_refused(tmp_path):
    from boxmot_b200.synthetic import make_osnet_state
    from boxmot_b200.weights import export_blob

    ain = _state("osnet_ain_x0_5", 1)
    ain.pop("conv3.1.IN.bias")
    with pytest.raises(ValueError, match="missing keys.*conv3.1.IN.bias"):
        export_blob(ain, tmp_path / "a.b200reid")
    ibn = _state("osnet_ibn_x1_0", 1)
    ibn.pop("conv2.1.IN.weight")
    with pytest.raises(ValueError, match="conv2.1.IN.weight"):
        export_blob(ibn, tmp_path / "b.b200reid")
    for arch, where in (("osnet_x1_0", "conv3.0"), ("osnet_x0_25", "conv2.0")):
        odd = make_osnet_state(arch, seed=2)   # an instance norm where neither network has one
        odd[f"{where}.IN.weight"], odd[f"{where}.IN.bias"] = torch.ones(4), torch.zeros(4)
        with pytest.raises(ValueError, match="unexpected keys"):
            export_blob(odd, tmp_path / "c.b200reid")
    ibn_narrow = make_osnet_state("osnet_x0_5", seed=2)   # osnet_ibn exists at x1_0 only
    for j in range(2):
        ibn_narrow[f"conv2.{j}.IN.weight"], ibn_narrow[f"conv2.{j}.IN.bias"] = torch.ones(128), torch.zeros(128)
    with pytest.raises(ValueError):
        export_blob(ibn_narrow, tmp_path / "d.b200reid")


@pytest.mark.parametrize("name", ["osnet_ain_x1_0", "osnet_ain_x0_75", "osnet_ain_x0_5", "osnet_ain_x0_25",
                                  "osnet_ibn_x1_0"])
def test_reference_class_state_dicts_export(name, tmp_path):
    """The reference classes' own state dicts (built without downloads) export, and their keys are the synthetic
    makers' exactly."""
    refharness = pytest.importorskip("tests.golden.refharness")
    if not refharness.reference_available():
        pytest.skip("reference tree not present")
    refharness.install_reference()
    from boxmot.reid.backbones import osnet, osnet_ain

    from boxmot_b200.weights import export_blob, read_blob

    mod = osnet if name == "osnet_ibn_x1_0" else osnet_ain
    sd = getattr(mod, name)(num_classes=10, pretrained=False).state_dict()
    assert set(sd) == set(_state(name, 0, num_classes=10))
    header, _ = read_blob(export_blob(sd, tmp_path / f"{name}.b200reid"))
    assert header[2] == 4
