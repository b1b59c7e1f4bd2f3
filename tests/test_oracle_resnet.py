"""ResNet50 / ResNet101 on the host: the functional oracle (oracle/resnet.py) against the reference classes' embeddings
(strict loads and a resnet50_fc512 checkpoint loaded as plain resnet50), crop staging against the reference's crops,
the arch-5 blob (weights.fold_resnet) walked in float64 against the oracle, checkpoint round trip, and refusal of
BasicBlock ResNets, ResNeXt and incomplete state dicts."""
import hashlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import resnet as orn
from oracle.reid import get_crops
from tests.common import GOLDEN

CASES = ("resnet50", "resnet101", "fc512")


def _golden():
    z = np.load(GOLDEN / "reid_resnet_reference.npz")
    img = np.random.default_rng(int(z["image_seed"])).integers(0, 255, size=(540, 960, 3), dtype=np.uint8)
    return z, img


def _case_state(z, case):
    from boxmot_b200.synthetic import make_resnet_state

    return make_resnet_state(int(z[f"{case}_depth"]), seed=int(z[f"{case}_seed"]), with_fc512=bool(z[f"{case}_fc512"]),
                             num_classes=int(z["num_classes"]))


@pytest.mark.parametrize("mode", ["resize", "resize_pad"])
def test_resnet_crops_match_reference_golden(mode):
    z, img = _golden()
    crops = get_crops(z["boxes"], img, mode).numpy()
    assert hashlib.sha256(np.ascontiguousarray(crops).tobytes()).hexdigest() == str(z[f"crops_sha256_{mode}"])


@pytest.mark.parametrize("mode", ["resize", "resize_pad"])
@pytest.mark.parametrize("case", CASES)
def test_resnet_oracle_matches_reference_class(case, mode):
    z, img = _golden()
    feats = orn.get_features(_case_state(z, case), z["boxes"], img, mode)
    assert feats.shape == (len(z["boxes"]), 2048)
    np.testing.assert_allclose(feats, z[f"{case}_features_{mode}"], rtol=0, atol=2e-6)


def blob_forward_resnet(blob, x):
    """Float64 walk of an arch-5 blob (the order csrc/reid_model.cu reads it) on NCHW x: the un-normalised feature."""
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

    def conv(x, w, k, stride, pad):   # w [k*k*ci][co] K-major -> conv2d weight [co][ci][k][k]
        ci = w.shape[0] // (k * k)
        return F.conv2d(x, w.reshape(k, k, ci, -1).permute(3, 2, 0, 1), stride=stride, padding=pad)

    x = x.double()
    x = F.max_pool2d(F.relu(conv(x, take(147, 64), 7, 2, 3) + take(64).view(1, -1, 1, 1)), 3, 2, 1)
    cin = 64
    for li, n_blocks in enumerate(header[3:7]):
        width = 64 << li
        for j in range(n_blocks):
            stride = 2 if (j == 0 and li > 0) else 1
            t = F.relu(conv(x, take(cin, width), 1, 1, 0) + take(width).view(1, -1, 1, 1))
            t = F.relu(conv(t, take(9 * width, width), 3, stride, 1) + take(width).view(1, -1, 1, 1))
            if j == 0:
                w3 = take(width + cin, 4 * width)
                y = conv(t, w3[:width], 1, 1, 0) + conv(x[:, :, ::stride, ::stride], w3[width:], 1, 1, 0)
                x = F.relu(y + take(4 * width).view(1, -1, 1, 1))
            else:
                x = F.relu(conv(t, take(width, 4 * width), 1, 1, 0) + take(4 * width).view(1, -1, 1, 1) + x)
            cin = 4 * width
    assert o == payload.size
    return x.mean(dim=(2, 3))


@pytest.mark.parametrize("case", CASES)
def test_resnet_folded_blob_equals_oracle(tmp_path, case):
    from boxmot_b200.weights import ARCH_RESNET, export_blob, read_blob

    z, _ = _golden()
    sd = _case_state(z, case)
    blob = export_blob(sd, tmp_path / f"{case}.b200reid")
    header, _ = read_blob(blob)
    depth = int(z[f"{case}_depth"])
    assert header[2] == ARCH_RESNET and header[3:8] == (3, 4, 6 if depth == 50 else 23, 3, 2048)
    x = torch.randn(2, 3, 256, 128, generator=torch.Generator().manual_seed(1))
    want = orn.resnet_forward({k: v.double() for k, v in sd.items()}, x.double())
    got = blob_forward_resnet(blob, x)
    assert float((got - want).abs().max()) < 1e-6 * max(1.0, float(want.abs().max()))   # float32 weights


def test_resnet_fc512_checkpoint_roundtrip(tmp_path):
    """A resnet50_fc512 checkpoint as released (`state_dict`, `module.` prefixes): the fc head is ignored, as the
    reference ignores it when it builds plain resnet50 for that file name; the blob equals the one of the bare trunk."""
    from boxmot_b200.synthetic import make_resnet_state
    from boxmot_b200.weights import export_blob, read_blob

    sd = make_resnet_state(50, seed=4, with_fc512=True)
    pt = tmp_path / "resnet50_fc512_market1501.pt"
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, pt)
    blob = export_blob(pt)
    trunk = {k: v for k, v in sd.items() if not k.startswith(("fc.", "classifier."))}
    plain = export_blob(trunk, tmp_path / "trunk.b200reid")
    assert blob.read_bytes() == plain.read_bytes()
    header, payload = read_blob(blob)
    assert header[7] == 2048 and payload.size == header[8]


def test_resnet_variants_are_refused(tmp_path):
    from boxmot_b200.synthetic import make_resnet_state
    from boxmot_b200.weights import export_blob

    sd = make_resnet_state(50, seed=1)
    missing = dict(sd)
    missing.pop("layer2.1.bn2.running_var")
    with pytest.raises(ValueError, match="layer2.1.bn2.running_var"):
        export_blob(missing, tmp_path / "missing.b200reid")
    odd = {k: v for k, v in sd.items() if not k.startswith("layer3.5.")}   # five layer3 blocks: no known depth
    with pytest.raises(ValueError):
        export_blob(odd, tmp_path / "odd.b200reid")


@pytest.mark.parametrize("arch", ["resnet18", "resnet34", "resnext50_32x4d"])
def test_reference_basicblock_and_resnext_state_dicts_are_refused(tmp_path, arch):
    """The reference's own resnet18 / resnet34 (BasicBlock) and resnext50_32x4d (grouped 3x3, resnet50's key names)."""
    refharness = pytest.importorskip("tests.golden.refharness")
    if not refharness.reference_available():
        pytest.skip("reference tree not present")
    refharness.install_reference()
    from boxmot.reid.backbones import resnet as ref_resnet

    from boxmot_b200.weights import export_blob

    m = getattr(ref_resnet, arch)(num_classes=10, pretrained=False)
    with pytest.raises(ValueError, match="not a Bottleneck resnet50"):
        export_blob(m.state_dict(), tmp_path / f"{arch}.b200reid")


def test_reference_resnet_state_dict_keys_match_synthetic():
    refharness = pytest.importorskip("tests.golden.refharness")
    if not refharness.reference_available():
        pytest.skip("reference tree not present")
    refharness.install_reference()
    from boxmot.reid.backbones import resnet as ref_resnet

    from boxmot_b200.synthetic import make_resnet_state

    for depth in (50, 101):
        ref = getattr(ref_resnet, f"resnet{depth}")(num_classes=751, pretrained=False).state_dict()
        syn = make_resnet_state(depth, seed=0)
        assert sorted(ref) == sorted(syn)
        assert all(tuple(ref[k].shape) == tuple(syn[k].shape) for k in ref)

