"""CLIP-ReID ViT-B/16 on the host: the functional oracle (oracle/clip.py) against the reference's embeddings (market- and
veri-shaped checkpoints loaded by the reference's own loader), crop staging at 256x128 and 256x256 against the
reference's crops, the arch-6 blob (weights.fold_clip) walked in float64 against the oracle, checkpoint round trip,
the refusals, and the property of the synthetic weights that makes the tests meaningful (non-uniform attention)."""
import hashlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import clip as oc
from tests.common import GOLDEN

CASES = ("market", "veri")


def _golden():
    z = np.load(GOLDEN / "reid_clip_reference.npz")
    img = np.random.default_rng(int(z["image_seed"])).integers(0, 255, size=(540, 960, 3), dtype=np.uint8)
    return z, img


def _case_state(z, case):
    from boxmot_b200.synthetic import make_clip_state

    return make_clip_state(int(z[f"{case}_seed"]), vehicle=bool(z[f"{case}_vehicle"]), num_classes=int(z["num_classes"]))


@pytest.mark.parametrize("mode", ["resize", "resize_pad"])
@pytest.mark.parametrize("case", CASES)
def test_clip_crops_match_reference_golden(case, mode):
    z, img = _golden()
    hw = (256, 256) if bool(z[f"{case}_vehicle"]) else (256, 128)
    crops = oc.get_crops(z["boxes"], img, mode, hw).numpy()
    assert crops.shape == (len(z["boxes"]), 3, *hw)
    assert hashlib.sha256(np.ascontiguousarray(crops).tobytes()).hexdigest() == str(z[f"{case}_crops_sha256_{mode}"])


@pytest.mark.parametrize("mode", ["resize", "resize_pad"])
@pytest.mark.parametrize("case", CASES)
def test_clip_oracle_matches_reference(case, mode):
    """The reference runs in float32, the oracle in float64: on these weights the two differ by at most 5.3e-7 on
    L2-normalised rows whose largest entry is about 0.16, so 2e-6 leaves a margin of four."""
    z, img = _golden()
    feats = oc.get_features(_case_state(z, case), z["boxes"], img, mode)
    assert feats.shape == (len(z["boxes"]), 1280)
    np.testing.assert_allclose(feats, z[f"{case}_features_{mode}"], rtol=0, atol=2e-6)


def blob_forward_clip(blob, x):
    """Float64 walk of an arch-6 blob (the order csrc/reid_model.cu reads it) on NCHW x: the un-normalised 1280-d row."""
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

    d, layers, heads = header[3], header[4], header[5]
    gh, gw = header[11], header[12]
    T = 1 + gh * gw
    x = x.double().permute(0, 2, 3, 1)   # NHWC
    n = x.shape[0]
    patches = x.reshape(n, gh, 16, gw, 16, 3).permute(0, 1, 3, 2, 4, 5).reshape(n, gh * gw, 768)
    w, b = take(768, d), take(d)
    tok = torch.cat([torch.zeros(n, 1, d, dtype=torch.float64), patches @ w + b], 1) + take(T, d)

    def ln(t, g, beta):
        return F.layer_norm(t, (d,), g, beta, eps=1e-5)

    h = ln(tok, take(d), take(d))
    for _ in range(layers):
        y = ln(h, take(d), take(d))
        qkv = y @ take(d, 3 * d) + take(3 * d)
        q, k, v = (z.reshape(n, T, heads, 64).transpose(1, 2) for z in qkv.split(d, -1))
        a = (torch.softmax(q @ k.transpose(-1, -2), -1) @ v).transpose(1, 2).reshape(n, T, d)   # q pre-scaled
        h = h + a @ take(d, d) + take(d)
        y = ln(h, take(d), take(d))
        m = y @ take(d, 4 * d) + take(4 * d)
        h = h + (m * torch.sigmoid(1.702 * m)) @ take(4 * d, d) + take(d)
    xh = F.layer_norm(h[:, 0], (d,), eps=1e-5)
    g, beta, wp, bp = take(d), take(d), take(d, 512), take(512)
    assert o == payload.size
    return torch.cat([xh * g + beta, xh @ wp + bp], 1)


@pytest.mark.parametrize("case", CASES)
def test_clip_folded_blob_equals_oracle(tmp_path, case):
    from boxmot_b200.weights import ARCH_CLIP, export_blob, read_blob

    z, _ = _golden()
    sd = _case_state(z, case)
    vehicle = bool(z[f"{case}_vehicle"])
    blob = export_blob(sd, tmp_path / f"{case}.b200reid")
    header, _ = read_blob(blob)
    assert header[2] == ARCH_CLIP and header[3:8] == (768, 12, 12, 512, 1280)
    assert header[9:13] == ((256, 256, 16, 16) if vehicle else (256, 128, 16, 8))
    x = torch.randn(2, 3, 256, 256 if vehicle else 128, generator=torch.Generator().manual_seed(1))
    want = oc.clip_forward(oc.double_state(sd), x.double())
    got = blob_forward_clip(blob, x)
    assert float((got - want).abs().max()) < 1e-5 * max(1.0, float(want.abs().max()))   # float32 weights


def test_clip_checkpoint_roundtrip(tmp_path):
    """A CLIP-ReID checkpoint as released (`state_dict`, `module.` prefixes, classifier and prompt / text keys): the
    keys the reference discards are ignored; the blob equals the one of build_transformer's own state."""
    from boxmot_b200.synthetic import make_clip_state
    from boxmot_b200.weights import export_blob, read_blob

    sd = make_clip_state(4)
    pt = tmp_path / "clip_market1501.pt"
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}}, pt)
    blob = export_blob(pt)
    bare = {k: v for k, v in sd.items()
            if not k.startswith(("classifier", "prompt_learner.", "text_encoder.")) and "num_batches" not in k}
    plain = export_blob(bare, tmp_path / "bare.b200reid")
    assert blob.read_bytes() == plain.read_bytes()
    header, payload = read_blob(blob)
    assert header[7] == 1280 and payload.size == header[8]


def test_clip_variants_are_refused(tmp_path):
    from boxmot_b200.synthetic import make_clip_state
    from boxmot_b200.weights import export_blob

    sd = make_clip_state(1, extras=False)
    missing = dict(sd)
    missing.pop("image_encoder.transformer.resblocks.3.ln_2.bias")
    with pytest.raises(ValueError, match="resblocks.3.ln_2.bias"):
        export_blob(missing, tmp_path / "missing.b200reid")
    deeper = dict(sd)   # a 13th block
    for k in [k for k in sd if ".resblocks.11." in k]:
        deeper[k.replace(".resblocks.11.", ".resblocks.12.")] = sd[k]
    with pytest.raises(ValueError, match="resblocks.12"):
        export_blob(deeper, tmp_path / "deeper.b200reid")
    wider = dict(sd)   # ViT-L/14-like width on the class embedding
    wider["image_encoder.class_embedding"] = torch.zeros(1024)
    with pytest.raises(ValueError, match="class_embedding"):
        export_blob(wider, tmp_path / "wider.b200reid")
    rn50 = {k: v for k, v in sd.items() if not k.startswith("image_encoder.transformer.")}   # CLIP-RN50's visual
    rn50["image_encoder.attnpool.positional_embedding"] = torch.zeros(129, 2048)
    with pytest.raises(ValueError, match="attnpool"):
        export_blob(rn50, tmp_path / "rn50.b200reid")


@pytest.mark.parametrize("fname, vehicle", [("clip_veri.pt", False), ("clip_vehicleid.pt", False),
                                            ("clip_market1501.pt", True), ("clip_duke.pt", True)])
def test_clip_file_name_must_match_the_grid(tmp_path, fname, vehicle):
    """The reference picks the crop size from the file name and would silently discard a positional table of the other
    size (running with a random one): refuse instead."""
    from boxmot_b200.synthetic import make_clip_state
    from boxmot_b200.weights import export_blob

    pt = tmp_path / fname
    torch.save(make_clip_state(2, vehicle=vehicle), pt)
    with pytest.raises(ValueError, match="positional table"):
        export_blob(pt)


@pytest.mark.parametrize("vehicle", [False, True])
def test_synthetic_clip_attention_is_not_uniform(vehicle):
    """Uniform attention (every probability 1/T) would make the attention kernel's softmax and P.V untestable: the
    synthetic in_proj puts the largest probability of every row well above 1/T."""
    from boxmot_b200.synthetic import make_clip_state

    sd = oc.double_state(make_clip_state(3, vehicle=vehicle))
    x = torch.rand(2, 3, 256, 256 if vehicle else 128, generator=torch.Generator().manual_seed(2)).double() * 2 - 1
    T = 257 if vehicle else 129
    for block in (0, 11):
        rm = oc.attention_row_max(sd, x, block)
        assert float(rm.mean()) > 10.0 / T and float(rm.min()) > 3.0 / T
