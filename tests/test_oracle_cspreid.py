"""CSPReID-n on the host: the float64 oracle (tests/cspreid_oracle.py) against the reference class and the reference
golden at 256x128 and 256x256, the folded arch-10 blob walked in float64 against the unfolded oracle, the blob header,
name resolution (the checkpoint's model_name, then the file name; veri / vehicleid -> 256x256 crops), the refusals,
and the golden's regeneration when the reference is installed."""
import hashlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from boxmot_b200.weights import ARCH_CSPREID, cspreid_layout
from tests import cspreid_oracle as oc
from tests import vit_oracle as ov
from tests.common import GOLDEN
from tests.golden.refharness import install_reference, reference_available

FILES = ("cspreid_n_market1501", "cspreid_n_veri")
MODES = ("resize", "resize_pad")


def _save(path, sd, **extra):
    torch.save({"state_dict": {"module." + k: v for k, v in sd.items()}, **extra}, path)


def _golden():
    z = np.load(GOLDEN / "reid_cspreid_reference.npz")
    img = np.random.default_rng(int(z["image_seed"])).integers(0, 255, size=(540, 960, 3), dtype=np.uint8)
    return z, img


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("key", FILES)
def test_cspreid_oracle_matches_reference_golden(key, mode):
    from boxmot_b200.synthetic import make_cspreid_state

    z, img = _golden()
    hw = tuple(int(v) for v in z[f"{key}_input_hw"])
    x = ov.get_crops(z["boxes"], img, mode, hw)
    assert hashlib.sha256(x.numpy().tobytes()).hexdigest() == str(z[f"{key}_crops_sha256_{mode}"])
    sd = oc.double_state(make_cspreid_state(int(z[f"{key}_seed"]), num_classes=int(z["num_classes"])))
    got = oc.embed(sd, x.double()).numpy()
    want = z[f"{key}_features_{mode}"]
    assert np.abs(got - want).max() < 2e-6


@pytest.mark.skipif(not reference_available(), reason="reference not installed")
@pytest.mark.parametrize("hw", [(256, 128), (256, 256)])
def test_cspreid_oracle_matches_reference_class_in_float64(hw):
    install_reference()
    from boxmot.reid.backbones.cspreid_n import CSPReID_n

    from boxmot_b200.synthetic import make_cspreid_state

    sd = make_cspreid_state(7)
    m = CSPReID_n(num_classes=751).eval().double()
    m.load_state_dict(sd, strict=True)
    x = torch.rand(3, 3, *hw, generator=torch.Generator().manual_seed(1), dtype=torch.float64) * 4 - 2
    with torch.no_grad():
        want = m(x)
    taps = oc.forward_taps(oc.double_state(sd), x)
    assert torch.equal(taps[-1], want)
    assert taps[7].shape[2:] == (8, hw[1] // 32)


def _blob_forward(payload, x):
    """Float64 walk of the arch-10 blob (weights.fold_cspreid's layout) on x (n, 3, H, W): the folded network."""
    o = 0
    p = torch.from_numpy(payload.astype(np.float64))

    def take(*shape):
        nonlocal o
        k = int(np.prod(shape))
        t = p[o:o + k].reshape(shape)
        o += (k + 3) // 4 * 4
        return t

    def conv(name, x, stride=1):
        co, ci, k, _ = dict((n, s) for n, _, s in cspreid_layout())[name]
        w = take(k * k * ci, co).reshape(k, k, ci, co).permute(3, 2, 0, 1)
        return F.silu(F.conv2d(x, w, take(co), stride, k // 2))

    def c3k2(s, x, n):
        y = conv(f"stage{s}.0.cv1", x)
        outs = list(y.chunk(2, 1))
        cur = outs[-1]
        for i in range(n):
            b = f"stage{s}.0.bottlenecks.{i}"
            cur = cur + conv(b + ".cv2", conv(b + ".cv1", cur))
            outs.append(cur)
        return conv(f"stage{s}.0.cv2", torch.cat(outs, 1))

    x = conv("stem.1", conv("stem.0", x, 2), 2)
    for s, n in ((1, 1), (2, 1), (3, 2)):
        x = conv(f"stage{s}.1", c3k2(s, x, n), 2)
    x = c3k2(4, x, 1)
    x = conv("stage4.1.cv1", x)
    y1 = F.max_pool2d(x, 3, 1, 1)
    y2 = F.max_pool2d(y1, 3, 1, 1)
    x = conv("stage4.1.cv2", torch.cat([x, y1, y2, F.max_pool2d(y2, 3, 1, 1)], 1))
    w1, w2, dw, db, ws = take(512, 64), take(64, 512), take(9, 512), take(512), take(512)
    x = x * torch.sigmoid(F.silu(x.mean((2, 3)) @ w1) @ w2)[:, :, None, None]
    d = F.silu(F.conv2d(x, dw.T.reshape(512, 1, 3, 3), db, 1, 1, 1, 512))
    x = x * torch.sigmoid((d * ws[None, :, None, None]).sum(1, keepdim=True))
    pools = [x.mean((2, 3)), *F.adaptive_avg_pool2d(x, (2, 1))[:, :, :, 0].unbind(2)]
    rows = torch.stack([v @ take(512, 512) + take(512) for v in pools], 2).flatten(1)
    assert o == payload.size
    return rows


@pytest.mark.parametrize("fname", ["cspreid_n_market1501.pt", "cspreid_n_veri.pt"])
def test_cspreid_folded_blob_equals_oracle(tmp_path, fname):
    from boxmot_b200.synthetic import make_cspreid_state
    from boxmot_b200.weights import export_blob, read_blob

    sd = make_cspreid_state(4)
    pt = tmp_path / fname
    _save(pt, sd)
    header, payload = read_blob(export_blob(pt))
    hw = (256, 256) if "veri" in fname else (256, 128)
    assert header[2] == ARCH_CSPREID and list(header[3:8]) == [128, 256, 384, 512, 1536]
    assert tuple(header[9:11]) == hw and all(v == 0 for v in header[11:16])
    x = torch.rand(2, 3, *hw, generator=torch.Generator().manual_seed(3), dtype=torch.float64) * 4 - 2
    got = _blob_forward(payload, x)
    want = oc.forward_taps(oc.double_state(sd), x)[-1]
    # the blob is float32: folded weights carry 2^-24 relative rounding
    assert (got - want).abs().max() < 1e-4 * want.abs().max()


@pytest.mark.parametrize("fname,hw", [("cspreid_n_market1501.pt", (256, 128)), ("cspreid_n_veri.pt", (256, 256)),
                                      ("cspreid_n_vehicleid.pt", (256, 256)), ("my_cspreid_n_duke.pth", (256, 128))])
def test_cspreid_file_names_resolve_the_crop(tmp_path, fname, hw):
    from boxmot_b200.synthetic import make_cspreid_state
    from boxmot_b200.weights import export_blob, read_blob

    pt = tmp_path / fname
    torch.save(make_cspreid_state(1), pt)   # a bare state dict
    header, _ = read_blob(export_blob(pt))
    assert header[2] == ARCH_CSPREID and tuple(header[9:11]) == hw


def test_cspreid_model_name_and_in_memory_state(tmp_path):
    from boxmot_b200.synthetic import make_cspreid_state
    from boxmot_b200.weights import export_blob, read_blob

    sd = make_cspreid_state(2)
    pt = tmp_path / "weights_veri.pt"   # no model name in the file name: the checkpoint's model_name decides
    _save(pt, sd, model_name="cspreid_n")
    header, _ = read_blob(export_blob(pt))
    assert header[2] == ARCH_CSPREID and tuple(header[9:11]) == (256, 256)
    header, payload = read_blob(export_blob(sd, tmp_path / "mem.b200reid"))
    assert header[2] == ARCH_CSPREID and tuple(header[9:11]) == (256, 128)
    _, from_file = read_blob(export_blob(pt))
    assert np.array_equal(payload, from_file)


def test_cspreid_missing_or_misshaped_tensors_are_refused(tmp_path):
    from boxmot_b200.synthetic import make_cspreid_state
    from boxmot_b200.weights import export_blob

    sd = make_cspreid_state(1)
    missing = dict(sd)
    missing.pop("stage3.0.bottlenecks.1.cv2.bn.running_var")
    with pytest.raises(ValueError, match="stage3.0.bottlenecks.1.cv2.bn.running_var"):
        export_blob(missing, tmp_path / "missing.b200reid")
    pt = tmp_path / "cspreid_n_market1501.pt"
    wide = dict(sd)
    wide["head.bn_part1.reduction.weight"] = torch.zeros(256, 512, 1, 1)   # feat_dim 256
    _save(pt, wide)
    with pytest.raises(ValueError, match="head.bn_part1.reduction.weight"):
        export_blob(pt)


@pytest.mark.parametrize("other", ["lmbn_n", "vit_nano", "osnet_x0_25"])
def test_other_weights_under_a_cspreid_name_are_refused(tmp_path, other):
    from boxmot_b200 import synthetic
    from boxmot_b200.weights import export_blob

    sd = {"lmbn_n": lambda: synthetic.make_lmbn_n_state(0), "vit_nano": lambda: synthetic.make_vit_state("vit_nano", 0),
          "osnet_x0_25": lambda: synthetic.make_osnet_state("osnet_x0_25", 0)}[other]()
    pt = tmp_path / "cspreid_n_market1501.pt"
    _save(pt, sd)
    with pytest.raises(ValueError, match="cspreid_n"):
        export_blob(pt)


@pytest.mark.parametrize("name", ["osnet_x0_25_market1501.pt", "lmbn_n_duke.pt", "vit_nano_market1501.pt"])
def test_cspreid_weights_under_another_model_name_are_refused(tmp_path, name):
    from boxmot_b200.synthetic import make_cspreid_state
    from boxmot_b200.weights import export_blob

    pt = tmp_path / name
    _save(pt, make_cspreid_state(0))
    with pytest.raises(ValueError):
        export_blob(pt)


def test_synthetic_cspreid_bottlenecks_are_not_the_identity():
    """The reference zero-initialises the last BN gamma of every shortcut bottleneck; the synthetic state must not, or
    the residual branches would go untested."""
    from boxmot_b200.synthetic import make_cspreid_state

    sd = make_cspreid_state(0)
    for name, _, _ in cspreid_layout():
        if ".bottlenecks." in name and name.endswith(".cv2"):
            assert float(sd[name + ".bn.weight"].abs().min()) >= 0.5
            assert float(sd[name + ".bn.running_var"].min()) > 0.5


@pytest.mark.skipif(not reference_available(), reason="reference not installed")
def test_cspreid_golden_regenerates_bit_for_bit():
    from tests.golden import make_cspreid_golden

    fresh = make_cspreid_golden.compute()
    z = np.load(GOLDEN / "reid_cspreid_reference.npz")
    assert set(fresh) == set(z.files)
    for k, v in fresh.items():
        assert np.array_equal(np.asarray(v), z[k]), k
