"""Host-side contract of `BoostTrack` / `create_tracker("boosttrack")` (no GPU): constructor names and defaults and the
YAML defaults against tests/golden/boosttrack_contract.json (dumped from the unmodified reference by
tests/golden/make_boosttrack_golden.py), argument resolution through a stub engine, and the out-of-scope options."""
import inspect
import json
import warnings
from pathlib import Path

import numpy as np
import pytest

import boxmot_b200 as bb
import boxmot_b200.trackers as T

GOLDEN = json.loads((Path(__file__).parent / "golden" / "boosttrack_contract.json").read_text())


def test_constructor_names_and_defaults_match_the_reference():
    mine = {n: p.default for n, p in inspect.signature(bb.BoostTrack.__init__).parameters.items()}
    for name, value in GOLDEN["ctor"].items():
        assert name in mine, f"BoostTrack.{name} missing"
        assert mine[name] == value, f"BoostTrack.{name}: {mine[name]} != {value}"
    assert set(T.BOOSTTRACK_ENGINE_DEFAULTS) - {"det_thresh", "max_age", "min_hits", "iou_threshold"} <= set(GOLDEN["ctor"])


def test_yaml_defaults_match_the_reference_yaml():
    assert T.BOOSTTRACK_YAML_DEFAULTS == GOLDEN["yaml"]
    assert GOLDEN["per_class_noise_registry"] == 0 and bb.BoostTrack.per_class_noise == {}
    # the other trackers' table is unchanged
    assert set(T.TRACKER_DEFAULTS) == {"bytetrack", "botsort", "deepocsort", "strongsort", "ocsort"}


def test_create_tracker_resolution_with_a_stub_engine(monkeypatch):
    made = []

    class Engine:
        def __init__(self, kind, n_streams, cap_tracks, cap_dets, feat_dim, reid_blob=None, **params):
            self.kind, self.params, self.feat_dim = kind, params, feat_dim
            self.with_reid, self.has_reid_model = bool(params.get("with_reid")), reid_blob is not None
            self.cmc = None
            made.append((kind, cap_tracks, cap_dets, feat_dim, reid_blob, params))

        def set_cmc(self, method):
            self.cmc = method

    loaded = []

    class StubReID:
        def __init__(self, weights, device=None, half=False, preprocess=None):
            loaded.append(weights)
            self.blob_path, self.feature_dim = "/tmp/osnet.b200reid", 512

    import boxmot_b200.reid as R

    monkeypatch.setattr(T, "MultiStreamTracker", Engine)
    monkeypatch.setattr(R, "B200ReID", StubReID)
    with warnings.catch_warnings():
        warnings.simplefilter("error")   # no "CMC forced off" warning for this kind
        t = T.create_tracker("boosttrack", None, "osnet_x0_25_msmt17.pt", "cuda:0", False, False)
    kind, ct, cd, fd, blob, params = made[-1]
    assert kind == "boosttrack" and blob == "/tmp/osnet.b200reid" and loaded == ["osnet_x0_25_msmt17.pt"]
    assert isinstance(t, bb.BoostTrack) and t._engine.cmc == "ecc" and t.provides_reid
    assert params["det_thresh"] == 0.6 and params["max_age"] == 60 and params["with_reid"] is True
    assert params["use_rich_s"] and params["use_sb"] and params["use_vt"]
    # without weights there is no model, so ReID is off as in the reference
    t = T.create_tracker("boosttrack", evolve_param_dict={"use_cmc": True, "cmc_method": "sof", "with_reid": True})
    assert made[-1][5]["with_reid"] is False and t._engine.cmc == "sof"
    t = T.create_tracker("boosttrack", overrides=None, use_cmc=False, det_thresh=0.4)
    assert made[-1][5]["det_thresh"] == 0.4 and t._engine.cmc is None
    # a foreign backend is called on every row
    calls = []

    class Foreign:
        def get_features(self, xyxys, img):
            calls.append(len(xyxys))
            return np.ones((len(xyxys), 512), np.float32)

    t = T.create_tracker("boosttrack", reid_model=Foreign(), use_cmc=False)
    assert made[-1][5]["with_reid"] is True and made[-1][4] is None
    with pytest.raises(ValueError, match="Unknown tracker type"):
        T.create_tracker("hybridsort")


def test_out_of_scope_options_raise():
    with pytest.raises(NotImplementedError, match="adaptive_kf"):
        bb.BoostTrack(adaptive_kf=True)
    with pytest.raises(NotImplementedError, match="OBB"):
        bb.BoostTrack(is_obb=True)
    with pytest.raises(NotImplementedError, match="per_class"):
        bb.BoostTrack(per_class=True)
    with pytest.raises(NotImplementedError, match="cmc_method='orb'"):
        bb.BoostTrack(cmc_method="orb")
    bb.BoostTrack.per_class_noise[0] = {"r_diag": [1.0, 1.0, 10.0, 0.01]}
    try:
        with pytest.raises(NotImplementedError, match="per-class noise"):
            bb.BoostTrack()
    finally:
        bb.BoostTrack.per_class_noise.clear()
