"""Host-side contract of `OccluBoost` / `create_tracker("occluboost")` (no GPU): constructor names and defaults and the
YAML defaults against tests/golden/occluboost_contract.json (dumped from the unmodified reference by
tests/golden/make_occluboost_golden.py), argument resolution through a stub engine, the out-of-scope options, and the
gap rows rebuilt from resurrection events."""
import inspect
import json
import warnings
from pathlib import Path

import numpy as np
import pytest

import boxmot_b200 as bb
import boxmot_b200.trackers as T
from tests.occluboost_cases import OCCLUBOOST_YAML

GOLDEN = json.loads((Path(__file__).parent / "golden" / "occluboost_contract.json").read_text())


def test_constructor_names_and_defaults_match_the_reference():
    mine = {n: p.default for n, p in inspect.signature(bb.OccluBoost.__init__).parameters.items()}
    for name, value in GOLDEN["ctor"].items():
        assert name in mine, f"OccluBoost.{name} missing"
        assert mine[name] == value, f"OccluBoost.{name}: {mine[name]} != {value}"
    assert set(T.OCCLUBOOST_ENGINE_DEFAULTS) <= set(GOLDEN["ctor"])
    assert {k: v for k, v in GOLDEN["ctor"].items() if k in T.OCCLUBOOST_ENGINE_DEFAULTS} == T.OCCLUBOOST_ENGINE_DEFAULTS
    # BoostTrack's constructor, which the reference subclass forwards **kwargs to
    assert issubclass(bb.OccluBoost, bb.BoostTrack)


def test_yaml_defaults_match_the_reference_yaml():
    assert T.OCCLUBOOST_YAML_DEFAULTS == GOLDEN["yaml"] == OCCLUBOOST_YAML
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
        warnings.simplefilter("error")   # SOF runs on the device: no "CMC forced off" warning
        t = T.create_tracker("occluboost", None, "osnet_x0_25_msmt17.pt", "cuda:0", False, False)
    kind, ct, cd, fd, blob, params = made[-1]
    assert kind == "occluboost" and blob == "/tmp/osnet.b200reid" and loaded == ["osnet_x0_25_msmt17.pt"]
    assert isinstance(t, bb.OccluBoost) and t._engine.cmc == "sof" and t.provides_reid
    want = {k: v for k, v in T.OCCLUBOOST_YAML_DEFAULTS.items() if k not in ("use_cmc", "cmc_method", "adaptive_kf")}
    assert {k: params[k] for k in want} == want
    # the constructor defaults when built directly: GTA on, ECC
    t = bb.OccluBoost(reid_model=StubReID("w"), with_reid=True)
    assert made[-1][5]["gta_enabled"] is True and made[-1][5]["use_second_pass"] is False and t._engine.cmc == "ecc"
    t = T.create_tracker("occluboost", overrides=None, use_cmc=False, gta_enabled=True)
    assert made[-1][5]["gta_enabled"] is True and t._engine.cmc is None and made[-1][5]["with_reid"] is False
    with pytest.raises(ValueError, match="Unknown tracker type"):
        T.create_tracker("hybridsort")


def test_out_of_scope_options_raise():
    with pytest.raises(NotImplementedError, match="adaptive_kf"):
        bb.OccluBoost(adaptive_kf=True)
    with pytest.raises(NotImplementedError, match="OBB"):
        bb.OccluBoost(is_obb=True)
    with pytest.raises(NotImplementedError, match="per_class"):
        bb.OccluBoost(per_class=True)
    for method in ("orb", "sift"):
        with pytest.raises(NotImplementedError, match=f"cmc_method='{method}'"):
            bb.OccluBoost(cmc_method=method)
    bb.BoostTrack.per_class_noise[0] = {"r_diag": [1.0, 1.0, 10.0, 0.01]}
    try:
        with pytest.raises(NotImplementedError, match="per-class noise"):
            bb.OccluBoost()
    finally:
        bb.BoostTrack.per_class_noise.clear()


def test_gap_rows_from_events():
    ev = np.array([[7, 10, 14, 0, 0, 10, 20, 4, 8, 14, 28, 0.9, 2.0],    # gap 4: 3 rows
                   [8, 20, 21, 0, 0, 1, 1, 0, 0, 1, 1, 0.5, 0.0],        # gap 1: none
                   [9, 1, 80, 0, 0, 1, 1, 0, 0, 1, 1, 0.5, 0.0]])        # beyond max_gap: none
    rows = T.gta_rows(ev, True, 60, 0.0)
    assert rows.shape == (3, 9) and rows[:, 0].tolist() == [11, 12, 13] and (rows[:, 1] == 7).all()
    np.testing.assert_allclose(rows[1, 2:6], [2, 4, 12, 24])
    assert (rows[:, 6] == 0.9).all() and (rows[:, 7] == 2.0).all() and (rows[:, 8] == -1).all()
    assert T.gta_rows(ev, False, 60, 5.0).shape == (0, 9)
    sm = T.gta_rows(ev, True, 60, 5.0)   # smoothed in place of the straight line, same frames / ids
    assert sm.shape == (3, 9) and np.array_equal(sm[:, [0, 1, 6, 7, 8]], rows[:, [0, 1, 6, 7, 8]])
