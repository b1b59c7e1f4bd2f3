"""The BoostTrack device core (boxmot_b200/csrc/bt_core.cuh) compiled for the host (tests/btsim.py) against every
golden of the unmodified reference class: ids, det_ind, cls and conf exact, boxes within the row tolerance, Kalman
snapshots within the DeepOCSORT golden tolerance."""
import numpy as np
import pytest

from tests.boosttrack_cases import CASES
from tests.btsim import BtSimTracker, make_cfg
from tests.common import assert_rows_match, load_golden


def sim_kwargs(kwargs):
    return {k: v for k, v in kwargs.items() if k not in ("use_cmc", "cmc_method", "adaptive_kf")}


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_build_of_the_device_core_matches_the_reference(name):
    kwargs, make_frames, make_embs, make_warps = CASES[name]
    want, snaps = load_golden(name)
    frames = make_frames()
    embs = make_embs(frames) if make_embs else None
    warps = make_warps() if make_warps else None
    trk = BtSimTracker(make_cfg(**sim_kwargs(kwargs)))
    for f, d in enumerate(frames, start=1):
        got = trk.update(d, None if embs is None else embs[f - 1], None if warps is None else warps[f - 1])
        assert_rows_match(got, want[f - 1], f)
        if f in snaps:
            ids, mean, cov = snaps[f]
            gi, gx, gp = trk.snapshot()
            assert gi.tolist() == ids.tolist(), f"frame {f}: track list"
            np.testing.assert_allclose(gx, mean, rtol=1e-9, atol=1e-7, err_msg=f"frame {f}: means")
            np.testing.assert_allclose(gp, cov, rtol=1e-9, atol=1e-7, err_msg=f"frame {f}: covariances")
