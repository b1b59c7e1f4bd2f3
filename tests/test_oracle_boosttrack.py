"""The BoostTrack oracle (tests/boosttrack_oracle.py) against the goldens of the unmodified reference class
(tests/golden/make_boosttrack_golden.py): rows and Kalman snapshots, every case."""
import numpy as np
import pytest

from tests.boosttrack_cases import CASES
from tests.boosttrack_oracle import BoostTrackOracle
from tests.common import assert_rows_match, load_golden


class _Model:   # with_reid is effective only with a model; embeddings are supplied, so it is never called
    def get_features(self, xyxys, img):
        raise AssertionError("embeddings are supplied")


def run_oracle(name, frames=None):
    kwargs, make_frames, make_embs, make_warps = CASES[name]
    kw = {k: v for k, v in kwargs.items() if k not in ("use_cmc", "cmc_method", "adaptive_kf")}
    frames = make_frames() if frames is None else frames
    embs = make_embs(frames) if make_embs else None
    warps = make_warps() if make_warps else None
    o = BoostTrackOracle(reid_model=_Model() if kw.get("with_reid") else None, **kw)
    for f, d in enumerate(frames):
        yield f + 1, o.update(d.copy(), None, None if embs is None else embs[f], None if warps is None else warps[f]), o


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_reproduces_the_reference_boosttrack(name):
    want, snaps = load_golden(name)
    assert sum(len(w) for w in want) > 100
    for f, rows, o in run_oracle(name):
        assert_rows_match(rows, want[f - 1], f, exact_boxes=True)
        if f in snaps:
            ids, mean, cov = snaps[f]
            st = o.state_snapshot()
            assert [t.id for t in o.tracks] == ids.tolist(), f"frame {f}: track list"
            for i, tid in enumerate(ids):
                np.testing.assert_array_equal(st[int(tid)][0], mean[i])
                np.testing.assert_array_equal(st[int(tid)][1], cov[i])
