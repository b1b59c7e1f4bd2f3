"""The OccluBoost oracle (tests/occluboost_oracle.py) against the goldens of the unmodified reference class
(tests/golden/make_occluboost_golden.py): rows, snapshots and flush_gta() rows of every case, and every branch of the
update reached by the case table."""
from collections import Counter

import numpy as np
import pytest

from tests.common import GOLDEN, assert_rows_match, load_golden
from tests.occluboost_cases import CASES
from tests.occluboost_oracle import OccluBoostOracle


class _Model:   # with_reid is effective only with a model; embeddings are supplied, so it is never called
    def get_features(self, xyxys, img):
        raise AssertionError("embeddings are supplied")


def run_oracle(name):
    kwargs, make_frames, make_embs, make_warps = CASES[name]
    kw = {k: v for k, v in kwargs.items() if k not in ("use_cmc", "cmc_method", "adaptive_kf")}
    frames = make_frames()
    embs = make_embs(frames) if make_embs else None
    warps = make_warps() if make_warps else None
    o = OccluBoostOracle(reid_model=_Model() if kw.get("with_reid") else None, **kw)
    for f, d in enumerate(frames):
        yield f + 1, o.update(d.copy(), None, None if embs is None else embs[f], None if warps is None else warps[f]), o


_COUNTS = {}


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_reproduces_the_reference_occluboost(name):
    want, snaps = load_golden(name)
    z = np.load(GOLDEN / f"{name}.npz")
    assert sum(len(w) for w in want) > 100
    for f, rows, o in run_oracle(name):
        assert_rows_match(rows, want[f - 1], f, exact_boxes=True)
        if f in snaps:
            ids, mean, cov = snaps[f]
            st = o.state_snapshot()
            assert [t.id for t in o.tracks] == ids.tolist(), f"frame {f}: track list"
            assert [t.activated for t in o.tracks] == z[f"snap{f}_act"].tolist(), f"frame {f}: is_activated"
            for i, tid in enumerate(ids):
                np.testing.assert_allclose(st[int(tid)][0], mean[i], rtol=1e-9, atol=1e-9)
                np.testing.assert_allclose(st[int(tid)][1], cov[i], rtol=1e-9, atol=1e-9)
    assert np.array_equal(o.flush_gta(), z["gta"]), "flush_gta rows"
    _COUNTS[name] = Counter(o.counts)


def test_the_cases_reach_every_branch():
    total = Counter()
    for name in CASES:
        if name not in _COUNTS:
            for _ in run_oracle(name):
                pass
            _COUNTS[name] = Counter(_[2].counts)
        total += _COUNTS[name]
    for branch in ("recovery", "second", "gta_recovery", "resurrect", "gap_rows", "ams_damped", "duplicate_drop",
                   "tentative_expired", "updated_twice"):
        assert total[branch] > 0, f"no case reaches {branch}: {dict(total)}"
