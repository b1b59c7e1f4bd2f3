"""The SFSORT oracle (tests/sfsort_oracle.py) reproduces every golden of the unmodified reference class bit for bit --
rows, active ids, lost ids and lost states per frame -- and the cases reach every branch of the update."""
import numpy as np
import pytest

from tests import sfsort_oracle as so
from tests.sfsort_cases import CASES

_HITS = {}


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_golden(name):
    kwargs, make_frames, hw = CASES[name]
    rows, act, lost, lstate, ghw = so.load_case(name)
    assert ghw == hw
    o = so.make(**kwargs)
    for f, d in enumerate(make_frames()):
        out = o.update(d, hw)
        assert np.array_equal(out, rows[f]), f"frame {f}"
        assert o.active_ids() == act[f].tolist(), f"frame {f}"
        assert o.lost_ids() == lost[f].tolist(), f"frame {f}"
        assert o.lost_states() == lstate[f].tolist(), f"frame {f}"
    for k, v in o.hits.items():
        _HITS[k] = _HITS.get(k, 0) + v


def test_cases_reach_every_branch():
    if len(_HITS) == 0:
        for name in CASES:
            test_oracle_matches_golden(name)
    for k in ("birth", "match_pass2", "reacquire_pass1", "reacquire_pass2", "lost_central", "lost_marginal",
              "purge_central", "purge_marginal", "all_to_lost", "vanish", "pass2_skipped", "score_at_hth"):
        assert _HITS.get(k, 0) > 0, k
