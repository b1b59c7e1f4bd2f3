"""boxmot_b200/csrc/sf_core.cuh compiled for the host (tests/sfsim.py) reproduces every SFSORT golden: rows, active ids,
lost ids and lost states per frame (the duplicate-box case pins lapjv's order on tied costs)."""
import ctypes

import numpy as np
import pytest

from tests import sfsort_oracle as so
from tests.sfsort_cases import CASES
from tests.sfsim import SfSimTracker, make_cfg


@pytest.mark.parametrize("name", sorted(CASES))
def test_host_core_matches_golden(name):
    kwargs, make_frames, hw = CASES[name]
    rows, act, lost, lstate, _ = so.load_case(name)
    t = SfSimTracker(make_cfg(so.resolve(**kwargs)))
    for f, d in enumerate(make_frames()):
        out = t.update(d, hw)
        assert np.array_equal(out, rows[f]), f"frame {f}"
        assert t.ids(0) == act[f].tolist(), f"frame {f}"
        assert t.ids(1) == lost[f].tolist(), f"frame {f}"
        assert t.ids(2) == lstate[f].tolist(), f"frame {f}"


def test_host_core_capacity_error_is_sticky():
    t = SfSimTracker(make_cfg(so.resolve(), cap_tracks=8, cap_dets=32))
    dets = np.array([[10 * k, 10, 10 * k + 8, 30, 0.9, 0] for k in range(12)], np.float32)
    with pytest.raises(RuntimeError, match="error 1"):
        t.update(dets, (360, 640))
    with pytest.raises(RuntimeError, match="error 1"):
        t.update(dets[:2], (360, 640))


def test_density_table_equals_numpy_log10():
    """The thresholds read log10(count) from a table; the reference calls np.log10(count) on a python int.  The table
    the Python layer hands the engine equals those calls for every count up to 8192 detections per frame, and the host
    core reads that table.  The libm table of C ABI handles is documented to differ in the last bit for some counts."""
    from boxmot_b200.trackers import sfsort_log10_table

    want = np.array([np.log10(k) for k in range(1, 8193)], dtype=np.float64)
    assert np.array_equal(sfsort_log10_table(8193)[1:], want)
    cfg = make_cfg(so.resolve(dynamic_tuning=True), cap_tracks=8, cap_dets=8)
    assert np.array_equal(np.ctypeslib.as_array(ctypes.cast(cfg.log10_tab, ctypes.POINTER(ctypes.c_double)), (9,))[1:],
                          want[:8])
