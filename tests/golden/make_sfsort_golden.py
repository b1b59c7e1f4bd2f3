"""Golden vectors for SFSORT from the UNMODIFIED reference class (boxmot/trackers/bbox/sfsort/sfsort.py): per frame the
output rows, the ids of `active_tracks` and of `lost_tracks` in list order and the lost tracks' states, plus
tests/golden/sfsort_contract.json: constructor-resolved attributes for several argument sets, the `default:` values of
configs/trackers/sfsort.yaml, and `BoxMOTSFSORTConfig` as boxmot/native/trackers/sfsort.py binds it.
    python tests/golden/make_sfsort_golden.py"""
import ctypes
import json
import sys
from pathlib import Path

import numpy as np
import yaml

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parents[1]))
from tests.golden.refharness import REFERENCE_ROOT, install_reference  # noqa: E402

install_reference()
from boxmot.native.trackers import sfsort as native_sf  # noqa: E402
from boxmot.trackers.bbox.sfsort.sfsort import SFSORT  # noqa: E402

from tests.golden.make_boosttrack_golden import walk  # noqa: E402
from tests.sfsort_cases import CASES  # noqa: E402

ATTRS = ("high_th", "match_th_first", "new_track_th", "low_th", "match_th_second", "dynamic_tuning", "cth", "high_th_m",
         "new_track_th_m", "match_th_first_m", "marginal_timeout", "central_timeout", "det_thresh", "l_margin",
         "r_margin", "t_margin", "b_margin")
CLAMP_ARGS = [
    {},
    dict(match_th_first=0.9, new_track_th=0.5, low_th=0.8, cth=0.05),
    dict(high_th=0.3, new_track_th=0.2, low_th=0.4, cth=0.35, marginal_timeout=900, central_timeout=-3),
    dict(dynamic_tuning=True),
    dict(dynamic_tuning=True, high_th_m=0.5, new_track_th_m=0.01, match_th_first_m=0.05),
    dict(high_th=None, match_th_first=None, new_track_th=None, low_th=None, match_th_second=None, cth=None),
    dict(frame_width=640, frame_height=480, horizontal_margin=50, vertical_margin=700),
    dict(high_th=1.5, match_th_second=-0.2, high_th_m=0.3),
]


def run(tracker, frames, hw):
    img = np.zeros((hw[0], hw[1], 3), np.uint8)
    rows, act, lost, lstate = [], [], [], []
    off = {"offsets": [0], "act_off": [0], "lost_off": [0]}
    for dets in frames:
        out = np.asarray(tracker.update(dets.copy(), img))
        out = out.reshape(-1, 8) if out.size else np.empty((0, 8))
        rows.append(out.astype(np.float32))
        act += [t.id for t in tracker.active_tracks]
        lost += [t.id for t in tracker.lost_tracks]
        lstate += [t.state for t in tracker.lost_tracks]
        off["offsets"].append(off["offsets"][-1] + len(out))
        off["act_off"].append(len(act))
        off["lost_off"].append(len(lost))
    return dict(rows=np.concatenate(rows, 0), active=np.asarray(act, np.int64), lost=np.asarray(lost, np.int64),
                lost_state=np.asarray(lstate, np.int64), hw=np.asarray(hw, np.int64),
                **{k: np.asarray(v, np.int64) for k, v in off.items()})


def make_case(name):
    kwargs, make_frames, hw = CASES[name]
    return run(SFSORT(**kwargs), make_frames(), hw)


def contract():
    resolved = []
    for args in CLAMP_ARGS:
        t = SFSORT(**args)
        resolved.append({"args": args, "resolved": {a: getattr(t, a) for a in ATTRS}})
    y = walk(yaml.safe_load((REFERENCE_ROOT / "boxmot" / "configs" / "trackers" / "sfsort.yaml").read_text()), {})
    ctypes_names = {ctypes.c_float: "float", ctypes.c_int: "int"}
    fields = [[n, ctypes_names[t]] for n, t in native_sf._SFSORTCConfig._fields_]
    return {"resolved": resolved, "yaml": y, "BoxMOTSFSORTConfig": fields,
            "sizeof_BoxMOTSFSORTConfig": ctypes.sizeof(native_sf._SFSORTCConfig)}


if __name__ == "__main__":
    (HERE / "sfsort_contract.json").write_text(json.dumps(contract(), indent=1, sort_keys=True) + "\n")
    for name in (sys.argv[1:] or CASES):
        out = make_case(name)
        np.savez_compressed(HERE / f"{name}.npz", **out)
        print(name, out["rows"].shape, out["lost"].shape)
