"""Golden vectors for OccluBoost from the UNMODIFIED reference class (boxmot/trackers/bbox/occluboost/occluboost.py),
format of make_boosttrack_golden.py (rows per frame; snapshots of the live tracks' ids, 8-state means, covariances and
is_activated at a few frames) plus `gta` (the rows flush_gta() returns at the end), and
tests/golden/occluboost_contract.json: the constructor's parameter names / defaults and the `default:` values of
configs/trackers/occluboost.yaml.
    python tests/golden/make_occluboost_golden.py"""
import inspect
import json
import sys
from pathlib import Path

import numpy as np
import yaml

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parents[1]))
from tests.golden.refharness import REFERENCE_ROOT, install_reference  # noqa: E402

install_reference()
from boxmot.trackers.bbox.boosttrack import boosttrack as bt  # noqa: E402
from boxmot.trackers.bbox.occluboost import occluboost as ob  # noqa: E402

from tests.golden.make_boosttrack_golden import GivenWarps, StubReID, walk  # noqa: E402
from tests.occluboost_cases import CASES, SNAP_FRAMES  # noqa: E402


def run(tracker, frames, img, embs=None):
    rows, offsets, snaps = [], [0], {}
    for f, dets in enumerate(frames):
        e = None if embs is None else embs[f]
        out = np.asarray(tracker.update(dets.copy(), img, e))
        out = out.reshape(-1, 8) if out.size else np.empty((0, 8), np.float32)
        rows.append(out.astype(np.float32))
        offsets.append(offsets[-1] + len(out))
        if (f + 1) in SNAP_FRAMES:
            snaps[f"snap{f + 1}_ids"] = np.asarray([t.id for t in tracker.trackers], dtype=np.int64)
            snaps[f"snap{f + 1}_mean"] = np.asarray([t.kf.x for t in tracker.trackers], dtype=np.float64).reshape(-1, 8)
            snaps[f"snap{f + 1}_cov"] = np.asarray([t.kf.covariance for t in tracker.trackers]).reshape(-1, 8, 8)
            snaps[f"snap{f + 1}_act"] = np.asarray([getattr(t, "is_activated", True) for t in tracker.trackers], bool)
    return dict(rows=np.concatenate(rows, 0), offsets=np.asarray(offsets, np.int64),
                gta=np.asarray(tracker.flush_gta(), np.float64).reshape(-1, 9), **snaps)


def make_case(name):
    kwargs, make_frames, make_embs, make_warps = CASES[name]
    bt.KalmanBoxTracker.count = 0
    kw = dict(kwargs, use_cmc=False)
    kw.pop("cmc_method", None)
    frames = make_frames()
    embs = make_embs(frames) if make_embs else None
    trk = ob.OccluBoost(reid_model=StubReID() if kw.get("with_reid") else None, **kw)
    if make_warps:
        trk.cmc = GivenWarps(make_warps())
    return run(trk, frames, np.zeros((360, 640, 3), np.uint8), embs)


def contract():
    ctor = {}
    for n, p in inspect.signature(ob.OccluBoost.__init__).parameters.items():
        if n != "self" and p.kind not in (p.VAR_KEYWORD, p.VAR_POSITIONAL):
            ctor[n] = None if p.default is inspect._empty else p.default
    y = walk(yaml.safe_load((REFERENCE_ROOT / "boxmot" / "configs" / "trackers" / "occluboost.yaml").read_text()), {})
    return {"ctor": ctor, "yaml": y}


if __name__ == "__main__":
    (HERE / "occluboost_contract.json").write_text(json.dumps(contract(), indent=1, sort_keys=True) + "\n")
    for name in (sys.argv[1:] or CASES):
        out = make_case(name)
        np.savez_compressed(HERE / f"{name}.npz", **out)
        print(name, out["rows"].shape, out["gta"].shape)
