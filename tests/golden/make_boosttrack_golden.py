"""Golden vectors for BoostTrack / BoostTrack++ from the UNMODIFIED reference class
(boxmot/trackers/bbox/boosttrack/boosttrack.py), file format of make_ocsort_golden.py (rows per frame, snapshots of the
live tracks' ids, 8-state means and covariances at a few frames), plus tests/golden/boosttrack_contract.json: the
constructor's parameter names / defaults and the `default:` values of configs/trackers/boosttrack.yaml.
    python tests/golden/make_boosttrack_golden.py"""
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

from tests.boosttrack_cases import CASES, SNAP_FRAMES  # noqa: E402


class StubReID:
    """with_reid needs a model in the reference; embeddings are always supplied, so it is never called."""

    def get_features(self, xyxys, img):
        raise AssertionError("embeddings are supplied")


class GivenWarps:
    """Camera-motion estimator stand-in: the seeded warp of each frame."""

    def __init__(self, warps):
        self.warps, self.i = warps, 0

    def apply(self, img, dets):
        w = self.warps[self.i]
        self.i += 1
        return w


def walk(node, acc):
    """Every `<param>: {default: ...}` entry of a reference tracker YAML, nested conditional parameters included."""
    if isinstance(node, dict):
        for k, v in node.items():
            if isinstance(v, dict) and "default" in v:
                acc[str(k)] = v["default"]
            walk(v, acc)
    elif isinstance(node, list):
        for v in node:
            walk(v, acc)
    return acc


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
    return dict(rows=np.concatenate(rows, 0), offsets=np.asarray(offsets, np.int64), **snaps)


def make_case(name):
    kwargs, make_frames, make_embs, make_warps = CASES[name]
    bt.KalmanBoxTracker.count = 0
    kw = dict(kwargs, use_cmc=False)
    kw.pop("cmc_method", None)
    frames = make_frames()
    embs = make_embs(frames) if make_embs else None
    trk = bt.BoostTrack(reid_model=StubReID() if kw.get("with_reid") else None, **kw)
    if make_warps:
        trk.cmc = GivenWarps(make_warps())
    return run(trk, frames, np.zeros((360, 640, 3), np.uint8), embs)


def contract():
    ctor = {}
    for n, p in inspect.signature(bt.BoostTrack.__init__).parameters.items():
        if n != "self" and p.kind not in (p.VAR_KEYWORD, p.VAR_POSITIONAL):
            ctor[n] = None if p.default is inspect._empty else p.default
    y = walk(yaml.safe_load((REFERENCE_ROOT / "boxmot" / "configs" / "trackers" / "boosttrack.yaml").read_text()), {})
    return {"ctor": ctor, "yaml": y, "per_class_noise_registry": len(bt.KalmanFilterXYHR().cov_update_policy._per_class_noise)}


if __name__ == "__main__":
    (HERE / "boosttrack_contract.json").write_text(json.dumps(contract(), indent=1, sort_keys=True) + "\n")
    for name in (sys.argv[1:] or CASES):
        out = make_case(name)
        np.savez_compressed(HERE / f"{name}.npz", **out)
        print(name, out["rows"].shape)
