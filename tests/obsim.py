"""Host simulation of the OccluBoost device core (tests only; never a product path).

Builds tests/_obsim/obsim.cpp with g++ (BMB_HOSTSIM: boxmot_b200/csrc/ob_core.cuh compiled for one host "thread") into
a per-user temporary directory and exposes it through ctypes, so `-m "not gpu"` tests can check the device source
against the reference goldens without a GPU.
"""
from __future__ import annotations

import ctypes
import getpass
import hashlib
import os
import subprocess
import tempfile
from pathlib import Path

import numpy as np

from tests.btsim import BtCfg, make_cfg as make_bt_cfg
from tests.occluboost_oracle import OB_DEFAULTS

ROOT = Path(__file__).resolve().parents[1]
SRC = ROOT / "tests" / "_obsim" / "obsim.cpp"
CSRC = ROOT / "boxmot_b200" / "csrc"

c_int, c_double = ctypes.c_int, ctypes.c_double
OB_INTS = ("use_second_pass", "recovery_max_age", "second_pass_max_age", "second_pass_min_hits", "confirm_hits",
           "tentative_max_age", "ams_on", "ams_buffer_size", "gta", "gta_min_track_length", "gta_max_gap")
OB_DOUBLES = ("lambda_emb_mult", "recovery_appearance_thresh", "recovery_iou_thresh", "feat_alpha", "track_low_thresh",
              "second_iou_thresh", "second_appearance_thresh", "new_track_thresh", "instant_confirm_thresh",
              "duplicate_iou_thresh", "ams_alpha0", "ams_threshold", "ams_shrink_ratio", "gta_appearance_thresh")


class ObCfg(ctypes.Structure):
    _fields_ = [("bt", BtCfg)] + [(n, c_int) for n in OB_INTS] + [(n, c_double) for n in OB_DOUBLES]


def build() -> Path:
    deps = [SRC] + sorted(CSRC.glob("*.cuh")) + sorted(CSRC.glob("*.h"))
    key = hashlib.sha1(b"".join(p.read_bytes() for p in deps)).hexdigest()[:16]
    out_dir = Path(tempfile.gettempdir()) / f"boxmot_b200_obsim_{getpass.getuser()}"
    out_dir.mkdir(parents=True, exist_ok=True)
    out = out_dir / f"obsim_{key}.so"
    if not out.exists():
        tmp = out.with_suffix(f".{os.getpid()}.tmp.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off", f"-I{CSRC}", "-o",
                               str(tmp), str(SRC)])
        os.replace(tmp, out)
    return out


def make_cfg(feat_dim=512, cap_tracks=512, cap_dets=320, **kw):
    o = dict(OB_DEFAULTS)
    o.update({k: kw.pop(k) for k in list(kw) if k in OB_DEFAULTS})
    bt = make_bt_cfg(feat_dim=feat_dim, cap_tracks=cap_tracks, cap_dets=cap_dets, **kw)
    c = ObCfg()
    c.bt = bt
    with_reid = bool(bt.with_reid)
    alpha0 = float(np.clip(o["ams_alpha0"], 0.0, 1.0))
    c.use_second_pass, c.recovery_max_age = int(bool(o["use_second_pass"])), int(o["recovery_max_age"])
    c.second_pass_max_age, c.second_pass_min_hits = int(o["second_pass_max_age"]), int(o["second_pass_min_hits"])
    c.confirm_hits, c.tentative_max_age = max(int(o["confirm_hits"]), 1), max(int(o["tentative_max_age"]), 0)
    c.ams_on, c.ams_buffer_size = int(bool(o["ams_enabled"]) and alpha0 < 1.0), int(max(o["ams_buffer_size"], 2))
    c.gta = int(bool(o["gta_enabled"]) and with_reid)
    c.gta_min_track_length, c.gta_max_gap = max(int(o["gta_min_track_length"]), 1), max(int(o["gta_max_gap"]), 1)
    c.lambda_emb_mult = float(o["lambda_emb_multiplier"])
    for n in ("recovery_appearance_thresh", "recovery_iou_thresh", "feat_alpha", "track_low_thresh", "second_iou_thresh",
              "second_appearance_thresh", "instant_confirm_thresh", "duplicate_iou_thresh", "gta_appearance_thresh"):
        setattr(c, n, float(o[n]))
    c.new_track_thresh = max(float(o["new_track_thresh"]), 0.0)
    c.ams_alpha0, c.ams_threshold = alpha0, float(max(o["ams_threshold"], 0.0))
    c.ams_shrink_ratio = float(np.clip(o["ams_shrink_ratio"], 0.0, 1.0))
    return c


def lib():
    h = ctypes.CDLL(str(build()))
    h.obsim_create.restype = ctypes.c_void_p
    h.obsim_create.argtypes = [ctypes.c_void_p, ctypes.c_void_p, c_int]
    h.obsim_destroy.argtypes = [ctypes.c_void_p]
    h.obsim_set_warp.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
    h.obsim_update.argtypes = [ctypes.c_void_p, ctypes.c_void_p, c_int, ctypes.c_void_p, ctypes.c_void_p]
    h.obsim_snapshot.argtypes = [ctypes.c_void_p] * 5 + [c_int]
    h.obsim_take_events.argtypes = [ctypes.c_void_p, ctypes.c_void_p, c_int]
    h.obsim_ams_alpha.restype = c_double
    h.obsim_ams_alpha.argtypes = [ctypes.c_void_p, c_int, c_int, ctypes.c_void_p, c_double, c_double, c_double]
    assert h.obsim_cfg_size() == ctypes.sizeof(ObCfg)
    return h


class ObSimTracker:
    def __init__(self, cfg: ObCfg):
        self.lib = lib()
        self.cfg = cfg
        self.pow = np.array([0.9 ** k for k in range(max(8, cfg.bt.max_age + 2))], dtype=np.float64)
        self.h = self.lib.obsim_create(ctypes.byref(cfg), self.pow.ctypes.data, len(self.pow))
        self.width = self.lib.obsim_ev_width()

    def __del__(self):
        if getattr(self, "h", None):
            self.lib.obsim_destroy(self.h)

    def update(self, dets, embs=None, warp=None):
        dets = np.ascontiguousarray(np.asarray(dets, np.float32).reshape(-1, 6))
        if warp is not None:
            w = np.ascontiguousarray(warp, np.float64).reshape(6)
            self.lib.obsim_set_warp(self.h, w.ctypes.data)
        e = None
        if embs is not None and len(dets):
            e = np.ascontiguousarray(embs, np.float32)
        out = np.zeros((max(len(dets), 1), 8), np.float32)
        n = self.lib.obsim_update(self.h, dets.ctypes.data if len(dets) else None, len(dets),
                                  e.ctypes.data if e is not None else None, out.ctypes.data)
        if n < 0:
            raise RuntimeError(f"obsim error {-n}")
        return out[:n]

    def snapshot(self):
        cap = self.cfg.bt.cap_tracks
        ids, act = np.zeros(cap, np.int32), np.zeros(cap, np.int32)
        xs, ps = np.zeros((cap, 8)), np.zeros((cap, 8, 8))
        n = self.lib.obsim_snapshot(self.h, ids.ctypes.data, xs.ctypes.data, ps.ctypes.data, act.ctypes.data, cap)
        return ids[:n], xs[:n], ps[:n], act[:n].astype(bool)

    def take_events(self):
        cap = self.cfg.bt.cap_tracks
        ev = np.zeros((cap, self.width))
        n = self.lib.obsim_take_events(self.h, ev.ctypes.data, cap)
        return ev[:n]
