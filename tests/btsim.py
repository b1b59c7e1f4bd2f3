"""Host simulation of the BoostTrack device core (tests only; never a product path).

Builds tests/_btsim/btsim.cpp with g++ (BMB_HOSTSIM: boxmot_b200/csrc/bt_core.cuh compiled for one host "thread") into
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

ROOT = Path(__file__).resolve().parents[1]
SRC = ROOT / "tests" / "_btsim" / "btsim.cpp"
CSRC = ROOT / "boxmot_b200" / "csrc"

c_int, c_double = ctypes.c_int, ctypes.c_double


class BtCfg(ctypes.Structure):
    _fields_ = [(n, c_int) for n in ("cap_tracks", "cap_dets", "feat_dim", "max_age", "min_hits", "with_reid", "use_dlo",
                                      "use_duo", "rich_s", "use_sb", "use_vt", "s_sim_corr", "cmc_every_frame")] + \
               [(n, c_double) for n in ("det_thresh", "iou_threshold", "lambda_iou", "lambda_mhd", "lambda_shape",
                                         "dlo_coef", "min_box_area", "ar_thresh")] + \
               [("conf_pow", ctypes.c_void_p), ("n_conf_pow", c_int)]


def build() -> Path:
    deps = [SRC] + sorted(CSRC.glob("*.cuh")) + sorted(CSRC.glob("*.h"))
    key = hashlib.sha1(b"".join(p.read_bytes() for p in deps)).hexdigest()[:16]
    out_dir = Path(tempfile.gettempdir()) / f"boxmot_b200_btsim_{getpass.getuser()}"
    out_dir.mkdir(parents=True, exist_ok=True)
    out = out_dir / f"btsim_{key}.so"
    if not out.exists():
        tmp = out.with_suffix(f".{os.getpid()}.tmp.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off", f"-I{CSRC}", "-o",
                               str(tmp), str(SRC)])
        os.replace(tmp, out)
    return out


def make_cfg(min_box_area=10, aspect_ratio_thresh=1.6, lambda_iou=0.5, lambda_mhd=0.25, lambda_shape=0.25,
             use_dlo_boost=True, use_duo_boost=True, dlo_boost_coef=0.65, s_sim_corr=False, use_rich_s=False,
             use_sb=False, use_vt=False, with_reid=False, det_thresh=0.3, max_age=30, min_hits=3, iou_threshold=0.3,
             feat_dim=512, cap_tracks=512, cap_dets=320):
    c = BtCfg()
    c.cap_tracks, c.cap_dets, c.feat_dim = cap_tracks, cap_dets, feat_dim if with_reid else 0
    c.max_age, c.min_hits, c.with_reid = max_age, min_hits, int(bool(with_reid))
    c.use_dlo, c.use_duo, c.rich_s = int(use_dlo_boost), int(use_duo_boost), int(use_rich_s)
    c.use_sb, c.use_vt, c.s_sim_corr, c.cmc_every_frame = int(use_sb), int(use_vt), int(s_sim_corr), 0
    c.det_thresh, c.iou_threshold, c.lambda_iou, c.lambda_mhd = det_thresh, iou_threshold, lambda_iou, lambda_mhd
    c.lambda_shape, c.dlo_coef, c.min_box_area, c.ar_thresh = lambda_shape, dlo_boost_coef, min_box_area, aspect_ratio_thresh
    return c


class BtSimTracker:
    def __init__(self, cfg: BtCfg):
        self.lib = ctypes.CDLL(str(build()))
        assert self.lib.btsim_cfg_size() == ctypes.sizeof(BtCfg)
        self.lib.btsim_create.restype = ctypes.c_void_p
        self.lib.btsim_create.argtypes = [ctypes.c_void_p, ctypes.c_void_p, c_int]
        self.lib.btsim_destroy.argtypes = [ctypes.c_void_p]
        self.lib.btsim_set_warp.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        self.lib.btsim_update.argtypes = [ctypes.c_void_p, ctypes.c_void_p, c_int, ctypes.c_void_p, ctypes.c_void_p]
        self.lib.btsim_snapshot.argtypes = [ctypes.c_void_p] * 4 + [c_int]
        self.cfg = cfg
        self.pow = np.array([0.9 ** k for k in range(max(8, cfg.max_age + 2))], dtype=np.float64)
        self.h = self.lib.btsim_create(ctypes.byref(cfg), self.pow.ctypes.data, len(self.pow))

    def __del__(self):
        if getattr(self, "h", None):
            self.lib.btsim_destroy(self.h)

    def update(self, dets, embs=None, warp=None):
        dets = np.ascontiguousarray(np.asarray(dets, np.float32).reshape(-1, 6))
        if warp is not None:
            w = np.ascontiguousarray(warp, np.float64).reshape(6)
            self.lib.btsim_set_warp(self.h, w.ctypes.data)
        e = None
        if embs is not None and len(dets):
            e = np.ascontiguousarray(embs, np.float32)
        out = np.zeros((max(len(dets), 1), 8), np.float32)
        n = self.lib.btsim_update(self.h, dets.ctypes.data if len(dets) else None, len(dets),
                                  e.ctypes.data if e is not None else None, out.ctypes.data)
        if n < 0:
            raise RuntimeError(f"btsim error {-n}")
        return out[:n]

    def snapshot(self):
        cap = self.cfg.cap_tracks
        ids = np.zeros(cap, np.int32)
        xs = np.zeros((cap, 8))
        ps = np.zeros((cap, 8, 8))
        n = self.lib.btsim_snapshot(self.h, ids.ctypes.data, xs.ctypes.data, ps.ctypes.data, cap)
        return ids[:n], xs[:n], ps[:n]
