"""Host simulation of the SFSORT device core (tests only; never a product path).

Builds tests/_sfsim/sfsim.cpp with g++ (BMB_HOSTSIM: boxmot_b200/csrc/sf_core.cuh compiled for one host "thread") into
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
SRC = ROOT / "tests" / "_sfsim" / "sfsim.cpp"
CSRC = ROOT / "boxmot_b200" / "csrc"

c_int, c_float, c_double = ctypes.c_int, ctypes.c_float, ctypes.c_double


class SfCfg(ctypes.Structure):
    _fields_ = [(n, c_int) for n in ("cap_tracks", "cap_dets", "dynamic", "hth_f64", "nth_f64", "marginal_timeout",
                                      "central_timeout", "margins_given")] + \
               [("margin", c_float * 4)] + \
               [(n, c_double) for n in ("h_margin", "v_margin", "high_th", "new_track_th", "match_th_first", "low_th",
                                         "match_th_second", "cth", "high_th_m", "new_track_th_m", "match_th_first_m")] + \
               [("log10_tab", ctypes.c_void_p), ("n_log10", c_int)]


def build() -> Path:
    deps = [SRC] + sorted(CSRC.glob("*.cuh")) + sorted(CSRC.glob("*.h"))
    key = hashlib.sha1(b"".join(p.read_bytes() for p in deps)).hexdigest()[:16]
    out_dir = Path(tempfile.gettempdir()) / f"boxmot_b200_sfsim_{getpass.getuser()}"
    out_dir.mkdir(parents=True, exist_ok=True)
    out = out_dir / f"sfsim_{key}.so"
    if not out.exists():
        tmp = out.with_suffix(f".{os.getpid()}.tmp.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off", f"-I{CSRC}", "-o",
                               str(tmp), str(SRC)])
        os.replace(tmp, out)
    return out


def make_cfg(resolved: dict, cap_tracks=512, cap_dets=512) -> SfCfg:
    """SfCfg of the constructor-resolved parameters (tests/sfsort_oracle.resolve)."""
    from tests.sfsort_oracle import margins

    r = resolved
    c = SfCfg()
    c.cap_tracks, c.cap_dets = cap_tracks, cap_dets
    c.dynamic = c.hth_f64 = c.nth_f64 = int(r["dynamic_tuning"])
    c.marginal_timeout, c.central_timeout = r["marginal_timeout"], r["central_timeout"]
    c.h_margin, c.v_margin = float(r["horizontal_margin"]), float(r["vertical_margin"])
    if r["frame_width"] is not None and r["frame_height"] is not None:
        c.margins_given = 1
        c.margin[:] = margins(r["frame_width"], r["frame_height"], r["horizontal_margin"], r["vertical_margin"])
    for n in ("high_th", "new_track_th", "match_th_first", "low_th", "match_th_second", "cth", "high_th_m",
              "new_track_th_m", "match_th_first_m"):
        setattr(c, n, float(r[n]))
    from boxmot_b200.trackers import sfsort_log10_table

    c._log10 = sfsort_log10_table(cap_dets + 1)   # what the Python layer hands the engine
    c.log10_tab, c.n_log10 = c._log10.ctypes.data, len(c._log10)
    return c


class SfSimTracker:
    def __init__(self, cfg: SfCfg):
        self.lib = ctypes.CDLL(str(build()))
        assert self.lib.sfsim_cfg_size() == ctypes.sizeof(SfCfg)
        self.lib.sfsim_create.restype = ctypes.c_void_p
        self.lib.sfsim_create.argtypes = [ctypes.c_void_p]
        self.lib.sfsim_destroy.argtypes = [ctypes.c_void_p]
        self.lib.sfsim_update.argtypes = [ctypes.c_void_p, ctypes.c_void_p, c_int, c_int, c_int, ctypes.c_void_p]
        self.lib.sfsim_list.argtypes = [ctypes.c_void_p, c_int, ctypes.c_void_p]
        self.cfg = cfg
        self.h = self.lib.sfsim_create(ctypes.byref(cfg))

    def __del__(self):
        if getattr(self, "h", None):
            self.lib.sfsim_destroy(self.h)

    def update(self, dets, hw=(0, 0)):
        dets = np.ascontiguousarray(np.asarray(dets, np.float32).reshape(-1, 6))
        out = np.zeros((max(len(dets), 1), 8), np.float32)
        n = self.lib.sfsim_update(self.h, dets.ctypes.data if len(dets) else None, len(dets), int(hw[0]), int(hw[1]),
                                  out.ctypes.data)
        if n < 0:
            raise RuntimeError(f"sfsim error {-n}")
        return out[:n]

    def ids(self, which):
        buf = np.zeros(self.cfg.cap_tracks, np.int32)
        n = self.lib.sfsim_list(self.h, int(which), buf.ctypes.data)
        return buf[:n].tolist()
