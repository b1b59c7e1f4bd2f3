"""Host build of boxmot_b200/csrc/cmc_sof.cuh (tests only; never a product path).

Builds tests/_sofsim/sofsim.cpp with g++ (BMB_HOSTSIM, no FMA contraction) and exposes the SOF arithmetic through
ctypes: the gray-level stages (eigenvalue map, corners, cornerSubPix, pyramidal LK, RANSAC + refine) and the whole
`SOF.apply` step.  The CPU tests pin it on the installed OpenCV; the GPU tests pin the kernels on it bit for bit.
"""
from __future__ import annotations

import ctypes
import os
import subprocess
import tempfile
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
SRC = ROOT / "tests" / "_sofsim" / "sofsim.cpp"
CSRC = ROOT / "boxmot_b200" / "csrc"
_LIB = None

P = ctypes.c_void_p
C_INT, C_FLOAT, C_DOUBLE = ctypes.c_int, ctypes.c_float, ctypes.c_double
_SIGS = {
    "sofsim_eig": (None, [P, C_INT, C_INT, P]),
    "sofsim_mask": (None, [C_INT, C_INT, P, C_INT, C_INT, C_FLOAT, P]),
    "sofsim_corners": (C_INT, [P, C_INT, C_INT, P, P]),
    "sofsim_subpix": (None, [P, C_INT, C_INT, P, C_INT]),
    "sofsim_levels": (C_INT, [C_INT, C_INT]),
    "sofsim_lk": (None, [P, P, C_INT, C_INT, P, C_INT, P, P]),
    "sofsim_ransac": (C_INT, [P, P, C_INT, C_FLOAT, P, P, P]),
    "sofsim_create": (P, [C_DOUBLE, C_INT, C_DOUBLE, C_FLOAT]),
    "sofsim_destroy": (None, [P]),
    "sofsim_apply": (None, [P, P, C_INT, C_INT, P, C_INT, C_INT, P, P, P]),
}


def lib():
    """Compile (into a per-user temporary directory, so a read-only tree works) and load the host build."""
    global _LIB
    if _LIB is None:
        deps = [SRC, CSRC / "cmc_sof.cuh", CSRC / "cmc_ecc.cuh", CSRC / "tracker_core.cuh"]
        stamp = max(int(d.stat().st_mtime) for d in deps)
        out_dir = Path(tempfile.gettempdir()) / f"boxmot_b200_sofsim_{os.getuid()}"
        out_dir.mkdir(exist_ok=True)
        out = out_dir / f"sofsim_{stamp}.so"
        if not out.exists():
            tmp = out.with_suffix(f".{os.getpid()}.tmp.so")
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-ffp-contract=off",
                                   f"-I{CSRC}", "-o", str(tmp), str(SRC)])
            os.replace(tmp, out)
        L = ctypes.CDLL(str(out))
        for name, (res, args) in _SIGS.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        _LIB = L
    return _LIB


def _u8(a):
    return np.ascontiguousarray(a, dtype=np.uint8)


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def eig(gray):
    g = _u8(gray)
    out = np.empty(g.shape, np.float32)
    lib().sofsim_eig(g.ctypes.data, g.shape[0], g.shape[1], out.ctypes.data)
    return out


def mask(h, w, dets, scale=0.15):
    d = _f32(np.zeros((0, 4)) if dets is None else dets)
    out = np.empty((h, w), np.uint8)
    lib().sofsim_mask(h, w, d.ctypes.data, len(d), d.shape[1] if d.ndim == 2 and len(d) else 4, scale, out.ctypes.data)
    return out


def corners(gray, m):
    g, m = _u8(gray), _u8(m)
    xy = np.empty((1000, 2), np.float32)
    n = lib().sofsim_corners(g.ctypes.data, g.shape[0], g.shape[1], m.ctypes.data, xy.ctypes.data)
    return xy[:n].copy()


def subpix(gray, pts):
    g, xy = _u8(gray), _f32(pts).copy()
    lib().sofsim_subpix(g.ctypes.data, g.shape[0], g.shape[1], xy.ctypes.data, len(xy))
    return xy


def levels(h, w):
    return lib().sofsim_levels(h, w)


def lk(prev, cur, pts):
    a, b, p = _u8(prev), _u8(cur), _f32(pts).reshape(-1, 2)
    out = np.empty_like(p)
    st = np.empty(len(p), np.int32)
    lib().sofsim_lk(a.ctypes.data, b.ctypes.data, a.shape[0], a.shape[1], p.ctypes.data, len(p), out.ctypes.data,
                    st.ctypes.data)
    return out, st


def ransac(src, dst, thr=3.0):
    """estimateAffinePartial2D(src, dst, RANSAC, thr): (2x3 float64 model or None, inlier mask uint8)."""
    s, d = _f32(src).reshape(-1, 2), _f32(dst).reshape(-1, 2)
    M = np.zeros((2, 3), np.float64)
    inl = np.zeros(len(s), np.uint8)
    n_inl = ctypes.c_int(0)
    ok = lib().sofsim_ransac(s.ctypes.data, d.ctypes.data, len(s), thr, M.ctypes.data, inl.ctypes.data,
                             ctypes.byref(n_inl))
    return (M if ok else None), inl


class HostSOF:
    """SOF.apply composed serially from the host build; `status` after apply: 0 init, 1 estimated, 2 rejected."""

    def __init__(self, scale=0.15, min_inliers=8, min_inlier_ratio=0.2, ransac_reproj_threshold=3.0):
        self.scale = scale
        self._h = lib().sofsim_create(scale, min_inliers, min_inlier_ratio, ransac_reproj_threshold)
        self.status, self.reg = None, None

    def __del__(self):
        if getattr(self, "_h", None):
            lib().sofsim_destroy(self._h)
            self._h = None

    def apply(self, img, dets=None):
        im = _u8(img)
        d = _f32(np.zeros((0, 4)) if dets is None or len(dets) == 0 else np.asarray(dets)[:, :4])
        rows, cols = im.shape[:2]
        warp = np.zeros((2, 3), np.float32)
        st = ctypes.c_int(-1)
        self.reg = np.empty((int(np.rint(rows * self.scale)), int(np.rint(cols * self.scale))), np.uint8)
        lib().sofsim_apply(self._h, im.ctypes.data, rows, cols, d.ctypes.data, len(d), 4, warp.ctypes.data,
                           ctypes.byref(st), self.reg.ctypes.data)
        self.status = st.value
        return warp
