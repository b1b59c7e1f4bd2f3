"""Build libboxmot_b200.so in-tree with nvcc for sm_90a (cross-compiles without a GPU)."""
from __future__ import annotations

import os
import shutil
import subprocess
from pathlib import Path

PKG = Path(__file__).resolve().parent
CSRC = PKG / "csrc"
LIB = PKG / "libboxmot_b200.so"

# -fmad=false for the float64 tracker translation units: the reference's numpy arithmetic never contracts
# a*b+c, and the Kalman / IoU / cost expressions are reproduced operation by operation.
TRACKER_SOURCES = ["tracker_engine.cu", "ss_kernels.cu", "cmc_kernels.cu", "cmc_sof_kernels.cu", "capi.cu"]
REID_SOURCES = ["reid_model.cu"]
COMMON = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
          "-Xcompiler", "-fPIC,-fvisibility=hidden"]


def _nvcc() -> str:
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not Path(nvcc).exists():
        raise RuntimeError("nvcc not found: libboxmot_b200.so cannot be built")
    return nvcc


def _stale(out: Path, deps) -> bool:
    if not out.exists():
        return True
    t = out.stat().st_mtime
    return any(Path(d).stat().st_mtime > t for d in deps)


def build_library(force: bool = False, verbose: bool = False) -> Path:
    nvcc = _nvcc()
    headers = list(CSRC.glob("*.cuh")) + list(CSRC.glob("*.h")) + [PKG.parent / "include" / "boxmot_b200.h"]
    objs = []
    build_dir = CSRC / "_obj"
    build_dir.mkdir(exist_ok=True)
    for name in TRACKER_SOURCES + REID_SOURCES:
        src = CSRC / name
        obj = build_dir / (src.stem + ".o")
        if force or _stale(obj, [src] + headers):
            cmd = [nvcc, *COMMON, "-c", str(src), "-o", str(obj)]
            if name in TRACKER_SOURCES:
                cmd.insert(1, "-fmad=false")
            if name == "tracker_engine.cu":
                # 512 threads for the BoT-SORT / ByteTrack frame kernel: the parallel cost-build phases gain more than
                # the Kalman update loses to spills
                cmd.insert(1, "-DBMB_FRAME_THREADS=512")
            if verbose:
                cmd.insert(1, "-Xptxas=-v")
            subprocess.check_call(cmd)
        objs.append(obj)
    if force or _stale(LIB, objs):
        tmp = LIB.with_suffix(f".{os.getpid()}.tmp")
        subprocess.check_call([nvcc, *COMMON, "-shared", "-o", str(tmp), *map(str, objs), "-lcudart"])
        os.replace(tmp, LIB)
    return LIB


if __name__ == "__main__":
    import sys

    print(build_library(force="--force" in sys.argv, verbose="-v" in sys.argv))
