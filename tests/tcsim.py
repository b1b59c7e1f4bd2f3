"""Harness for the tensor-core OSNet kernels (tests only; never a product path).

Builds tests/_tcsim/tcsim.cu with nvcc for sm_90a and exposes through ctypes:
- host-only helpers of boxmot_b200/csrc/reid_tc_host.cuh (f2bf and the hi / lo split, pack_b, pack_f), the k_gemm_tc
  instance table with the CTAs per SM each instance is compiled for, and gemm_smem_layout;
- one launch of one k_gemm_tc instance (`gemm`) or of one k_chain_tc shape (`chain`), operands packed by the product's
  host code.

It also holds the numpy side: the split-BF16 encoder and decoder of packed B and of activation planes
[crops][C8][HW][8], and float64 references of the GEMM epilogues with the error bounds the tests apply.

Error model of one output of a k_gemm_tc GEMM (reid_tc.cuh header): with A = A_hi + A_lo and W = W_hi + W_lo the
kernel accumulates A_hi W_hi + A_lo W_hi + A_hi W_lo in FP32 over 3 K / 16 wgmma instructions and splits the result
again (|x - hi - lo| <= 2^-17 |x|).  Against the float64 value of the same three products on the decoded operands:
    |err| <= 2^-16 |ref| + (3 K / 16 + 2) 3 * 2^-23 S,    S = sum_k |A_hi W_hi| + |A_lo W_hi| + |A_hi W_lo| + |bias|
(each wgmma adds at most 3 ulp of the running magnitude, bounded by S: the products of a k-step are aligned to the
largest exponent and truncated, so a k-step with one dominant product loses more than one rounding; 2 ulp per wgmma
was exceeded by 8 % on an H100 with a pixel whose K values span 1e-3 .. 1e3).  Against the float64 value of the plain float32
operands (A, W), the operand splits (2^-17 each) and the dropped A_lo W_lo (2^-18) add at most 2^-15 sum_k |A W|.
"""
from __future__ import annotations

import ctypes
import os
import shutil
import subprocess
import tempfile
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
SRC = ROOT / "tests" / "_tcsim" / "tcsim.cu"
CSRC = ROOT / "boxmot_b200" / "csrc"
DEPS = [SRC, CSRC / "reid_tc.cuh", CSRC / "reid_tc_host.cuh", CSRC / "wgmma.cuh", CSRC / "engine.h"]
_LIB = None

GM_PLAIN, GM_POOL, GM_TAIL, GM_TAIL_POOL2, GM_HEAD = range(5)
MODE_NAMES = {GM_PLAIN: "plain", GM_POOL: "pool", GM_TAIL: "tail", GM_TAIL_POOL2: "tail+pool", GM_HEAD: "head"}

P = ctypes.c_void_p
C_INT, C_LL = ctypes.c_int, ctypes.c_longlong


class GemmCfg(ctypes.Structure):
    _fields_ = [(n, C_INT) for n in ("NP", "NP2", "mode", "H", "W", "n_src")] + [
        ("c8", C_INT * 2), ("kc", C_INT * 2)] + [
        (n, C_INT) for n in ("n_stage", "tiles_per_cta", "relu", "midp", "out_planes", "out_f32", "N", "N2", "feat",
                             "out_ld", "cap", "off", "count")]


class GemmIO(ctypes.Structure):
    _fields_ = [("a", P * 2)] + [(n, P) for n in ("w", "bias", "wfold", "w2", "bias2", "head_w", "head_b", "out_row")] + [
        ("out_hi", P), ("out_lo", P), ("out_n", C_LL), ("out2_hi", P), ("out2_lo", P), ("out2_n", C_LL),
        ("out_f32", P), ("f32_n", C_LL), ("head_out", P), ("head_n", C_LL)]


class ChainCfg(ctypes.Structure):
    _fields_ = [(n, C_INT) for n in ("shape", "mid", "hid", "N", "cap", "off", "n_launch")] + [("counts", C_INT * 4)]


class ChainIO(ctypes.Structure):
    _fields_ = [(n, P) for n in ("x", "pw", "dw", "b", "g1w", "g1b", "g2w", "g2b", "w3", "y_hi", "y_lo", "sums", "gates",
                                 "bfold", "arrivals")]


_SIGS = {
    "tcsim_last_error": (ctypes.c_char_p, []),
    "tcsim_f2bf": (None, [P, C_LL, P]),
    "tcsim_split": (None, [P, C_LL, P, P]),
    "tcsim_pack_b": (C_LL, [P, C_INT, C_INT, C_INT, C_INT, C_INT, C_INT, C_INT, C_INT, P]),
    "tcsim_pack_f": (C_LL, [P, C_INT, C_INT, C_INT, P]),
    "tcsim_n_instances": (C_INT, []),
    "tcsim_instance": (None, [C_INT, P, P, P, P]),
    "tcsim_smem_layout": (None, [C_INT] * 8 + [P]),
    "tcsim_smem_limit": (C_INT, []),
    "tcsim_gemm": (C_INT, [ctypes.POINTER(GemmCfg), ctypes.POINTER(GemmIO), P]),
    "tcsim_chain_shape": (None, [C_INT, P]),
    "tcsim_chain": (C_INT, [ctypes.POINTER(ChainCfg), ctypes.POINTER(ChainIO)]),
}


def nvcc():
    found = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return found if Path(found).exists() else None


def lib():
    """Compile (into a per-user temporary directory, so a read-only tree works) and load the harness."""
    global _LIB
    if _LIB is None:
        cc = nvcc()
        if cc is None:
            raise RuntimeError("nvcc not found: the tensor-core kernel harness cannot be built")
        stamp = max(int(d.stat().st_mtime) for d in DEPS)
        out_dir = Path(tempfile.gettempdir()) / f"boxmot_b200_tcsim_{os.getuid()}"
        out_dir.mkdir(exist_ok=True)
        out = out_dir / f"tcsim_{stamp}.so"
        if not out.exists():
            tmp = out.with_suffix(f".{os.getpid()}.tmp.so")
            subprocess.check_call([cc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-shared",
                                   "-Xcompiler", "-fPIC", f"-I{CSRC}", "-o", str(tmp), str(SRC)])
            os.replace(tmp, out)
        L = ctypes.CDLL(str(out))
        for name, (res, args) in _SIGS.items():
            fn = getattr(L, name)
            fn.restype, fn.argtypes = res, args
        _LIB = L
    return _LIB


def _ptr(a):
    return None if a is None else a.ctypes.data


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


# ---- host-only entry points -------------------------------------------------------------------------------------------
def c_f2bf(x):
    x = _f32(x)
    out = np.empty(x.shape, np.uint16)
    lib().tcsim_f2bf(_ptr(x), x.size, _ptr(out))
    return out


def c_split(x):
    x = _f32(x)
    hi, lo = np.empty(x.shape, np.uint16), np.empty(x.shape, np.uint16)
    lib().tcsim_split(_ptr(x), x.size, _ptr(hi), _ptr(lo))
    return hi, lo


def c_pack_b(w, K, N, K8, NP, k_row0=0, identity=False, prefix=0):
    w = _f32(np.zeros((max(K, 1), N)) if w is None else w)
    out = np.empty((K8, 2 * NP, 8), np.uint16)
    at = lib().tcsim_pack_b(_ptr(w), K, N, w.shape[1], K8, NP, k_row0, int(identity), prefix, _ptr(out))
    return out, at


def c_pack_f(src, n_pad, prefix=0):
    src = _f32(src)
    out = np.empty(n_pad, np.float32)
    at = lib().tcsim_pack_f(_ptr(src), len(src), n_pad, prefix, _ptr(out))
    return out, at


def instances():
    """[(NP, NP2, mode, CTAs per SM the instance is compiled for)] in kGemmInstances order."""
    L = lib()
    res = []
    for i in range(L.tcsim_n_instances()):
        v = [ctypes.c_int() for _ in range(4)]
        L.tcsim_instance(i, *[ctypes.byref(x) for x in v])
        res.append(tuple(x.value for x in v))
    return res


def smem_layout(K8, NP, NP2, n_stage, tail, pool, slot_bytes, pool2=False):
    out = np.zeros(7, np.int64)
    lib().tcsim_smem_layout(K8, NP, NP2, n_stage, int(tail), int(pool), slot_bytes, int(pool2), _ptr(out))
    return dict(zip(("b", "b2", "ring", "a2", "f", "gate", "total"), out.tolist()))


def chain_shape(shape):
    out = np.zeros(5, np.int32)
    lib().tcsim_chain_shape(shape, _ptr(out))
    return dict(zip(("CP", "CR", "W", "H", "R"), out.tolist()))


# ---- numpy encoders / decoders ----------------------------------------------------------------------------------------
def f2bf(x):
    """Round float32 to BF16 bits, nearest even (f2bf of reid_tc_host.cuh, __float2bfloat16_rn for finite x)."""
    u = _f32(x).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFFFFFF
    return (u >> 16).astype(np.uint16)


def bf2f(h):
    return (np.asarray(h, np.uint16).astype(np.uint32) << 16).view(np.float32)


def split(x):
    """hi = bf16(x), lo = bf16(x - hi): pack_b's split, and split2 of the kernels."""
    x = _f32(x)
    hi = f2bf(x)
    return hi, f2bf(x - bf2f(hi))


def split_tz(x):
    """split2_tz of the depthwise walkers: hi = the upper 16 bits (truncation), lo = bf16_rn(x - hi)."""
    x = _f32(x)
    hi = (x.view(np.uint32) >> 16).astype(np.uint16)
    return hi, f2bf(x - bf2f(hi))


def join(hi, lo):
    """float64 value hi + lo of split planes (exact)."""
    return bf2f(hi).astype(np.float64) + bf2f(lo).astype(np.float64)


def pack_b(w, K8, NP, k_row0=0):
    """W [K][N] float32 -> packed B [K8][2 NP][8] uint16 (row n = hi of column n, row NP + n = lo), like pack_b."""
    w = _f32(w)
    K, N = w.shape
    hi, lo = split(w)
    out = np.zeros((K8 * 8, 2 * NP), np.uint16)
    out[k_row0:k_row0 + K, :N] = hi
    out[k_row0:k_row0 + K, NP:NP + N] = lo
    return np.ascontiguousarray(out.reshape(K8, 8, 2 * NP).transpose(0, 2, 1))


def unpack_b(packed, N):
    """Packed B [K8][2 NP][8] -> (W_hi, W_lo) as float64 [K][N]."""
    K8, NP2, _ = packed.shape
    NP = NP2 // 2
    m = packed.transpose(0, 2, 1).reshape(K8 * 8, 2 * NP)
    return bf2f(m[:, :N]).astype(np.float64), bf2f(m[:, NP:NP + N]).astype(np.float64)


def to_planes(x):
    """float32 NHWC [crops][HW][C8 * 8] -> (hi, lo) planes [crops][C8][HW][8]."""
    x = _f32(x)
    c, hw, k = x.shape
    hi, lo = split(x)
    f = lambda p: np.ascontiguousarray(p.reshape(c, hw, k // 8, 8).transpose(0, 2, 1, 3))
    return f(hi), f(lo)


def from_planes(hi, lo, HW=None):
    """Planes [crops][C8][HW][8] (flat or shaped) -> (hi, lo) NHWC [crops][HW][C8 * 8] as float64."""
    hi, lo = np.asarray(hi), np.asarray(lo)
    c, c8, hw, _ = hi.shape
    f = lambda p: bf2f(p).astype(np.float64).transpose(0, 2, 1, 3).reshape(c, hw, c8 * 8)
    return f(hi), f(lo)


# ---- float64 references and bounds -------------------------------------------------------------------------------------
def gemm_terms(a, w, bias):
    """The three products of the kernel on decoded operands: a, w float32 [.., K], [K, N].

    Returns (ref, S, drops, ref32, S32): ref = A_hi W_hi + A_lo W_hi + A_hi W_lo + bias in float64, S the sum of
    magnitudes of its terms, drops the three products themselves (what dropping one would cost), ref32 / S32 the same for
    the plain float32 operands."""
    ah, al = (bf2f(p).astype(np.float64) for p in split(a))
    wh, wl = (bf2f(p).astype(np.float64) for p in split(w))
    b = np.asarray(bias, np.float64)
    t = (ah @ wh, al @ wh, ah @ wl)
    ref = t[0] + t[1] + t[2] + b
    S = np.abs(ah) @ np.abs(wh) + np.abs(al) @ np.abs(wh) + np.abs(ah) @ np.abs(wl) + np.abs(b)
    a64, w64 = np.asarray(a, np.float64), np.asarray(w, np.float64)
    return ref, S, t, a64 @ w64 + b, np.abs(a64) @ np.abs(w64) + np.abs(b)


def acc_bound(S, K):
    """FP32 accumulation over the 3 K / 16 wgmma of a K-deep GEMM (plus bias add)."""
    return (3 * K / 16 + 2) * 3 * 2.0 ** -23 * S


def out_bound(ref, S, K, split_out=True):
    """Decoded output against the float64 value of the same products: accumulation, plus the output split."""
    return acc_bound(S, K) + (2.0 ** -16 if split_out else 2.0 ** -23) * np.abs(ref)


def plain_bound(S32):
    """Additional error against the float64 value of the plain float32 operands: operand splits and the dropped lo lo."""
    return 2.0 ** -15 * S32


def relu(x):
    return np.maximum(x, 0.0)


def pool2x2(x, H, W):
    """2x2 average pool of NHWC [crops][H * W][C] -> [crops][H / 2 * W / 2][C] (float64)."""
    c, _, k = x.shape
    v = x.reshape(c, H // 2, 2, W // 2, 2, k)
    return v.mean(axis=(2, 4)).reshape(c, (H // 2) * (W // 2), k)


def drop_ratio(drops, bound):
    """min over the three products of max over outputs of |product| / bound: how far above its bound the error of
    dropping the least significant product would land."""
    return min(float((np.abs(d) / bound).max()) for d in drops)


# ---- launches -----------------------------------------------------------------------------------------------------------
BF16_CANARY = 0xFFC1      # a NaN in BF16
F32_CANARY = np.uint32(0xFFC00001).view(np.float32)
SLACK = 4096              # canary elements behind every output tensor


def gemm(NP, NP2, mode, H, W, a, w, bias, *, kc, n_stage, tiles_per_cta, N=None, relu_=True, midp=0, wfold=None,
         w2=None, bias2=None, N2=None, out_planes=None, out_f32=False, head_w=None, head_b=None, out_row=None,
         out_ld=None, out_rows=None, cap=None, off=0, count=None):
    """One launch of k_gemm_tc<NP, NP2, mode> over `cap` crops (device count `count`, window offset `off`).

    a: list of float32 [cap][H W][C8 * 8] sources.  Returns None when the layout does not fit shared memory, else a dict
    of the raw outputs (canary-filled buffers with SLACK elements behind each) and the launch info."""
    L = lib()
    a = [_f32(x) for x in a]
    cap = a[0].shape[0] if cap is None else cap
    count = cap if count is None else count
    N = NP if N is None else N
    HW = H * W
    c8 = [x.shape[2] // 8 for x in a]
    tail, pool, pool2 = mode in (GM_TAIL, GM_TAIL_POOL2), mode == GM_POOL, mode == GM_TAIL_POOL2
    if out_planes is None:
        out_planes = mode in (GM_PLAIN, GM_POOL, GM_TAIL) and not out_f32
    cfg = GemmCfg(NP=NP, NP2=NP2, mode=mode, H=H, W=W, n_src=len(a), n_stage=n_stage, tiles_per_cta=tiles_per_cta,
                  relu=int(relu_), midp=midp, out_planes=int(out_planes), out_f32=int(out_f32), N=N,
                  N2=(N2 if N2 is not None else NP2), feat=0 if head_w is None else head_w.shape[1],
                  out_ld=out_ld or 0, cap=cap, off=off, count=count)
    for s in range(len(a)):
        cfg.c8[s], cfg.kc[s] = c8[s], kc[s]
    keep = []

    def hold(x):
        keep.append(x)
        return _ptr(x)

    io = GemmIO()
    for s in range(len(a)):
        io.a[s] = hold(a[s])
    io.w, io.bias = hold(_f32(w)), hold(_f32(bias))
    if midp:
        io.wfold = hold(_f32(wfold))
    res = {}
    out_hw = HW // 4 if pool else HW
    n_out = cap * (NP // 8) * out_hw * 8
    res["out_hi"] = np.full(n_out + SLACK, BF16_CANARY, np.uint16)
    res["out_lo"] = np.full(n_out + SLACK, BF16_CANARY, np.uint16)
    io.out_hi, io.out_lo, io.out_n = hold(res["out_hi"]), hold(res["out_lo"]), n_out + SLACK
    if out_f32:
        res["out_f32"] = np.full(cap * HW * N + SLACK, F32_CANARY, np.float32)
        io.out_f32, io.f32_n = hold(res["out_f32"]), cap * HW * N + SLACK
    if tail:
        io.w2, io.bias2 = hold(_f32(w2)), hold(_f32(bias2))
        n2 = cap * (NP2 // 8) * (HW // 4 if pool2 else HW) * 8
        res["out2_hi"] = np.full(n2 + SLACK, BF16_CANARY, np.uint16)
        res["out2_lo"] = np.full(n2 + SLACK, BF16_CANARY, np.uint16)
        io.out2_hi, io.out2_lo, io.out2_n = hold(res["out2_hi"]), hold(res["out2_lo"]), n2 + SLACK
    if mode == GM_HEAD:
        io.head_w, io.head_b = hold(_f32(head_w)), hold(_f32(head_b))
        io.out_row = hold(np.ascontiguousarray(out_row, np.int32))
        res["head"] = np.full(out_rows * out_ld + SLACK, F32_CANARY, np.float32)
        io.head_out, io.head_n = hold(res["head"]), out_rows * out_ld + SLACK
    info = np.zeros(4, np.int32)
    rc = L.tcsim_gemm(ctypes.byref(cfg), ctypes.byref(io), _ptr(info))
    if rc < 0:
        raise RuntimeError(L.tcsim_last_error().decode())
    if rc == 1:
        return None
    res.update(smem=int(info[0]), ctas=int(info[1]), groups=int(info[2]), out_hw=out_hw)
    return res


def chain(shape, xs, pw, dw, b, g1w, g1b, g2w, g2b, w3, counts, off=0):
    """Consecutive k_chain_tc launches (one per entry of `counts`, input xs[i]) on one set of buffers."""
    L = lib()
    g = chain_shape(shape)
    CP, CR, W, H, R = g["CP"], g["CR"], g["W"], g["H"], g["R"]
    xs = _f32(xs)
    cap = xs.shape[1]
    N = w3.shape[1]
    NP = (N + 15) // 16 * 16
    tiles = H // R
    res = {
        "y_hi": np.full(cap * 4 * CP * H * W + SLACK, BF16_CANARY, np.uint16),
        "y_lo": np.full(cap * 4 * CP * H * W + SLACK, BF16_CANARY, np.uint16),
        "sums": np.full(4 * cap * tiles * CP, F32_CANARY, np.float32),
        "gates": np.full(cap * 4 * CP, F32_CANARY, np.float32),
        "bfold": np.full(cap * (4 * CP // 8) * 2 * NP * 8, BF16_CANARY, np.uint16),
        "arrivals": np.full(cap, -7, np.int32),
    }
    ins = [xs, _f32(pw), _f32(dw), _f32(b), _f32(g1w), _f32(g1b), _f32(g2w), _f32(g2b), _f32(w3)]
    cfg = ChainCfg(shape=shape, mid=CR, hid=g1w.shape[1], N=N, cap=cap, off=off, n_launch=len(counts))
    for i, c in enumerate(counts):
        cfg.counts[i] = c
    io = ChainIO(*[_ptr(x) for x in ins], *[_ptr(res[k]) for k in ("y_hi", "y_lo", "sums", "gates", "bfold", "arrivals")])
    if L.tcsim_chain(ctypes.byref(cfg), ctypes.byref(io)) < 0:
        raise RuntimeError(L.tcsim_last_error().decode())
    res.update(CP=CP, CR=CR, W=W, H=H, R=R, NP=NP, tiles=tiles)
    return res


# ---- synthetic operands -------------------------------------------------------------------------------------------------
def activations(rng, cap, HW, K, nonneg=False):
    """Activations [cap][HW][K] that exercise the split: normal values, ~20 % exact zeros, values on round-to-nearest-even
    ties of the hi part, one pixel row per crop whose K values span 1e-3 .. 1e3."""
    a = rng.normal(size=(cap, HW, K)).astype(np.float32)
    if nonneg:
        a = np.abs(a)
    a[rng.random(a.shape) < 0.2] = 0.0
    ties = rng.random(a.shape) < 0.05            # hi exactly halfway between two BF16 values
    u = a.view(np.uint32)
    u[ties] = (u[ties] & np.uint32(0xFFFF0000)) | np.uint32(0x8000)
    a[:, 7, :] *= np.logspace(-3, 3, K, dtype=np.float32)[None, :]
    return a


def weights(rng, K, N, scale=None):
    return (rng.normal(size=(K, N)) * (scale if scale is not None else 1.0 / np.sqrt(K))).astype(np.float32)
