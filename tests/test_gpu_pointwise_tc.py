"""Tensor-core (wgmma tf32 x3) pointwise GEMM against float64 numpy and against the CUDA-core kernel, at the layer shapes
of OSNet_x0_25 (and padding cases N=24, K=88)."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _gemm(a, w, bias, res, relu, tc):
    from boxmot_b200 import _lib

    lib = _lib.require_device()
    m, k = a.shape
    n = w.shape[1]
    out = np.empty((m, n), np.float32)
    ms = ctypes.c_float(0)
    ok = lib.boxmot_b200_pointwise_gemm(a.ctypes.data, m, k, w.ctypes.data, n, bias.ctypes.data,
                                        res.ctypes.data if res is not None else None, int(relu), int(tc),
                                        out.ctypes.data, ctypes.byref(ms))
    assert ok == 1, _lib.last_error(lib)
    return out, ms.value


@pytest.mark.parametrize("m,k,n,relu,use_res", [
    (128, 16, 16, 1, 0), (256 * 128, 16, 16, 1, 0), (4096, 64, 16, 1, 0), (2048, 32, 64, 1, 0), (2048, 88, 96, 1, 0),
    (1024, 24, 96, 1, 1), (1024, 96, 24, 1, 0), (512, 128, 128, 1, 1), (512, 128, 32, 0, 0), (2048, 64, 64, 1, 0)])
def test_tcgen05_pointwise_matches_fp64(m, k, n, relu, use_res):
    rng = np.random.default_rng(m + k + n)
    a = rng.normal(size=(m, k)).astype(np.float32) * 3
    w = (rng.normal(size=(k, n)) / np.sqrt(k)).astype(np.float32)
    bias = rng.normal(size=n).astype(np.float32)
    res = rng.normal(size=(m, n)).astype(np.float32) if use_res else None
    want = a.astype(np.float64) @ w.astype(np.float64) + bias + (res if use_res else 0)
    if relu:
        want = np.maximum(want, 0)
    got_tc, ms_tc = _gemm(a, w, bias, res, relu, 1)
    got_cc, ms_cc = _gemm(a, w, bias, res, relu, 0)
    scale = np.abs(want).max()
    err_tc = np.abs(got_tc - want).max() / scale
    err_cc = np.abs(got_cc - want).max() / scale
    print(f"M={m} K={k} N={n}: tensor cores {ms_tc * 1e3:.1f} us err {err_tc:.2e} | cuda-core {ms_cc * 1e3:.1f} us err {err_cc:.2e}")
    assert err_cc < 2e-6
    assert err_tc < 2e-6, "tf32 x3 split must keep float32-class accuracy"


@pytest.mark.parametrize("m,k,n", [(262144, 16, 16), (262144, 64, 16), (262144, 32, 64), (262144, 64, 64),
                                   (65536, 88, 96), (65536, 96, 96), (16384, 128, 128)])
def test_tcgen05_pointwise_large_timing(m, k, n):
    rng = np.random.default_rng(1)
    a = rng.normal(size=(m, k)).astype(np.float32)
    w = (rng.normal(size=(k, n)) / np.sqrt(k)).astype(np.float32)
    bias = np.zeros(n, np.float32)
    got_tc, ms_tc = _gemm(a, w, bias, None, 1, 1)
    got_cc, ms_cc = _gemm(a, w, bias, None, 1, 0)
    gb = (m * k + m * n) * 4 / 1e9
    print(f"M={m} K={k} N={n}: tensor cores {ms_tc * 1e3:.1f} us ({gb / ms_tc * 1e3:.0f} GB/s) | cuda-core {ms_cc * 1e3:.1f} us "
          f"({gb / ms_cc * 1e3:.0f} GB/s)")
    np.testing.assert_allclose(got_tc, got_cc, rtol=0, atol=2e-5 * np.abs(got_cc).max())
