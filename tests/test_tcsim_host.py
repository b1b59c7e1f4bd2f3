"""Host side of the tensor-core kernel harness (tests/tcsim.py, tests/_tcsim/tcsim.cu), no GPU needed: the harness
compiles, the numpy split-BF16 encoders and decoders agree bit for bit with the product's f2bf / pack_b / pack_f, the
instance table and shared-memory layout are what the plan relies on, and the float64 references with their bounds hold
on an emulation of the kernel's FP32 accumulation while a dropped product would exceed them."""
import numpy as np
import pytest

from tests import tcsim

pytestmark = pytest.mark.skipif(tcsim.nvcc() is None, reason="nvcc is not installed")


def _special_floats(rng):
    """Round-to-nearest-even ties on both parities, values just off a tie, tiny and subnormal magnitudes, big values."""
    base = rng.integers(0, 1 << 32, size=4000, dtype=np.uint64).astype(np.uint32)
    base = base[np.isfinite(base.view(np.float32))]
    hi = base & np.uint32(0xFFFF0000)
    ties = np.concatenate([hi | np.uint32(0x8000), hi | np.uint32(0x7FFF), hi | np.uint32(0x8001),
                           (hi & np.uint32(0xFFFEFFFF)) | np.uint32(0x8000), (hi | np.uint32(0x10000)) | np.uint32(0x8000)])
    ties = ties[np.isfinite(ties.view(np.float32)) & (np.abs(ties.view(np.float32)) < 3e38)]
    tiny = np.array([1e-45, -1e-45, 1e-40, 5.877e-39, 1.1754944e-38, -1.1754942e-38, 1e-30, 0.0, -0.0], np.float32)
    vals = [ties.view(np.float32), base.view(np.float32), tiny, rng.normal(size=2000).astype(np.float32),
            np.float32(3.0e38) * rng.uniform(-1, 1, 50).astype(np.float32)]
    v = np.concatenate(vals).astype(np.float32)
    return v[np.isfinite(v)]


def test_harness_compiles_and_lists_instances():
    inst = tcsim.instances()
    assert len(inst) == 13 and len(set(i[:3] for i in inst)) == 13
    by_mode = {}
    for np_, np2, mode, ctas in inst:
        by_mode.setdefault(mode, []).append((np_, np2))
        assert ctas in (1, 2)
    assert sorted(by_mode[tcsim.GM_PLAIN]) == [(16, 0), (32, 0), (64, 0), (96, 0), (128, 0)]
    assert sorted(by_mode[tcsim.GM_POOL]) == [(64, 0), (96, 0)]
    assert sorted(by_mode[tcsim.GM_TAIL]) == [(64, 16), (96, 32), (128, 32)]
    assert sorted(by_mode[tcsim.GM_TAIL_POOL2]) == [(64, 64), (96, 96)]
    assert by_mode[tcsim.GM_HEAD] == [(128, 0)]
    # two CTAs per SM except NP = 128 and the tails of width >= 96 (gemm_min_ctas)
    for np_, np2, mode, ctas in inst:
        one = np_ == 128 or (mode in (tcsim.GM_TAIL, tcsim.GM_TAIL_POOL2) and np_ >= 96)
        assert ctas == (1 if one else 2), (np_, np2, mode)
    shapes = [tcsim.chain_shape(s) for s in range(3)]
    assert [(g["CP"], g["CR"], g["W"], g["H"]) for g in shapes] == [(16, 16, 32, 64), (32, 24, 16, 32), (32, 32, 8, 16)]
    assert all(g["H"] % g["R"] == 0 for g in shapes)


def test_f2bf_and_split_match_the_product_bit_for_bit():
    v = _special_floats(np.random.default_rng(0))
    assert np.array_equal(tcsim.f2bf(v), tcsim.c_f2bf(v))
    hi, lo = tcsim.split(v)
    chi, clo = tcsim.c_split(v)
    assert np.array_equal(hi, chi) and np.array_equal(lo, clo)
    # the tie rule: 0x3f808000 (1 + 2^-8, odd hi below) rounds up, 0x3f818000 ... rounds to the even neighbour
    t = np.array([0x3F808000, 0x3F818000, 0x3F807FFF, 0x3F808001], np.uint32).view(np.float32)
    assert tcsim.c_f2bf(t).tolist() == [0x3F80, 0x3F82, 0x3F80, 0x3F81]
    # the split is within 2^-17 |x| for normal numbers, and hi + lo is exact for subnormal-free inputs of BF16 range
    n = v[(np.abs(v) > 1e-30) & (np.abs(v) < 1e30)]
    h, l = tcsim.split(n)
    assert (np.abs(tcsim.join(h, l) - n.astype(np.float64)) <= 2.0 ** -17 * np.abs(n.astype(np.float64))).all()
    th, tl = tcsim.split_tz(n)
    assert np.array_equal(th, (n.view(np.uint32) >> 16).astype(np.uint16))
    assert (np.abs(tcsim.join(th, tl) - n.astype(np.float64)) <= 2.0 ** -16 * np.abs(n.astype(np.float64))).all()


@pytest.mark.parametrize("K,N,K8,NP,k_row0,identity,prefix", [
    (16, 16, 2, 16, 0, False, 0), (64, 24, 8, 32, 0, False, 5), (16, 64, 10, 64, 64, False, 100),
    (64, 64, 16, 64, 64, True, 64), (24, 24, 4, 32, 0, False, 1), (128, 128, 16, 128, 0, False, 63)])
def test_pack_b_matches_the_numpy_encoder(K, N, K8, NP, k_row0, identity, prefix):
    rng = np.random.default_rng(K * N + k_row0)
    w = (np.eye(K, N) if identity else rng.normal(size=(K, N)) * np.logspace(-3, 3, K)[:, None]).astype(np.float32)
    if not identity:
        w[rng.random(w.shape) < 0.1] = 0.0
    packed, at = tcsim.c_pack_b(None if identity else w, K, N, K8, NP, k_row0, identity, prefix)
    assert at == (prefix + 63) // 64 * 64, "packed tensors start 128-byte aligned"
    assert np.array_equal(packed, tcsim.pack_b(w, K8, NP, k_row0))
    wh, wl = tcsim.unpack_b(packed, N)
    hi, lo = tcsim.split(w)
    assert np.array_equal(wh[k_row0:k_row0 + K], tcsim.bf2f(hi)) and np.array_equal(wl[k_row0:k_row0 + K], tcsim.bf2f(lo))
    assert not wh[:k_row0].any() and not wh[k_row0 + K:].any()
    assert not packed.reshape(K8, 2 * NP, 8)[:, N:NP].any() and not packed[:, NP + N:].any()


def test_pack_f_and_planes_round_trip():
    src = np.arange(1, 25, dtype=np.float32)
    out, at = tcsim.c_pack_f(src, 32, prefix=6)
    assert at == 8 and np.array_equal(out[:24], src) and not out[24:].any()
    rng = np.random.default_rng(3)
    x = tcsim.activations(rng, 3, 256, 24)
    hi, lo = tcsim.to_planes(x)
    assert hi.shape == (3, 3, 256, 8)
    dh, dl = tcsim.from_planes(hi, lo)
    sh, sl = tcsim.split(x)
    assert np.array_equal(dh, tcsim.bf2f(sh)) and np.array_equal(dl, tcsim.bf2f(sl))


def test_smem_layout():
    L = tcsim.smem_layout(10, 64, 16, 3, True, False, 4 * 128 * 16 * 2)
    assert L["b"] == 0 and L["b2"] == 10 * 2 * 64 * 16 and L["ring"] % 128 == 0
    assert L["a2"] == L["ring"] + 3 * 16384 and L["total"] == L["gate"] + 4 * 32 * 4 + 64 + 128
    P = tcsim.smem_layout(16, 64, 64, 2, True, False, 2 * 128 * 16 * 2, pool2=True)
    assert P["f"] == P["a2"], "the pooled tail's float tile aliases the tail operand"


def _emulate(a, w, bias):
    """The kernel's arithmetic in float32: per k-step of 16, the three products summed and added to the accumulator."""
    ah, al = (tcsim.bf2f(p) for p in tcsim.split(a))
    wh, wl = (tcsim.bf2f(p) for p in tcsim.split(w))
    acc = np.zeros(a.shape[:-1] + (w.shape[1],), np.float32)
    for k0 in range(0, a.shape[-1], 16):
        s = slice(k0, k0 + 16)
        for x, y in ((ah, wh), (al, wh), (ah, wl)):
            acc = (acc + (x[..., s].astype(np.float64) @ y[s].astype(np.float64)).astype(np.float32)).astype(np.float32)
    return acc + np.asarray(bias, np.float32)


@pytest.mark.parametrize("K,N", [(16, 16), (64, 32), (80, 64), (128, 96), (224, 96), (256, 128)])
def test_reference_bounds_hold_and_would_catch_a_dropped_product(K, N):
    rng = np.random.default_rng(K + N)
    a = tcsim.activations(rng, 2, 256, K)
    w = tcsim.weights(rng, K, N)
    bias = rng.normal(size=N).astype(np.float32) - 0.5
    ref, S, drops, ref32, S32 = tcsim.gemm_terms(a, w, bias)
    got = _emulate(a, w, bias).astype(np.float64)
    h, l = tcsim.split(got)
    dec = tcsim.join(h, l)
    b = tcsim.out_bound(ref, S, K)
    assert (np.abs(dec - ref) <= b).all()
    assert (np.abs(dec - ref32) <= b + tcsim.plain_bound(S32)).all()
    # without A_hi W_lo or A_lo W_hi the result lands far outside the bound on these operands
    assert tcsim.drop_ratio(drops[1:], b) >= 20, tcsim.drop_ratio(drops[1:], b)
