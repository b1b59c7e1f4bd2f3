"""Every float32 CUDA-core ReID kernel on its own against float64: the kernels osnet_x1_0 / _x0_75 / _x0_5, OSNet-AIN /
OSNet-IBN, LMBN_n and MobileNetV2_x1_4 run (csrc/reid_model.cu, csrc/lmbn_head.cuh), launched through the same launcher
methods a loaded model uses (boxmot_b200_f32_* in include/boxmot_b200.h), at the layer shapes those models have.

Error model (u = 2^-24, float32 round-to-nearest; every kernel accumulates with fmaf or float adds, no fast math):
- A K-deep fmaf chain plus a bias, in any order and any split into partial sums, is within
  (K + 2) u (sum_k |a_k| |w_k| + |b|) of the exact value.  A residual add is one more rounding: the pointwise bound is
  (K + 3) u (|A| |W| + |b| + |r|).  The gated prologue builds A from four fmaf, so a gated column adds 4 u (|g| |x|)
  per input, folded in as (K + 7) u with |A| = sum_b |g_b| |x_b|.  ReLU and ReLU6 are 1-Lipschitz and keep the bound.
- LightConv3x3 = C-deep 1x1 (float32 intermediate in shared memory) then a 9-tap depthwise + bias: composed, the error
  is within (C + 12) u (dw(|X| |Wpw|, |Wdw|) + |b|), dw = the depthwise convolution of the absolute values.  A chain of
  levels adds the previous level's bound pushed through |Wpw| and |Wdw| (the ReLU is 1-Lipschitz).
- Channel sums of a tile of P pixels: P u sum |y| against the float64 sum of the kernel's own outputs.
- ChannelGate: the mean carries (tiles + 1) u sum |s| / HW; fc1 and fc2 are fmaf chains as above plus the input error
  through |W|; the sigmoid 1 / (1 + expf(-s)) has slope <= 1/4 and expf is within 2 ulp, so 0.25 e_s + 4 u.
- Head: the average pool carries (HW + 1) u mean|x|, the fc an (C + 5)-deep chain, the ReLU nothing, the L2 norm
  e_s / ||s|| + |y| (||e_s|| / ||s|| + (F / 2 + 3) u) for an F-element row.
- Stems and the depthwise 3x3: K-deep fmaf chains (147, 27, 9 taps).  Max pools are exact; the 2x2 average is three
  adds (3 u) and an exact multiply by 0.25.

Every output array is filled with NaN canaries (a fixed payload) and has SLACK canaries after each tensor; the crop
window leaves one crop of the arrays outside it, and a window with no crop in it must write nothing.  A crop's result
must be bit-identical when it runs alone at position 0.  Inputs carry ~20 % exact zeros, one pixel row per crop spanning
1e-3 .. 1e3, negative-mean biases (the ReLU bites) and different gates per crop.  Each case prints its worst
error / bound ratio.
"""
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
CANARY = np.array([0x7FC0DEAD], np.uint32).view(np.float32)[0]
SLACK = 68                  # canaries after each tensor (a multiple of 4: branch tensors follow at float4 alignment)
CAP, OFF, COUNT = 4, 2, 5   # the window covers crops 0..2 of the 4 on the host (count - off = 3); crop 3 stays untouched
VALID = COUNT - OFF
EMPTY = (3, 2)              # (off, count) with no crop in the window

# (kind, C, W, R) of the LightConv launch each shipped float32 level shape gets: 1 generic k_lightconv, 2 k_lightconv2
LIGHT_SHAPES = {
    # osnet_x1_0 / ain_x1_0 / ibn_x1_0
    (64, 64, 32): (1, 64, 32, 1), (96, 32, 16): (2, 96, 16, 4), (128, 16, 8): (2, 128, 8, 8),
    # osnet_x0_75 / ain_x0_75
    (48, 64, 32): (1, 48, 32, 1), (72, 32, 16): (1, 72, 16, 4), (96, 16, 8): (1, 96, 8, 8),
    # osnet_x0_5 / ain_x0_5
    (32, 64, 32): (1, 32, 32, 4), (48, 32, 16): (1, 48, 16, 4), (64, 16, 8): (1, 64, 8, 8),
    # osnet_ain_x0_25 stage 2 (stages 3 and 4 run the chain kernel)
    (16, 64, 32): (2, 16, 32, 16),
    # LMBN_n trunk (96 x 32), trunk stage 3 and branch heads (48 x 16), branches after their transition (24 x 8)
    (64, 96, 32): (1, 64, 32, 1), (96, 48, 16): (2, 96, 16, 4), (128, 24, 8): (2, 128, 8, 8),
}
# (C, H, W) -> (3, C, W, R) of the whole-branch chain kernel (osnet_ain_x0_25 stages 3 and 4)
CHAIN_SHAPES = {(24, 32, 16): (3, 24, 16, 16), (32, 16, 8): (3, 32, 8, 16)}
OSNET_WIDTHS = {"x1_0": (64, 256, 384, 512), "x0_75": (48, 192, 288, 384), "x0_5": (32, 128, 192, 256),
                "x0_25": (16, 64, 96, 128)}


def _lib():
    from boxmot_b200 import _lib

    return _lib.require_device(), _lib


def _p(a):
    return None if a is None else a.ctypes.data


def _canvas(n):
    return np.full(n, CANARY, np.float32)


def _is_canary(a):
    return a.view(np.uint32) == CANARY.view(np.uint32)


def _call(fn, *args):
    lib, _l = _lib()
    ok = getattr(lib, fn)(*args)
    assert ok, _l.last_error(lib)


def _check(name, got, want, bound):
    got = np.asarray(got)
    assert np.isfinite(got).all(), f"{name}: non-finite output (an unwritten canary?)"
    err = np.abs(got.astype(np.float64) - want)
    ratio = float((err / np.maximum(bound, 1e-300)).max()) if err.size else 0.0
    print(f"{name}: worst error / bound = {ratio:.3g}")
    assert (err <= bound).all(), f"{name}: error / bound {ratio:.3g}"


def _act(rng, shape, nonneg=False, scale=1.0):
    """(n, h, w, c) float32: normal, ~20 % exact zeros, one pixel row per crop spanning 1e-3 .. 1e3."""
    n, h, w, c = shape
    x = rng.normal(size=shape) * scale
    if nonneg:
        x = np.abs(x)
    x[rng.random(shape) < 0.2] = 0.0
    for i in range(n):
        y = rng.integers(h)
        x[i, y] = np.sign(x[i, y]) * np.logspace(-3, 3, w * c).reshape(w, c)[:, rng.permutation(c)]
    return x.astype(np.float32)


def _weights(rng, k, n, scale=1.0):
    return (rng.normal(size=(k, n)) * scale / np.sqrt(k)).astype(np.float32)


def _bias(rng, n):
    return (rng.normal(size=n) * 0.5 - 0.2).astype(np.float32)


def _window_slices(per_crop, total):
    """Per-crop views of an output canvas of CAP crops, plus the slack after them."""
    return [slice(i * per_crop, (i + 1) * per_crop) for i in range(CAP)], slice(CAP * per_crop, total)


def _assert_untouched(name, canvas, per_crop, n_valid):
    crops, tail = _window_slices(per_crop, canvas.size)
    for i in range(n_valid, CAP):
        assert _is_canary(canvas[crops[i]]).all(), f"{name}: crop {i} outside the window was written"
    assert _is_canary(canvas[tail]).all(), f"{name}: the slack after the tensor was written"


# ---- float64 references ----------------------------------------------------------------------------------------------
def _dw(x, w9, bias=None, stride=1):
    """Depthwise 3x3 pad 1 of x (n, h, w, c) float64 with w9 (9, c)."""
    n, h, w, c = x.shape
    xp = np.zeros((n, h + 2, w + 2, c))
    xp[:, 1:-1, 1:-1] = x
    oh, ow = h // stride, w // stride
    out = np.zeros((n, oh, ow, c)) if bias is None else np.broadcast_to(bias.astype(np.float64), (n, oh, ow, c)).copy()
    for ky in range(3):
        for kx in range(3):
            out += xp[:, ky:ky + stride * oh:stride, kx:kx + stride * ow:stride] * w9[ky * 3 + kx].astype(np.float64)
    return out


def _light_ref(x, wpw, wdw, b, e_in=None):
    """One LightConv3x3 in float64 -> (y, error bound of the float32 kernel given an input error bound e_in)."""
    C = wpw.shape[0]
    x = x.astype(np.float64)
    t = x @ wpw.astype(np.float64)
    y = np.maximum(_dw(t, wdw, b), 0.0)
    aw, ad = np.abs(wpw.astype(np.float64)), np.abs(wdw.astype(np.float64))
    bound = (C + 12) * U * (_dw(np.abs(x) @ aw, ad) + np.abs(b.astype(np.float64)))
    if e_in is not None:
        bound += _dw(e_in @ aw, ad)
    return y, bound


def _tile_sums(y, R):
    n, H, W, C = y.shape
    s = y.astype(np.float64).reshape(n, H // R, R * W, C)
    return s.sum(axis=2), R * W * U * np.abs(s).sum(axis=2) + 1e-30


# ---- k_pointwise2 ----------------------------------------------------------------------------------------------------
# (name, hw, K, N, mid (gated; 0 = plain), residual, relu, weight scale)
PW_CASES = [
    ("conv1 x1_0 BN64", 37, 64, 64, 0, False, 1, 1.0),
    ("conv1 x0_25 BN16 K%16", 130, 44, 16, 0, False, 1, 1.0),
    ("transition x0_75 BN64", 37, 192, 192, 0, False, 1, 1.0),
    ("conv1 x0_75 BN32 N%32", 96, 192, 48, 0, False, 1, 1.0),
    ("conv1 x0_75 BN32 N=72", 37, 288, 72, 0, False, 1, 1.0),
    ("MobileNetV2 expand N=24 ReLU6", 130, 44, 24, 0, False, 2, 6.0),
    ("MobileNetV2 expand N=44 K=24 ReLU6", 96, 24, 44, 0, False, 2, 6.0),
    ("MobileNetV2 project N=136 residual", 37, 88, 136, 0, True, 0, 1.0),
    ("plain BN16 residual", 37, 32, 16, 0, True, 0, 1.0),
    ("gated x1_0 identity BN64", 37, 64, 256, 64, True, 1, 1.0),
    ("gated x1_0 downsample BN64", 37, 64 + 64, 256, 64, False, 1, 1.0),
    ("gated x0_75 downsample BN32", 96, 72 + 192, 288, 72, False, 1, 1.0),
    ("gated x0_25 downsample K%16 BN32", 130, 24 + 64, 96, 24, False, 1, 1.0),
    ("gated AIN conv3 BN64 no ReLU", 37, 48, 192, 48, False, 0, 1.0),
    ("gated BN16", 130, 16 + 16, 16, 16, False, 1, 1.0),
]


def _bn(N):
    return 64 if N % 64 == 0 else (32 if N % 32 == 0 or N > 16 else 16)


def _pw_operands(rng, hw, K, N, mid, residual, scale):
    if mid:
        br = np.stack([_act(rng, (CAP, hw, 1, mid), nonneg=True) for _ in range(4)])
        g = rng.uniform(0.0, 1.0, (CAP, 4, mid)).astype(np.float32)
        g[rng.random(g.shape) < 0.1] = 0.0
        a = _act(rng, (CAP, hw, 1, K - mid)) if K > mid else None
    else:
        br = g = None
        a = _act(rng, (CAP, hw, 1, K))
    w = _weights(rng, K, N, scale)
    b = _bias(rng, N)
    r = _act(rng, (CAP, hw, 1, N)) if residual else None
    return a, br, g, w, b, r


def _pw_ref(a, br, g, w, b, r, mid, relu):
    if mid:
        A = np.einsum("bnpk,nbk->npk", br[:, :, :, 0].astype(np.float64), g.astype(np.float64))
        Aabs = np.abs(A)
        extra = 4
        if a is not None:
            A = np.concatenate([A, a[:, :, 0].astype(np.float64)], axis=2)
            Aabs = np.concatenate([Aabs, np.abs(a[:, :, 0].astype(np.float64))], axis=2)
    else:
        A = a[:, :, 0].astype(np.float64)
        Aabs = np.abs(A)
        extra = 0
    K = A.shape[2]
    y = A @ w.astype(np.float64) + b
    mag = Aabs @ np.abs(w.astype(np.float64)) + np.abs(b.astype(np.float64))
    if r is not None:
        y = y + r[:, :, 0]
        mag = mag + np.abs(r[:, :, 0].astype(np.float64))
    if relu:
        y = np.maximum(y, 0.0)
    if relu == 2:
        y = np.minimum(y, 6.0)
    return y, (K + 3 + extra) * U * mag


def _pw_run(a, br, g, w, b, r, n, hw, K, N, mid, relu, off, count):
    out = _canvas(n * hw * N + SLACK)
    inst = np.zeros(4, np.int32)
    _call("boxmot_b200_f32_pointwise", _p(a), _p(br), _p(g), n, hw, K, mid, _p(w), N, _p(b), _p(r), relu, off, count,
          _p(out), out.size, _p(inst))
    return out, tuple(int(v) for v in inst)


@pytest.mark.parametrize("case", PW_CASES, ids=[c[0] for c in PW_CASES])
def test_pointwise_matches_float64(case):
    name, hw, K, N, mid, residual, relu, scale = case
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    a, br, g, w, b, r = _pw_operands(rng, hw, K, N, mid, residual, scale)
    want, bound = _pw_ref(a, br, g, w, b, r, mid, relu)
    out, inst = _pw_run(a, br, g, w, b, r, CAP, hw, K, N, mid, relu, OFF, COUNT)
    assert inst == (_bn(N), 128, int(mid > 0), 0), inst
    if relu == 2:
        assert (want >= 6.0).any() and (want <= 0.0).any(), "the ReLU6 case must clamp on both sides"
    per = hw * N
    _assert_untouched(name, out, per, VALID)
    got = out[:VALID * per].reshape(VALID, hw, N)
    _check(f"pointwise {name}", got, want[:VALID], bound[:VALID])
    empty, _ = _pw_run(a, br, g, w, b, r, CAP, hw, K, N, mid, relu, *EMPTY)
    assert _is_canary(empty).all(), "an empty window wrote output"
    for i in (1, VALID - 1):   # position independence: the crop alone at position 0, bit for bit
        sel = slice(i, i + 1)
        one, _ = _pw_run(None if a is None else a[sel].copy(), None if br is None else br[:, sel].copy(),
                         None if g is None else g[sel].copy(), w, b, None if r is None else r[sel].copy(),
                         1, hw, K, N, mid, relu, 0, 1)
        assert np.array_equal(one[:per].view(np.uint32), got[i].reshape(-1).view(np.uint32)), f"crop {i} alone differs"
        assert _is_canary(one[per:]).all()


# ---- LightConv3x3 level: k_lightconv / k_lightconv2 ------------------------------------------------------------------
def _light_run(x, wpw, wdw, b, nb, n, H, W, C, off, count, with_sums):
    ostride = n * H * W * C + SLACK
    sstride = n * H * C + SLACK
    out = _canvas(nb * ostride)
    sums = _canvas(nb * sstride) if with_sums else None
    inst = np.zeros(4, np.int32)
    _call("boxmot_b200_f32_lightconv", _p(x), nb, n, H, W, C, _p(wpw), _p(wdw), _p(b), off, count, _p(out), ostride,
          _p(sums), sstride, _p(inst))
    return out.reshape(nb, ostride), None if sums is None else sums.reshape(nb, sstride), tuple(int(v) for v in inst)


def _light_operands(rng, nb, H, W, C):
    x = np.stack([_act(rng, (CAP, H, W, C), nonneg=True) for _ in range(nb)])
    wpw = np.stack([_weights(rng, C, C) for _ in range(nb)])
    wdw = (rng.normal(size=(nb, 9, C)) / 3).astype(np.float32)
    b = np.stack([_bias(rng, C) for _ in range(nb)])
    return x, wpw, wdw, b


@pytest.mark.parametrize("shape", list(LIGHT_SHAPES), ids=[f"C{c}_{h}x{w}" for c, h, w in LIGHT_SHAPES])
def test_lightconv_level_matches_float64(shape):
    C, H, W = shape
    nb = 3
    rng = np.random.default_rng(C * 1000 + H)
    x, wpw, wdw, b = _light_operands(rng, nb, H, W, C)
    out, sums, inst = _light_run(x, wpw, wdw, b, nb, CAP, H, W, C, OFF, COUNT, True)
    assert inst == LIGHT_SHAPES[shape], inst
    R = inst[3]
    per, sper = H * W * C, (H // R) * C
    worst = 0.0
    for br in range(nb):
        want, bound = _light_ref(x[br, :VALID], wpw[br], wdw[br], b[br])
        _assert_untouched("lightconv out", out[br], per, VALID)
        _assert_untouched("lightconv sums", sums[br], sper, VALID)
        got = out[br, :VALID * per].reshape(VALID, H, W, C)
        _check(f"lightconv C{C} {H}x{W} R{R} branch {br}", got, want, bound)
        s_want, s_bound = _tile_sums(got, R)
        _check(f"lightconv sums C{C} {H}x{W} R{R} branch {br}", sums[br, :VALID * sper].reshape(VALID, H // R, C),
               s_want, s_bound)
        worst = max(worst, float(np.abs(got - want).max()))
    # one branch without sums: the same bits, nothing else written
    out1, none, inst1 = _light_run(x[1:2].copy(), wpw[1:2].copy(), wdw[1:2].copy(), b[1:2].copy(), 1, CAP, H, W, C,
                                   OFF, COUNT, False)
    assert inst1 == inst and none is None
    assert np.array_equal(out1[0].view(np.uint32), out[1].view(np.uint32))
    empty, esums, _ = _light_run(x, wpw, wdw, b, nb, CAP, H, W, C, *EMPTY, True)
    assert _is_canary(empty).all() and _is_canary(esums).all(), "an empty window wrote output"
    i = VALID - 1
    one, osums, _ = _light_run(x[:, i:i + 1].copy(), wpw, wdw, b, nb, 1, H, W, C, 0, 1, True)
    for br in range(nb):
        assert np.array_equal(one[br, :per].view(np.uint32), out[br, i * per:(i + 1) * per].view(np.uint32))
        assert np.array_equal(osums[br, :sper].view(np.uint32), sums[br, i * sper:(i + 1) * sper].view(np.uint32))


# ---- k_lightchain ----------------------------------------------------------------------------------------------------
def _chain_run(x, wpw, wdw, b, n, H, W, C, off, count):
    ostride, sstride = n * H * W * C + SLACK, n * H * C + SLACK
    out, sums = _canvas(4 * ostride), _canvas(4 * sstride)
    inst = np.zeros(4, np.int32)
    _call("boxmot_b200_f32_lightchain", _p(x), n, H, W, C, _p(wpw), _p(wdw), _p(b), off, count, _p(out), ostride,
          _p(sums), sstride, _p(inst))
    return out.reshape(4, ostride), sums.reshape(4, sstride), tuple(int(v) for v in inst)


@pytest.mark.parametrize("shape", list(CHAIN_SHAPES), ids=[f"C{c}_{h}x{w}" for c, h, w in CHAIN_SHAPES])
def test_lightchain_matches_float64(shape):
    C, H, W = shape
    rng = np.random.default_rng(7 * C + H)
    x = _act(rng, (CAP, H, W, C), nonneg=True)
    wpw = np.stack([_weights(rng, C, C) for _ in range(10)])
    wdw = (rng.normal(size=(10, 9, C)) / 3).astype(np.float32)
    b = np.stack([_bias(rng, C) for _ in range(10)])
    out, sums, inst = _chain_run(x, wpw, wdw, b, CAP, H, W, C, OFF, COUNT)
    assert inst == CHAIN_SHAPES[shape], inst
    R = inst[3]
    per, sper = H * W * C, (H // R) * C
    for br in range(4):
        y, e = x[:VALID], None
        for lv in range(br + 1):
            l = br * (br + 1) // 2 + lv
            y, e = _light_ref(y, wpw[l], wdw[l], b[l], e)
        _assert_untouched("chain out", out[br], per, VALID)
        _assert_untouched("chain sums", sums[br], sper, VALID)
        got = out[br, :VALID * per].reshape(VALID, H, W, C)
        _check(f"lightchain C{C} {H}x{W} branch {br} (depth {br + 1})", got, y, e)
        s_want, s_bound = _tile_sums(got, R)
        _check(f"lightchain sums C{C} branch {br}", sums[br, :VALID * sper].reshape(VALID, H // R, C), s_want, s_bound)
    empty, esums, _ = _chain_run(x, wpw, wdw, b, CAP, H, W, C, *EMPTY)
    assert _is_canary(empty).all() and _is_canary(esums).all(), "an empty window wrote output"
    i = VALID - 1
    one, osums, _ = _chain_run(x[i:i + 1].copy(), wpw, wdw, b, 1, H, W, C, 0, 1)
    for br in range(4):
        assert np.array_equal(one[br, :per].view(np.uint32), out[br, i * per:(i + 1) * per].view(np.uint32))
        assert np.array_equal(osums[br, :sper].view(np.uint32), sums[br, i * sper:(i + 1) * sper].view(np.uint32))


# ---- k_gates ---------------------------------------------------------------------------------------------------------
# (mid, hid, tiles, HW): every shipped OSBlock's ChannelGate (hid = mid / 16), tile counts of its LightConv launch
GATE_CASES = [(16, 1, 4, 2048), (24, 1, 2, 512), (32, 2, 1, 128), (32, 2, 16, 2048), (48, 3, 64, 2048),
              (48, 3, 8, 512), (64, 4, 64, 2048), (64, 4, 96, 3072), (72, 4, 8, 512), (96, 6, 8, 512),
              (96, 6, 2, 128), (128, 8, 2, 128), (128, 8, 3, 192)]


def _gates_run(s, n, tiles, C, hid, hw, w1, b1, w2, b2, off, count):
    out = _canvas(n * 4 * C + SLACK)
    _call("boxmot_b200_f32_gates", _p(s), n, tiles, C, hid, hw, _p(w1), _p(b1), _p(w2), _p(b2), off, count, _p(out),
          out.size)
    return out


@pytest.mark.parametrize("case", GATE_CASES, ids=[f"mid{c[0]}_hid{c[1]}_tiles{c[2]}" for c in GATE_CASES])
def test_gates_match_float64(case):
    C, hid, tiles, hw = case
    rng = np.random.default_rng(C * 100 + tiles)
    s = (np.abs(rng.normal(size=(4, CAP, tiles, C))) * hw / tiles).astype(np.float32)
    s[rng.random(s.shape) < 0.2] = 0.0
    w1 = _weights(rng, C, hid, 3.0)
    b1 = _bias(rng, hid)
    w2 = _weights(rng, hid, C, 3.0)
    b2 = _bias(rng, C)
    out = _gates_run(s, CAP, tiles, C, hid, hw, w1, b1, w2, b2, OFF, COUNT)
    s64 = s[:, :VALID].astype(np.float64)
    mean = s64.sum(axis=2) / hw                                          # (4, n, C)
    e_mean = (tiles + 1) * U * np.abs(s64).sum(axis=2) / hw
    aw1, aw2 = np.abs(w1.astype(np.float64)), np.abs(w2.astype(np.float64))
    h = mean @ w1 + b1
    e_h = (C + 2) * U * (np.abs(mean) @ aw1 + np.abs(b1)) + e_mean @ aw1
    h = np.maximum(h, 0.0)
    z = h @ w2 + b2
    e_z = (hid + 2) * U * (np.abs(h) @ aw2 + np.abs(b2)) + e_h @ aw2
    want = 1.0 / (1.0 + np.exp(-z))
    bound = 0.25 * e_z + 4 * U
    _assert_untouched("gates", out, 4 * C, VALID)
    got = out[:VALID * 4 * C].reshape(VALID, 4, C)
    _check(f"gates mid {C} hid {hid} tiles {tiles}", got, want.transpose(1, 0, 2), bound.transpose(1, 0, 2))
    assert _is_canary(_gates_run(s, CAP, tiles, C, hid, hw, w1, b1, w2, b2, *EMPTY)).all()
    i = VALID - 1
    one = _gates_run(s[:, i:i + 1].copy(), 1, tiles, C, hid, hw, w1, b1, w2, b2, 0, 1)
    assert np.array_equal(one[:4 * C].view(np.uint32), got[i].reshape(-1).view(np.uint32))


# ---- k_head ----------------------------------------------------------------------------------------------------------
# (name, C, HW, feat, fc): OSNet x1_0 (C >= 256 threads), OSNet x0_25 (two thread groups per channel), MobileNetV2_x1_4
# and ResNet (C > blockDim: the pool re-reads the map)
HEAD_CASES = [("osnet_x1_0", 512, 128, 512, True), ("osnet_x0_25", 128, 128, 512, True),
              ("osnet_x0_75", 384, 128, 512, True), ("mobilenetv2_x1_4", 1792, 32, 1792, False),
              ("resnet50", 2048, 128, 2048, False)]
ROWS = np.array([6, 0, 4, 2, 8, 1, 3], np.int32)   # output row of crop off + i (off + n <= 7): scattered, not in order
N_ROWS = 9


def _head_run(x, n, hw, C, wfc, bfc, feat, rows, off, count, ld):
    out = _canvas(N_ROWS * ld + SLACK)
    _call("boxmot_b200_f32_head", _p(x), n, hw, C, _p(wfc), _p(bfc), feat, _p(rows), off, count, _p(out), out.size, ld)
    return out


def _l2_bound(s, e_s, feat):
    nrm = np.linalg.norm(s, axis=-1, keepdims=True)
    y = s / nrm
    return y, e_s / nrm + np.abs(y) * (np.linalg.norm(e_s, axis=-1, keepdims=True) / nrm + (feat / 2 + 3) * U)


@pytest.mark.parametrize("case", HEAD_CASES, ids=[c[0] for c in HEAD_CASES])
def test_head_matches_float64(case):
    name, C, hw, feat, fc = case
    rng = np.random.default_rng(C + hw)
    x = _act(rng, (CAP, hw, 1, C), nonneg=True)[:, :, 0]
    wfc = _weights(rng, C, feat) if fc else None
    bfc = _bias(rng, feat) if fc else None
    ld = feat + 13
    rows = ROWS.copy()
    out = _head_run(x, CAP, hw, C, wfc, bfc, feat, rows, OFF, COUNT, ld)
    x64 = x[:VALID].astype(np.float64)
    pooled = x64.mean(axis=1)
    e_p = (hw + 1) * U * np.abs(x64).mean(axis=1)
    if fc:
        aw = np.abs(wfc.astype(np.float64))
        s = pooled @ wfc + bfc
        e_s = (C + 5) * U * (np.abs(pooled) @ aw + np.abs(bfc)) + e_p @ aw
        s = np.maximum(s, 0.0)
    else:
        s, e_s = pooled, e_p
    want, bound = _l2_bound(s, e_s, feat)
    mat = out[:N_ROWS * ld].reshape(N_ROWS, ld)
    written = set(int(r) for r in rows[OFF:OFF + VALID])
    for r in range(N_ROWS):
        if r not in written:
            assert _is_canary(mat[r]).all(), f"row {r} belongs to no crop in the window but was written"
        else:
            assert _is_canary(mat[r, feat:]).all(), f"row {r}: written past feat"
    assert _is_canary(out[N_ROWS * ld:]).all()
    got = np.stack([mat[rows[OFF + i], :feat] for i in range(VALID)])
    _check(f"head {name}", got, want, bound)
    assert _is_canary(_head_run(x, CAP, hw, C, wfc, bfc, feat, rows, *EMPTY, ld)).all()
    i = VALID - 1
    one_rows = np.array([rows[OFF + i]], np.int32)
    one = _head_run(x[i:i + 1].copy(), 1, hw, C, wfc, bfc, feat, one_rows, 0, 1, ld)
    assert np.array_equal(one[:N_ROWS * ld].reshape(N_ROWS, ld)[one_rows[0], :feat].view(np.uint32),
                          got[i].view(np.uint32))


# ---- stems, pools, MobileNetV2 depthwise -----------------------------------------------------------------------------
def _conv_ref(x, w, b, k, stride, cin):
    """k x k pad k // 2 (7x7 pad 3, 3x3 pad 1) convolution of x (n, h, w, cin) float64, w (k*k*cin, C)."""
    n, h, wd, _ = x.shape
    p = k // 2
    xp = np.zeros((n, h + 2 * p, wd + 2 * p, cin))
    xp[:, p:p + h, p:p + wd] = x
    oh, ow = h // stride, wd // stride
    C = w.shape[1]
    out = np.zeros((n, oh, ow, C))
    mag = np.zeros((n, oh, ow, C))
    w64 = w.astype(np.float64).reshape(k, k, cin, C)
    for ky in range(k):
        for kx in range(k):
            patch = xp[:, ky:ky + stride * oh:stride, kx:kx + stride * ow:stride]
            out += patch @ w64[ky, kx]
            mag += np.abs(patch) @ np.abs(w64[ky, kx])
    if b is not None:
        out += b
        mag += np.abs(b.astype(np.float64))
    return out, (k * k * cin + 2) * U * mag


def _map_run(op, x, n, h, w, c, stride, weight, bias, off, count, per):
    out = _canvas(n * per + SLACK)
    _call("boxmot_b200_f32_map", op, _p(x), n, h, w, c, stride, _p(weight), _p(bias), off, count, _p(out), out.size)
    return out


# (name, op, h, w, c, stride)
MAP_CASES = ([(f"stem C{c} h{h}", 0, h, 128, c, 2) for c in (16, 32, 48, 64) for h in (256, 384)] +
             [("stem IN C64", 1, 256, 128, 64, 2), ("stem IN C16", 1, 256, 128, 16, 2), ("stem IN C32 h384", 1, 384, 128, 32, 2)] +
             [(f"maxpool C{c} h{h}", 2, h, 64, c, 2) for c, h in ((16, 128), (48, 128), (64, 192))] +
             [("avgpool C256 64x32", 3, 64, 32, 256, 2), ("avgpool C72 32x16", 3, 32, 16, 72, 2),
              ("avgpool C384 48x16", 3, 48, 16, 384, 2)] +
             [("stem3 C44", 4, 256, 128, 44, 2)] +
             [("dwconv C44 s1", 5, 128, 64, 44, 1), ("dwconv C132 s2", 5, 128, 64, 132, 2),
              ("dwconv C200 s2", 5, 64, 32, 200, 2), ("dwconv C536 s1", 5, 16, 8, 536, 1),
              ("dwconv C1344 s1", 5, 8, 4, 1344, 1)])


@pytest.mark.parametrize("case", MAP_CASES, ids=[c[0] for c in MAP_CASES])
def test_stems_pools_depthwise_match_float64(case):
    name, op, h, w, c, stride = case
    rng = np.random.default_rng(op * 1000 + c + h)
    cin = 3 if op in (0, 1, 4) else c
    x = _act(rng, (CAP, h, w, cin), nonneg=op in (2, 3), scale=2.0 if op in (4, 5) else 1.0)
    weight = bias = None
    if op in (0, 1):
        weight = _weights(rng, 147, c, 2.0)
        bias = _bias(rng, c)
    elif op == 4:
        weight = _weights(rng, 27, c, 4.0)
        bias = _bias(rng, c)
    elif op == 5:
        weight = (rng.normal(size=(9, c)) * 1.5).astype(np.float32)
        bias = _bias(rng, c)
    x64 = x[:VALID].astype(np.float64)
    if op in (0, 1):
        want, bound = _conv_ref(x64, weight, None if op == 1 else bias, 7, 2, 3)
        if op == 0:
            want = np.maximum(want, 0.0)
    elif op == 4:
        want, bound = _conv_ref(x64, weight, bias, 3, 2, 3)
    elif op == 5:
        want = _dw(x64, weight, bias, stride)
        bound = 11 * U * (_dw(np.abs(x64), np.abs(weight.astype(np.float64)), np.abs(bias), stride))
    elif op == 2:
        xp = np.full((VALID, h + 2, w + 2, c), -np.inf)
        xp[:, 1:-1, 1:-1] = x64
        want = np.max([xp[:, ky:ky + h:2, kx:kx + w:2] for ky in range(3) for kx in range(3)], axis=0)
        bound = np.zeros_like(want)
    else:
        q = x64.reshape(VALID, h // 2, 2, w // 2, 2, c)
        want = q.mean(axis=(2, 4))
        bound = 3 * U * np.abs(q).sum(axis=(2, 4)) * 0.25
    if op in (4, 5):
        want = np.clip(want, 0.0, 6.0)
        assert (want == 6.0).any() and (want == 0.0).any(), "ReLU6 must clamp on both sides"
    oh, ow = want.shape[1:3]
    per = oh * ow * c
    out = _map_run(op, x, CAP, h, w, c, stride, weight, bias, OFF, COUNT, per)
    _assert_untouched(name, out, per, VALID)
    got = out[:VALID * per].reshape(VALID, oh, ow, c)
    _check(f"{name}", got, want, bound)
    assert _is_canary(_map_run(op, x, CAP, h, w, c, stride, weight, bias, *EMPTY, per)).all()
    i = VALID - 1
    one = _map_run(op, x[i:i + 1].copy(), 1, h, w, c, stride, weight, bias, 0, 1, per)
    assert np.array_equal(one[:per].view(np.uint32), got[i].reshape(-1).view(np.uint32))


# ---- LMBN_n head: k_lmbn_pool, k_lmbn_neck, k_l2_normalise ------------------------------------------------------------
def test_lmbn_head_matches_float64():
    C, h, w = 512, 24, 8
    rng = np.random.default_rng(512)
    x = np.stack([_act(rng, (CAP, h, w, C), nonneg=True) for _ in range(3)])
    neck = [_weights(rng, C, C) for _ in range(5)] + [_bias(rng, C) for _ in range(5)]
    wsh, bsh = _weights(rng, C // 2, C), _bias(rng, C)
    chst = np.concatenate([rng.uniform(0.5, 1.5, C), rng.normal(size=C), rng.uniform(0.5, 1.5, C),
                           rng.normal(size=C)]).astype(np.float32)
    blob = np.concatenate([a.reshape(-1) for a in neck] + [wsh.reshape(-1), bsh, chst]).astype(np.float32)
    ld, feat = 7 * C + 5, 7 * C
    rows = ROWS.copy()

    def run(xx, n, rr, off, count):
        pooled, out = _canvas(n * 6 * C + SLACK), _canvas(N_ROWS * ld + SLACK)
        _call("boxmot_b200_f32_lmbn_head", _p(xx), n, h, w, _p(blob), _p(rr), off, count, _p(pooled), pooled.size,
              _p(out), out.size, ld)
        return pooled, out

    pooled, out = run(x, CAP, rows, OFF, COUNT)
    # poolings against float64
    x64 = x[:, :VALID].astype(np.float64).reshape(3, VALID, h * w, C)
    half = (h // 2) * w
    top, bot = x64[:, :, :half], x64[:, :, half:]
    pw = np.zeros((VALID, 6, C))
    pb = np.zeros((VALID, 6, C))
    pw[:, 0], pb[:, 0] = x64[0].mean(axis=1), (h * w + 1) * U * x64[0].mean(axis=1)
    pw[:, 1] = x64[0].max(axis=1)
    pw[:, 2] = x64[1].max(axis=1)
    pw[:, 3], pb[:, 3] = top[1].mean(axis=1), (half + 1) * U * top[1].mean(axis=1)
    pw[:, 4], pb[:, 4] = bot[1].mean(axis=1), (half + 1) * U * bot[1].mean(axis=1)
    pw[:, 5], pb[:, 5] = x64[2].mean(axis=1), (h * w + 1) * U * x64[2].mean(axis=1)
    _assert_untouched("lmbn pooled", pooled, 6 * C, VALID)
    gp = pooled[:VALID * 6 * C].reshape(VALID, 6, C)
    _check("lmbn pools", gp, pw, pb)
    # neck + L2 norm on the kernel's own pooled rows
    p64 = gp.astype(np.float64)
    vec = np.zeros((VALID, C, 7))
    err = np.zeros((VALID, C, 7))
    for k in range(5):
        aw = np.abs(neck[k].astype(np.float64))
        vec[:, :, k] = p64[:, k] @ neck[k] + neck[5 + k]
        err[:, :, k] = (C + 4) * U * (np.abs(p64[:, k]) @ aw + np.abs(neck[5 + k]))
    for hh in range(2):
        src = p64[:, 5, hh * (C // 2):(hh + 1) * (C // 2)]
        z = src @ wsh + bsh
        e_z = (C // 2 + 4) * U * (np.abs(src) @ np.abs(wsh.astype(np.float64)) + np.abs(bsh))
        sc, sh = chst[2 * hh * C:(2 * hh + 1) * C].astype(np.float64), chst[(2 * hh + 1) * C:(2 * hh + 2) * C]
        vec[:, :, 5 + hh] = np.maximum(z, 0.0) * sc + sh
        err[:, :, 5 + hh] = e_z * np.abs(sc) + 2 * U * (np.abs(np.maximum(z, 0.0) * sc) + np.abs(sh))
    want, bound = _l2_bound(vec.reshape(VALID, feat), err.reshape(VALID, feat), feat)
    mat = out[:N_ROWS * ld].reshape(N_ROWS, ld)
    written = set(int(r) for r in rows[OFF:OFF + VALID])
    for r in range(N_ROWS):
        if r not in written:
            assert _is_canary(mat[r]).all(), f"row {r} belongs to no crop in the window but was written"
        else:
            assert _is_canary(mat[r, feat:]).all()
    assert _is_canary(out[N_ROWS * ld:]).all()
    got = np.stack([mat[rows[OFF + i], :feat] for i in range(VALID)])
    _check("lmbn neck + L2", got, want, bound)
    ep, eo = run(x, CAP, rows, *EMPTY)
    assert _is_canary(ep).all() and _is_canary(eo).all()
    i = VALID - 1
    one_rows = np.array([rows[OFF + i]], np.int32)
    op_, oo = run(x[:, i:i + 1].copy(), 1, one_rows, 0, 1)
    assert np.array_equal(op_[:6 * C].view(np.uint32), gp[i].reshape(-1).view(np.uint32))
    assert np.array_equal(oo[:N_ROWS * ld].reshape(N_ROWS, ld)[one_rows[0], :feat].view(np.uint32), got[i].view(np.uint32))


# ---- coverage: every shipped float32 model's layers land on an instance tested above ---------------------------------
def _osnet_pointwise_layers(c):
    """(K, N, gated mid) of every 1x1 GEMM of an OSNet / OSNet-AIN / OSNet-IBN of stage widths c."""
    layers = []
    for s in range(3):
        for j in range(2):
            cin, cout = (c[s] if j == 0 else c[s + 1]), c[s + 1]
            mid = cout // 4
            layers.append((cin, mid, 0))
            layers.append((mid + (cin if cin != cout else 0), cout, mid))   # OSNet / IBN conv3 (+ downsample)
            layers.append((mid, cout, mid))                                  # AIN conv3 alone
            if cin != cout:
                layers.append((cin, cout, 0))                                # AIN downsample alone
        if s < 2:
            layers.append((c[s + 1], c[s + 1], 0))
    layers.append((c[3], c[3], 0))
    return layers


def _lmbn_pointwise_layers():
    layers = []
    for cin, cout in ((64, 256), (256, 256), (256, 384), (384, 384), (384, 512), (512, 512)):
        mid = cout // 4
        layers += [(cin, mid, 0), (mid + (cin if cin != cout else 0), cout, mid)]
    return layers + [(256, 256, 0), (384, 384, 0), (512, 512, 0)]


def _mobilenetv2_pointwise_layers():
    from boxmot_b200.synthetic import mobilenetv2_blocks

    p4 = lambda v: (v + 3) // 4 * 4
    _, blocks, feat = mobilenetv2_blocks(1.4)
    layers = []
    for cin, cout, t, _s in blocks:
        layers += [(p4(cin), p4(cin * t), 0), (p4(cin * t), p4(cout), 0)]
    return layers + [(p4(blocks[-1][1]), feat, 0)]


def test_shipped_shapes_land_on_tested_instances():
    """Every 1x1 GEMM and LightConv level of osnet_x1_0 / _x0_75 / _x0_5, OSNet-AIN / IBN (x0_25 included), LMBN_n and
    MobileNetV2_x1_4 goes through the dispatch; the instances they reach must be ones the tests above check, and
    together they must reach the generic and the shape-specialised LightConv, both chain instances and every pointwise
    tile width."""
    tested_pw = {(_bn(N), 128, int(mid > 0), 0) for _n, _hw, _K, N, mid, *_ in PW_CASES}
    reached_pw = {}
    layers = {f"osnet_{k}": _osnet_pointwise_layers(v) for k, v in OSNET_WIDTHS.items()}
    layers["lmbn_n"] = _lmbn_pointwise_layers()
    layers["mobilenetv2_x1_4"] = _mobilenetv2_pointwise_layers()
    rng = np.random.default_rng(0)
    hw = 3
    for model, ls in layers.items():
        for K, N, mid in sorted(set(ls)):
            a, br, g, w, b, r = _pw_operands(rng, hw, K, N, mid, False, 1.0)
            _, inst = _pw_run(a[:1].copy() if a is not None else None, None if br is None else br[:, :1].copy(),
                              None if g is None else g[:1].copy(), w, b, None, 1, hw, K, N, mid, 1, 0, 1)
            reached_pw.setdefault(inst, []).append((model, K, N, mid))
    untested = {i: v for i, v in reached_pw.items() if i not in tested_pw}
    assert not untested, f"pointwise instances reached by shipped models but not tested: {untested}"
    assert {i[0] for i in reached_pw} == {16, 32, 64} and {i[2] for i in reached_pw} == {0, 1}
    print("pointwise instances reached:", sorted(reached_pw))
    reached_light = set()
    for C, H, W in LIGHT_SHAPES:
        x, wpw, wdw, b = _light_operands(rng, 1, H, W, C)
        _, _, inst = _light_run(x[:, :1].copy(), wpw, wdw, b, 1, 1, H, W, C, 0, 1, True)
        assert inst == LIGHT_SHAPES[(C, H, W)], ((C, H, W), inst)
        reached_light.add(inst)
    for C, H, W in CHAIN_SHAPES:
        x = _act(rng, (1, H, W, C), nonneg=True)
        wpw = np.stack([_weights(rng, C, C) for _ in range(10)])
        wdw = (rng.normal(size=(10, 9, C)) / 3).astype(np.float32)
        b = np.stack([_bias(rng, C) for _ in range(10)])
        _, _, inst = _chain_run(x, wpw, wdw, b, 1, H, W, C, 0, 1)
        assert inst == CHAIN_SHAPES[(C, H, W)]
        reached_light.add(inst)
    assert {i[0] for i in reached_light} == {1, 2, 3}
    # every OSNet-family stage shape is one of the tested level or chain shapes
    for c in OSNET_WIDTHS.values():
        for s, (H, W) in enumerate(((64, 32), (32, 16), (16, 8))):
            shape = (c[s + 1] // 4, H, W)
            assert shape in LIGHT_SHAPES or shape in CHAIN_SHAPES, shape
    print("LightConv instances reached:", sorted(reached_light))
