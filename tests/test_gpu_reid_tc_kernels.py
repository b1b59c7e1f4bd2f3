"""Every tensor-core OSNet_x0_25 kernel on its own (tests/tcsim.py launches them with the product's packing), against a
float64 reference at bounds derived from the split-BF16 error model (tests/tcsim.py header):

- k_gemm_tc: all 13 instances at the shapes the plan launches, every ring depth that fits shared memory, every ring chunk
  that divides a source, tile groupings that do and do not divide the crop's tiles.  The MMA order does not depend on
  these, so every configuration of an instance must be bit-identical; one is checked against the decoded-operand and
  the plain-float32 references.  Crop windows, canaries around every output, the identity shortcut exact.
- k_chain_tc: the three stage shapes, all four branches, channel sums, gates and the gate (x) conv3 fold; back-to-back
  launches reset their arrival counters.
- Through B200ReID: embeddings are bitwise invariant to batch position, batch size and chunking; edge boxes through
  the fused front kernel.
"""
import itertools

import numpy as np
import pytest

from tests import tcsim
from tests.tcsim import GM_HEAD, GM_PLAIN, GM_POOL, GM_TAIL, GM_TAIL_POOL2

pytestmark = pytest.mark.gpu

CAP = 5
REPORT = {}

# (NP, NP2, mode) -> launches of the OSNet_x0_25 plan: (name, H, W, source C8s, midp, N, N2, identity shortcut)
SHAPES = {
    (16, 0, GM_PLAIN): [("conv1 block 0", 64, 32, [2], 0, 16, None, False)],
    (32, 0, GM_PLAIN): [("conv1 block 2", 32, 16, [8], 0, 24, None, False), ("conv1 block 4", 16, 8, [12], 0, 32, None, False)],
    (64, 0, GM_PLAIN): [("combine block 1", 64, 32, [8, 8], 16, 64, None, True)],
    (96, 0, GM_PLAIN): [("combine block 3", 32, 16, [16, 12], 32, 96, None, True)],
    (128, 0, GM_PLAIN): [("combine block 5", 16, 8, [16, 16], 32, 128, None, True), ("conv5", 16, 8, [16], 0, 128, None, False)],
    (64, 0, GM_POOL): [("transition 2", 64, 32, [8], 0, 64, None, False)],
    (96, 0, GM_POOL): [("transition 3", 32, 16, [12], 0, 96, None, False)],
    (64, 16, GM_TAIL): [("combine block 0 + conv1", 64, 32, [8, 2], 16, 64, 16, False)],
    (96, 32, GM_TAIL): [("combine block 2 + conv1", 32, 16, [16, 8], 32, 96, 24, False)],
    (128, 32, GM_TAIL): [("combine block 4 + conv1", 16, 8, [16, 12], 32, 128, 32, False)],
    (64, 64, GM_TAIL_POOL2): [("combine block 1 + transition", 64, 32, [8, 8], 16, 64, 64, True)],
    (96, 96, GM_TAIL_POOL2): [("combine block 3 + transition", 32, 16, [16, 12], 32, 96, 96, True)],
    (128, 0, GM_HEAD): [("conv5 + head", 16, 8, [16], 0, 128, None, False)],
}


def _plan_tpc(HW):
    t = HW // 128
    return 4 if t >= 16 else (2 if t >= 4 else 1)


def _configs(c8s, HW):
    kcs = [[k for k in (2, 4, 8) if c % k == 0] for c in c8s]
    tpcs = sorted({1, _plan_tpc(HW)} | ({3} if HW == 2048 else set()))
    for ns, kc, tpc in itertools.product((2, 3, 4), itertools.product(*kcs), tpcs):
        yield ns, list(kc), tpc


def _operands(seed, cap, H, W, c8s, midp, N, N2, identity, NP, NP2):
    rng = np.random.default_rng(seed)
    HW = H * W
    a = [tcsim.activations(rng, cap, HW, 8 * c, nonneg=(s == 1 or midp == 0 and N == 128)) for s, c in enumerate(c8s)]
    K = 8 * sum(c8s)
    w = tcsim.weights(rng, K, N)
    wfold = None
    if midp:
        # a different gate set per crop (a wrong crop index shows), the unused rows of B hold a huge value the kernel must
        # never read
        wfold = np.stack([tcsim.weights(rng, 4 * midp, N) * rng.uniform(0.1, 2.0) for _ in range(cap)])
        wfold[:, rng.random(4 * midp) < 0.15] = 0.0
        w[:4 * midp] = 3.0e4
        if identity:
            w[4 * midp:] = np.eye(K - 4 * midp, N, dtype=np.float32)
    bias = np.zeros(NP, np.float32)
    bias[:N] = rng.normal(size=N) * 0.5 - 0.3          # negative biases: the ReLU edge
    w2 = b2 = None
    if N2:
        w2 = np.zeros((NP, N2), np.float32)
        w2[:N] = tcsim.weights(rng, N, N2)
        b2 = np.zeros(NP2, np.float32)
        b2[:N2] = rng.normal(size=N2) * 0.3 - 0.1
    return a, w, wfold, bias, w2, b2


def _b_full(w, wfold, midp, n):
    """The B operand crop n multiplies: the crop's folded rows, then the shared rows."""
    if not midp:
        return w
    b = w.copy()
    b[:4 * midp] = wfold[n]
    return b


def _planes_out(res, key, cap, C8, HW):
    hi = res[key + "_hi"][:cap * C8 * HW * 8].reshape(cap, C8, HW, 8)
    lo = res[key + "_lo"][:cap * C8 * HW * 8].reshape(cap, C8, HW, 8)
    return hi, lo


def _check_canaries(res, key, n_valid, cap, C8, HW):
    hi, lo = _planes_out(res, key, cap, C8, HW)
    for p in (hi, lo):
        assert (p[n_valid:] == tcsim.BF16_CANARY).all(), f"{key}: written outside the valid crops"
    for k in (key + "_hi", key + "_lo"):
        assert (res[k][cap * C8 * HW * 8:] == tcsim.BF16_CANARY).all(), f"{key}: written past the tensor"


def _ratio(err, bound, what):
    r = float((err / bound).max())
    assert r <= 1.0, f"{what}: error {float(err.max()):.3e} exceeds its bound (worst error / bound {r:.3f})"
    return r


def _gemm_ref(a, w, wfold, bias, midp, N, NP, n):
    """float64 references of crop n: (decoded-operand ref, S, drops, plain ref, S32), columns 0..N-1."""
    A = np.concatenate([x[n] for x in a], axis=1)
    return tcsim.gemm_terms(A, _b_full(w, wfold, midp, n), bias[:N])


def _check_gemm(key, name, res, ops, H, W, c8s, midp, N, N2, NP, NP2, n_valid, cap, inter=None):
    """Compare one launch's outputs with the references; returns the worst error / bound ratio and the drop ratio."""
    a, w, wfold, bias, w2, b2 = ops
    mode = key[2]
    HW, K = H * W, 8 * sum(c8s)
    worst, drop = 0.0, np.inf
    for n in range(n_valid):
        ref, S, drops, ref32, S32 = _gemm_ref(a, w, wfold, bias, midp, N, NP, n)
        pre_b = tcsim.acc_bound(S, K)
        if mode in (GM_PLAIN, GM_TAIL):
            if res.get("out_f32") is not None:
                got = res["out_f32"][n * HW * N:(n + 1) * HW * N].reshape(HW, N).astype(np.float64)
                b = tcsim.out_bound(tcsim.relu(ref), S, K, split_out=False)
            else:
                hi, lo = _planes_out(res, "out", cap, NP // 8, HW)
                dh, dl = tcsim.from_planes(hi[n:n + 1], lo[n:n + 1])
                full = (dh + dl)[0]
                assert not full[:, N:].any(), f"{name}: padded output channels must be exact zeros"
                got = full[:, :N]
                b = tcsim.out_bound(tcsim.relu(ref), S, K)
            worst = max(worst, _ratio(np.abs(got - tcsim.relu(ref)), b, f"{name} crop {n} vs decoded operands"))
            worst = max(worst, _ratio(np.abs(got - tcsim.relu(ref32)), b + tcsim.plain_bound(S32), f"{name} crop {n} vs float32 math"))
            drop = min(drop, tcsim.drop_ratio(drops[1:], b))
            if mode == GM_TAIL:
                t = got                                      # the intermediate the tail read: these very planes
                r2, S2, d2, r2_32, S2_32 = tcsim.gemm_terms(t.astype(np.float32), w2[:N], b2[:N2])
                assert np.array_equal(t.astype(np.float32).astype(np.float64), t), "tail input is float32-exact"
                hi2, lo2 = _planes_out(res, "out2", cap, NP2 // 8, HW)
                d2h, d2l = tcsim.from_planes(hi2[n:n + 1], lo2[n:n + 1])
                g2 = (d2h + d2l)[0]
                assert not g2[:, N2:].any(), f"{name}: padded tail channels must be exact zeros"
                b2_ = tcsim.out_bound(tcsim.relu(r2), S2, NP)
                worst = max(worst, _ratio(np.abs(g2[:, :N2] - tcsim.relu(r2)), b2_, f"{name} crop {n} tail"))
                worst = max(worst, _ratio(np.abs(g2[:, :N2] - tcsim.relu(r2_32)), b2_ + tcsim.plain_bound(S2_32),
                                          f"{name} crop {n} tail vs float32 math"))
                drop = min(drop, tcsim.drop_ratio(d2[1:], b2_))
        elif mode == GM_POOL:
            hi, lo = _planes_out(res, "out", cap, NP // 8, HW // 4)
            dh, dl = tcsim.from_planes(hi[n:n + 1], lo[n:n + 1])
            got = (dh + dl)[0][:, :N]
            pre = tcsim.relu(ref)[None]
            want = tcsim.pool2x2(pre, H, W)[0]
            b = tcsim.pool2x2(pre_b[None] + 2.0 ** -21 * np.abs(pre), H, W)[0] + 2.0 ** -16 * np.abs(want)
            worst = max(worst, _ratio(np.abs(got - want), b, f"{name} crop {n} pooled"))
            want32 = tcsim.pool2x2(tcsim.relu(ref32)[None], H, W)[0]
            worst = max(worst, _ratio(np.abs(got - want32), b + tcsim.pool2x2(tcsim.plain_bound(S32)[None], H, W)[0],
                                      f"{name} crop {n} pooled vs float32 math"))
            drop = min(drop, min(float((np.abs(tcsim.pool2x2(d[None], H, W)[0]) / b).max()) for d in drops[1:]))
        elif mode == GM_TAIL_POOL2:
            # the block output is never written: take it from the plain instance of the same width, whose main loop
            # is the same code
            t = inter[n]
            r2, S2, d2, r2_32, S2_32 = tcsim.gemm_terms(t.astype(np.float32), w2[:N], b2[:N2])
            hi2, lo2 = _planes_out(res, "out2", cap, NP2 // 8, HW // 4)
            d2h, d2l = tcsim.from_planes(hi2[n:n + 1], lo2[n:n + 1])
            got = (d2h + d2l)[0]
            pre = tcsim.relu(r2)[None]
            want = tcsim.pool2x2(pre, H, W)[0]
            b = tcsim.pool2x2(tcsim.acc_bound(S2, NP)[None] + 2.0 ** -21 * np.abs(pre), H, W)[0] + 2.0 ** -16 * np.abs(want)
            worst = max(worst, _ratio(np.abs(got[:, :N2] - want), b, f"{name} crop {n} pooled tail"))
            want32 = tcsim.pool2x2(tcsim.relu(r2_32)[None], H, W)[0]
            worst = max(worst, _ratio(np.abs(got[:, :N2] - want32), b + tcsim.pool2x2(tcsim.plain_bound(S2_32)[None], H, W)[0],
                                      f"{name} crop {n} pooled tail vs float32 math"))
            drop = min(drop, min(float((np.abs(tcsim.pool2x2(d[None], H, W)[0]) / b).max()) for d in d2[1:]))
    return worst, drop


@pytest.mark.parametrize("key", list(SHAPES), ids=lambda k: f"np{k[0]}_np2{k[1]}_{tcsim.MODE_NAMES[k[2]]}")
def test_gemm_instance_every_config(key):
    NP, NP2, mode = key
    limit = tcsim.lib().tcsim_smem_limit()
    assert limit > 0, tcsim.lib().tcsim_last_error()
    ran, skipped, worst_all, drop_all = [], [], 0.0, np.inf
    for si, (name, H, W, c8s, midp, N, N2, identity) in enumerate(SHAPES[key]):
        HW = H * W
        ops = _operands(1000 * NP + 10 * mode + si, CAP, H, W, c8s, midp, N, N2, identity, NP, NP2)
        a, w, wfold, bias, w2, b2 = ops
        out_f32 = mode == GM_PLAIN and name == "conv5"
        head = dict(head_w=None)
        if mode == GM_HEAD:
            rng = np.random.default_rng(5)
            head = dict(head_w=tcsim.weights(rng, N, 512), head_b=(rng.normal(size=512) * 0.1).astype(np.float32),
                        out_row=np.array([6, 2, 0, 4, 1], np.int32), out_ld=520, out_rows=8)
        first = None
        for ns, kc, tpc in _configs(c8s, HW):
            cfg = f"{name}: n_stage {ns} kc {kc} tiles/CTA {tpc}"
            res = tcsim.gemm(NP, NP2, mode, H, W, a, w, bias, kc=kc, n_stage=ns, tiles_per_cta=tpc, N=N, midp=midp,
                             wfold=wfold, w2=w2, bias2=b2, N2=N2, out_f32=out_f32, **head)
            if res is None:
                skipped.append(cfg)
                continue
            ran.append(cfg + f" ({res['smem']} B, {res['ctas']} CTA/SM)")
            outs = {k: v for k, v in res.items() if isinstance(v, np.ndarray)}
            if first is None:
                first = outs
                continue
            for k in outs:
                assert np.array_equal(outs[k].view(np.uint8), first[k].view(np.uint8)), f"{cfg}: {k} differs from the first configuration"
        assert first is not None, f"{name}: no configuration fits shared memory"
        res = first
        if mode in (GM_PLAIN, GM_POOL, GM_TAIL, GM_TAIL_POOL2):
            inter = None
            if mode == GM_TAIL_POOL2:
                plain = tcsim.gemm(NP, 0, GM_PLAIN, H, W, a, w, bias, kc=[2] * len(c8s), n_stage=2, tiles_per_cta=1,
                                   N=N, midp=midp, wfold=wfold)
                hi, lo = _planes_out(plain, "out", CAP, NP // 8, HW)
                dh, dl = tcsim.from_planes(hi, lo)
                inter = (dh + dl)[:, :, :N]
            w_, d_ = _check_gemm(key, name, res, ops, H, W, c8s, midp, N, N2, NP, NP2, CAP, CAP, inter)
            if mode != GM_TAIL_POOL2 and not out_f32:
                C8o, HWo = NP // 8, (HW // 4 if mode == GM_POOL else HW)
                _check_canaries(res, "out", CAP, CAP, C8o, HWo)
            if mode in (GM_TAIL, GM_TAIL_POOL2):
                _check_canaries(res, "out2", CAP, CAP, NP2 // 8, HW // 4 if mode == GM_TAIL_POOL2 else HW)
            if out_f32:
                assert (res["out_f32"][CAP * HW * N:].view(np.uint32) == tcsim.F32_CANARY.view(np.uint32)).all()
        else:
            plain = tcsim.gemm(NP, 0, GM_PLAIN, H, W, a, w, bias, kc=[2], n_stage=2, tiles_per_cta=1, N=N, out_f32=True)
            pre = plain["out_f32"][:CAP * HW * N].reshape(CAP, HW, N)
            w_, d_ = _check_head(name, res, ops, head, H, W, c8s, N, NP, CAP, 0, pre=pre)
        worst_all, drop_all = max(worst_all, w_), min(drop_all, d_)
        assert drop_all >= 20, f"{name}: dropping a product would exceed the bound only {drop_all:.1f}x: the bound is too loose"
    REPORT[key] = (worst_all, drop_all, ran, skipped)
    print(f"\n[{NP},{NP2},{tcsim.MODE_NAMES[mode]}] worst error/bound {worst_all:.3f}, dropped product/bound >= {drop_all:.0f}")
    for r in ran:
        print("  ran", r)
    for s in skipped:
        print("  skipped (shared memory)", s)


def _head_ref(pre, hw, hb, extra=0.0):
    """GAP -> fc -> ReLU -> L2 of float64 pre-activations [HW][N] with a bound of the kernel's float32 epilogue, given
    an elementwise bound `extra` on the pre-activations themselves."""
    pooled = pre.mean(0)
    e_pool = (extra + 2.0 ** -19 * np.abs(pre)).mean(0)
    feat = tcsim.relu(hb + pooled @ hw)
    e_feat = e_pool @ np.abs(hw) + 2.0 ** -19 * (np.abs(hb) + np.abs(pooled) @ np.abs(hw))
    nrm = np.linalg.norm(feat)
    want = feat / nrm
    bound = (e_feat + np.abs(want) * (np.abs(want) @ e_feat)) / nrm * 1.01 + 2.0 ** -21 * np.abs(want)
    return want, bound, nrm


def _check_head(name, res, ops, head, H, W, c8s, N, NP, cap, off, n_valid=None, pre=None):
    """The scattered embeddings against float64 of the whole conv5 + head (bound propagated through the fc: too loose
    to see a dropped product), and -- given the plain conv5 instance's output `pre`, whose main loop is the same code --
    against float64 of the epilogue alone, where the dropped-product check applies."""
    a, w, wfold, bias, _, _ = ops
    n_valid = cap if n_valid is None else n_valid
    K, HW = 8 * sum(c8s), H * W
    hw, hb, rows, ld = head["head_w"].astype(np.float64), head["head_b"].astype(np.float64), head["out_row"], head["out_ld"]
    out = res["head"][:head["out_rows"] * ld].reshape(head["out_rows"], ld)
    written = {int(rows[off + n]) for n in range(n_valid)}
    worst, drop = 0.0, np.inf
    for n in range(n_valid):
        ref, S, drops, ref32, S32 = _gemm_ref(a, w, None, bias, 0, N, NP, n)
        got = out[rows[off + n], :512].astype(np.float64)
        for r, extra in ((ref, 0.0), (ref32, tcsim.plain_bound(S32))):
            want, bound, _ = _head_ref(tcsim.relu(r), hw, hb, tcsim.acc_bound(S, K) + extra)
            worst = max(worst, _ratio(np.abs(got - want), bound, f"{name} crop {n} embedding"))
        if pre is not None:
            p = pre[n].astype(np.float64)
            want, bound, nrm = _head_ref(p, hw, hb)
            worst = max(worst, _ratio(np.abs(got - want), bound, f"{name} crop {n} embedding from the conv5 output"))
            d = min(float((np.abs((tcsim.relu(ref + dd) - tcsim.relu(ref)).mean(0) @ hw) / nrm / bound).max())
                    for dd in drops[1:])
            drop = min(drop, d)
    for r in range(head["out_rows"]):
        cols = slice(512, ld) if r in written else slice(0, ld)
        assert (out[r, cols].view(np.uint32) == tcsim.F32_CANARY.view(np.uint32)).all(), f"{name}: row {r} written outside the crops' rows"
    assert (res["head"][head["out_rows"] * ld:].view(np.uint32) == tcsim.F32_CANARY.view(np.uint32)).all()
    return worst, drop


@pytest.mark.parametrize("key", [(64, 16, GM_TAIL), (96, 0, GM_POOL), (128, 0, GM_HEAD), (32, 0, GM_PLAIN)],
                         ids=lambda k: f"np{k[0]}_np2{k[1]}_{tcsim.MODE_NAMES[k[2]]}")
@pytest.mark.parametrize("window", ["off32_3of5", "count_le_off", "single_crop"])
def test_gemm_crop_windows(key, window):
    """The (d_n, off, cap) window: a chunk at offset 32 with 3 of 5 crops valid, a chunk with none, a single crop."""
    NP, NP2, mode = key
    name, H, W, c8s, midp, N, N2, identity = SHAPES[key][0]
    cap, off, count = {"off32_3of5": (5, 32, 35), "count_le_off": (5, 32, 20), "single_crop": (1, 0, 1)}[window]
    n_valid = max(0, min(count - off, cap))
    ops = _operands(7 + NP, cap, H, W, c8s, midp, N, N2, identity, NP, NP2)
    a, w, wfold, bias, w2, b2 = ops
    head = dict(head_w=None)
    if mode == GM_HEAD:
        rng = np.random.default_rng(6)
        head = dict(head_w=tcsim.weights(rng, N, 512), head_b=(rng.normal(size=512) * 0.1).astype(np.float32),
                    out_row=np.arange(off + cap, dtype=np.int32)[::-1].copy(), out_ld=515, out_rows=off + cap + 1)
    res = tcsim.gemm(NP, NP2, mode, H, W, a, w, bias, kc=[2] * len(c8s), n_stage=3, tiles_per_cta=_plan_tpc(H * W), N=N,
                     midp=midp, wfold=wfold, w2=w2, bias2=b2, N2=N2, cap=cap, off=off, count=count, **head)
    if mode == GM_HEAD:
        _check_head(name, res, ops, head, H, W, c8s, N, NP, cap, off, n_valid)
        return
    HWo = H * W // 4 if mode == GM_POOL else H * W
    _check_canaries(res, "out", n_valid, cap, NP // 8, HWo)
    if mode == GM_TAIL:
        _check_canaries(res, "out2", n_valid, cap, NP2 // 8, H * W)
    if n_valid:
        _check_gemm(key, name, res, ops, H, W, c8s, midp, N, N2, NP, NP2, n_valid, cap)


@pytest.mark.parametrize("NP,H,W,c8s", [(64, 64, 32, [8, 8]), (96, 32, 16, [16, 12]), (128, 16, 8, [16, 16])])
def test_identity_shortcut_is_exact(NP, H, W, c8s):
    """The combine GEMM with the gate rows at zero and no bias passes the block input through its identity block of B
    unchanged: hi * 1 + lo * 1 in FP32 is exact, and so is its split."""
    rng = np.random.default_rng(NP)
    midp = 8 * c8s[0] // 4
    a = [np.zeros((3, H * W, 8 * c8s[0]), np.float32), tcsim.activations(rng, 3, H * W, 8 * c8s[1], nonneg=True)]
    K = 8 * sum(c8s)
    w = np.zeros((K, NP), np.float32)
    w[4 * midp:] = np.eye(K - 4 * midp, NP, dtype=np.float32)
    res = tcsim.gemm(NP, 0, GM_PLAIN, H, W, a, w, np.zeros(NP, np.float32), kc=[2, 2], n_stage=2, tiles_per_cta=1,
                     midp=midp, wfold=rng.normal(size=(3, 4 * midp, NP)).astype(np.float32) * 0)
    hi, lo = _planes_out(res, "out", 3, NP // 8, H * W)
    dh, dl = tcsim.from_planes(hi, lo)
    xh, xl = tcsim.from_planes(*tcsim.to_planes(a[1]))
    assert np.array_equal(dh + dl, xh + xl)


def _lightconv_ref(x, pw, dw, b, H, W):
    """float64 LightConv3x3 on NHWC [H][W][C]: 1x1 (decoded split weights) -> depthwise 3x3 (zero padding) -> bias ->
    ReLU.  Returns (y, T, S_T) with S_T the magnitude sum of the 1x1."""
    wh, wl = (tcsim.bf2f(p).astype(np.float64) for p in tcsim.split(pw))
    T = x @ (wh + wl)
    S = np.abs(x) @ (np.abs(wh) + np.abs(wl))
    Tp = np.pad(T, ((1, 1), (1, 1), (0, 0)))
    y = np.broadcast_to(b.astype(np.float64), T.shape).copy()
    for ky in range(3):
        for kx in range(3):
            y += Tp[ky:ky + H, kx:kx + W] * dw[ky * 3 + kx].astype(np.float64)
    return tcsim.relu(y), T, S


def _dw_abs(E, dw, H, W):
    Ep = np.pad(E, ((1, 1), (1, 1), (0, 0)))
    out = np.zeros_like(E)
    for ky in range(3):
        for kx in range(3):
            out += Ep[ky:ky + H, kx:kx + W] * np.abs(dw[ky * 3 + kx]).astype(np.float64)
    return out


def _dw_signed(T, dw, H, W):
    Tp = np.pad(T, ((1, 1), (1, 1), (0, 0)))
    out = np.zeros_like(T)
    for ky in range(3):
        for kx in range(3):
            out += Tp[ky:ky + H, kx:kx + W] * dw[ky * 3 + kx].astype(np.float64)
    return out


def _chain_operands(shape, seed, cap, n_launch=1):
    g = tcsim.chain_shape(shape)
    CP, CR, W, H = g["CP"], g["CR"], g["W"], g["H"]
    rng = np.random.default_rng(seed)
    xs = np.zeros((n_launch, cap, H * W, CP), np.float32)
    xs[..., :CR] = tcsim.activations(rng, n_launch * cap, H * W, CR, nonneg=True).reshape(n_launch, cap, H * W, CR)
    hid = max(1, CR // 16)
    N = {0: 64, 1: 96, 2: 128}[shape]
    ops = dict(pw=np.stack([tcsim.weights(rng, CR, CR) for _ in range(10)]),
               dw=(rng.normal(size=(10, 9, CR)) * 0.4).astype(np.float32),
               b=(rng.normal(size=(10, CR)) * 0.2 - 0.05).astype(np.float32),
               g1w=tcsim.weights(rng, CR, hid), g1b=(rng.normal(size=hid) * 0.1).astype(np.float32),
               g2w=tcsim.weights(rng, hid, CR, scale=2.0), g2b=(rng.normal(size=CR) * 0.5).astype(np.float32),
               w3=tcsim.weights(rng, CR, N))
    return xs, ops


@pytest.mark.parametrize("shape", [0, 1, 2], ids=["S2_16ch_64x32", "S3_24ch_32x16", "S4_32ch_16x8"])
def test_chain_matches_float64(shape):
    cap = 3
    xs, ops = _chain_operands(shape, 40 + shape, cap)
    res = tcsim.chain(shape, xs, counts=[cap], **ops)
    CP, CR, W, H, R, NP, tiles = (res[k] for k in ("CP", "CR", "W", "H", "R", "NP", "tiles"))
    C8 = CP // 8
    assert (res["arrivals"] == 0).all(), "the arrival counters must reset for the next launch"
    yh = res["y_hi"][:cap * 4 * C8 * H * W * 8].reshape(cap, 4 * C8, H * W, 8)
    yl = res["y_lo"][:cap * 4 * C8 * H * W * 8].reshape(cap, 4 * C8, H * W, 8)
    assert (res["y_hi"][cap * 4 * C8 * H * W * 8:] == tcsim.BF16_CANARY).all()
    sums = res["sums"].reshape(4, cap, tiles, CP)
    gates = res["gates"].reshape(cap, 4, CP)
    fold = res["bfold"].reshape(cap, 4 * CP // 8, 2 * NP, 8)
    worst, drop = 0.0, np.inf
    N = ops["w3"].shape[1]
    for n in range(cap):
        xh, xl = tcsim.from_planes(*tcsim.to_planes(xs[0, n:n + 1]))
        x0 = (xh + xl)[0][:, :CR].reshape(H, W, CR)
        dh, dl = tcsim.from_planes(yh[n:n + 1], yl[n:n + 1])
        y_all = (dh + dl)[0].reshape(H, W, 4 * CP)
        means, e_means = [], []
        for br in range(4):
            l0 = br * (br + 1) // 2
            x, E = x0, np.zeros_like(x0)
            for lv in range(br + 1):
                L = l0 + lv
                y, T, S = _lightconv_ref(x, ops["pw"][L], ops["dw"][L], ops["b"][L], H, W)
                wabs = np.abs(ops["pw"][L]).astype(np.float64)
                E_T = E @ wabs + tcsim.acc_bound(S, CP) + 2.0 ** -15 * S
                E = _dw_abs(E_T, ops["dw"][L], H, W) + 2.0 ** -20 * (_dw_abs(np.abs(T), ops["dw"][L], H, W) + np.abs(ops["b"][L])) \
                    + 2.0 ** -16 * y
                if br == 0:
                    whh, wll = (tcsim.bf2f(p).astype(np.float64) for p in tcsim.split(ops["pw"][L]))
                    d = np.abs(_dw_signed(x @ wll, ops["dw"][L], H, W))
                x = y
            got = y_all[:, :, br * CP:br * CP + CR]
            assert not y_all[:, :, br * CP + CR:(br + 1) * CP].any(), "padded branch channels must be exact zeros"
            worst = max(worst, _ratio(np.abs(got - x), E, f"chain shape {shape} crop {n} branch {br}"))
            if br == 0:
                drop = min(drop, float((d / E).max()))
            # per-tile channel sums of the branch output (float32 sums over R x W pixels)
            ts = x.reshape(tiles, R, W, CR).sum(axis=(1, 2))
            e_ts = (E + 2.0 ** -14 * x).reshape(tiles, R, W, CR).sum(axis=(1, 2))
            worst = max(worst, _ratio(np.abs(sums[br, n, :, :CR] - ts), e_ts, f"chain shape {shape} crop {n} branch {br} sums"))
            assert not sums[br, n, :, CR:].any()
            means.append(ts.sum(0) / (H * W))
            e_means.append(e_ts.sum(0) / (H * W) * 1.001)
        hidw = ops["g1w"].astype(np.float64)
        for br in range(4):
            h = tcsim.relu(ops["g1b"] + means[br] @ hidw)
            e_h = e_means[br] @ np.abs(hidw) + 2.0 ** -20 * (np.abs(ops["g1b"]) + np.abs(means[br]) @ np.abs(hidw))
            s = ops["g2b"] + h @ ops["g2w"].astype(np.float64)
            e_s = e_h @ np.abs(ops["g2w"]) + 2.0 ** -20 * (np.abs(ops["g2b"]) + np.abs(h) @ np.abs(ops["g2w"]))
            g = 1 / (1 + np.exp(-s))
            e_g = 0.25 * e_s + 2.0 ** -21
            worst = max(worst, _ratio(np.abs(gates[n, br, :CR] - g), e_g, f"chain shape {shape} crop {n} gates {br}"))
            assert not gates[n, br, CR:].any()
            wh, wl = tcsim.unpack_b(fold[n], N)
            v = g[:, None] * ops["w3"].astype(np.float64)
            got = (wh + wl)[br * CP:br * CP + CR]
            e_v = e_g[:, None] * np.abs(ops["w3"]) + 2.0 ** -16 * np.abs(v) + 2.0 ** -22 * np.abs(v)
            worst = max(worst, _ratio(np.abs(got - v), e_v, f"chain shape {shape} crop {n} bfold {br}"))
            assert not (wh + wl)[br * CP + CR:(br + 1) * CP].any(), "padded rows of the folded conv3 must be exact zeros"
        fo = fold[n].reshape(4 * CP // 8, 2 * NP, 8)
        assert not fo[:, N:NP].any() and not fo[:, NP + N:].any()
    assert drop >= 20, f"chain shape {shape}: a dropped A_hi W_lo would exceed the bound only {drop:.1f}x"
    REPORT[("chain", shape)] = (worst, drop)
    print(f"\n[chain shape {shape}] worst error/bound {worst:.3f}, dropped product/bound >= {drop:.0f}")


@pytest.mark.parametrize("shape", [0, 1, 2], ids=["S2", "S3", "S4"])
def test_chain_back_to_back_launches_equal_separate_runs(shape):
    """Three launches with different counts and inputs on one set of buffers (the arrival counters reset themselves)
    leave exactly what separate launches leave."""
    cap = 5
    xs, ops = _chain_operands(shape, 70 + shape, cap, n_launch=3)
    counts = [5, 2, 4]
    seq = tcsim.chain(shape, xs, counts=counts, **ops)
    assert (seq["arrivals"] == 0).all()
    last = tcsim.chain(shape, xs[2:3], counts=[4], **ops)
    first = tcsim.chain(shape, xs[0:1], counts=[5], **ops)
    CP, H, W, NP, tiles = seq["CP"], seq["H"], seq["W"], seq["NP"], seq["tiles"]
    per = {"y_hi": 4 * CP * H * W, "y_lo": 4 * CP * H * W, "gates": 4 * CP, "bfold": (4 * CP // 8) * 2 * NP * 8}
    for k, size in per.items():
        s, l, f = (r[k][:cap * size].reshape(cap, size) for r in (seq, last, first))
        assert np.array_equal(s[:4].view(np.uint8), l[:4].view(np.uint8)), f"{k}: crops of the last launch"
        assert np.array_equal(s[4].view(np.uint8), f[4].view(np.uint8)), f"{k}: the crop only the first launch covered"
    s, l = (r["sums"].reshape(4, cap, tiles * CP) for r in (seq, last))
    assert np.array_equal(s[:, :4], l[:, :4])


# ---- network level, through B200ReID --------------------------------------------------------------------------------------
def _reid(tmp_path, seed=21, **kw):
    from boxmot_b200.reid import B200ReID
    from boxmot_b200.weights import export_blob
    from oracle import reid as orid

    sd = orid.make_osnet_state("osnet_x0_25", seed=seed)
    return sd, B200ReID(export_blob(sd, tmp_path / f"tc_{seed}.b200reid"), **kw)


def _boxes(rng, n, hw=(480, 640)):
    cx, cy = rng.uniform(0, hw[1], n), rng.uniform(0, hw[0], n)
    w, h = rng.uniform(20, 120, n), rng.uniform(40, 240, n)
    return np.stack([cx - w / 2, cy - h / 2, cx + w / 2, cy + h / 2], 1).astype(np.float32)


def test_embeddings_are_bitwise_batch_invariant(tmp_path, monkeypatch):
    """Every crop runs CTA-local in a fixed order: its embedding does not depend on the other crops of the batch, its
    position, the number of chunks or the chunk size."""
    monkeypatch.delenv("BOXMOT_B200_REID_CHUNK", raising=False)
    _, reid = _reid(tmp_path)
    rng = np.random.default_rng(8)
    img = rng.integers(0, 255, size=(480, 640, 3), dtype=np.uint8)
    boxes = _boxes(rng, 300)
    full = reid.get_features(boxes, img)                 # 300 crops: two chunks
    probe = [0, 1, 77, 255, 256, 299]
    for i in probe:
        assert np.array_equal(reid.get_features(boxes[i:i + 1], img)[0], full[i]), f"crop {i} alone"
    perm = rng.permutation(40)
    sub = reid.get_features(boxes[perm], img)
    assert np.array_equal(sub, full[perm]), "permuted batch"
    monkeypatch.setenv("BOXMOT_B200_REID_CHUNK", "24")
    _, reid24 = _reid(tmp_path)
    assert np.array_equal(reid24.get_features(boxes[:60], img), full[:60]), "chunk of 24 crops"


@pytest.mark.parametrize("preprocess", ["resize", "resize_pad"])
def test_front_kernel_edge_boxes(tmp_path, monkeypatch, preprocess):
    """Edge boxes through the fused front kernel at chunk boundaries (chunk 8, 19 boxes): resized crops (tap 50) bit-exact,
    the pooled stem (tap 2) within the per-stage bound."""
    from oracle import reid as orid

    monkeypatch.setenv("BOXMOT_B200_REID_CHUNK", "8")
    sd, reid = _reid(tmp_path, seed=23, preprocess=preprocess)
    rng = np.random.default_rng(9)
    img = rng.integers(0, 255, size=(240, 320, 3), dtype=np.uint8)
    boxes = np.array([
        [400, 300, 480, 400],        # fully outside: blank crop
        [-50, -40, -10, -5],         # fully outside, negative
        [100.2, 50, 100.4, 90],      # zero width after rounding
        [0, 0, 60, 120], [260, 0, 320, 120], [0, 120, 60, 240], [260, 120, 320, 240],   # each corner / border
        [-30, 20, 40, 200], [280, 20, 350, 200], [100, -25, 160, 60], [100, 200, 160, 300],
        [-100, -100, 500, 400],      # larger than the image
        [150, 40, 151, 200],         # 1 px wide
        [155, 100, 215, 101],        # 1 px high
        [0, 0, 320, 240],            # strong down-scaling (2.5x horizontally)
        [10, 10, 300, 30],
        [50, 60, 90, 180], [200, 30, 230, 230], [120, 120, 122, 124],
    ], np.float32)
    assert len(boxes) == 19
    _, want = orid.osnet_forward(sd, orid.get_crops(boxes, img, preprocess), return_stages=True)
    w_pool = want["pool"].permute(0, 2, 3, 1).contiguous().numpy().reshape(len(boxes), -1)
    u8_want = orid.crop_boxes(boxes, img, preprocess).astype(np.float32)
    for s in range(0, len(boxes), 8):           # a debug tap exposes the first chunk of the call
        sl = slice(s, min(s + 8, len(boxes)))
        u8 = reid.debug_stage(boxes[sl], img, 50).reshape(-1, 256, 128, 3)
        assert np.array_equal(u8, u8_want[sl]), f"resized crops {sl} must be bit-exact"
        g = reid.debug_stage(boxes[sl], img, 2)
        w = w_pool[sl]
        tol = 5e-5 * max(1.0, float(np.abs(w).max()))
        assert np.abs(g - w).max() < tol, f"pooled stem {sl}: max err {np.abs(g - w).max():.3e}"
    # 19 boxes = three chunks of 8: embeddings within the bound of tests/test_gpu_reid.py, and bit-identical to one chunk
    feats = reid.get_features(boxes, img)
    ref = orid.get_features(sd, boxes, img, preprocess)
    err = np.abs(feats - ref).max(axis=1)
    assert (err <= 1e-4 * np.abs(ref).max(axis=1)).all(), f"embedding error {err.max():.3e}"
    monkeypatch.delenv("BOXMOT_B200_REID_CHUNK")
    _, one = _reid(tmp_path, seed=23, preprocess=preprocess)
    assert np.array_equal(one.get_features(boxes, img), feats)
