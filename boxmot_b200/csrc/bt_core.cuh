// bt_core.cuh -- BoostTrack / BoostTrack++ per-stream, per-frame update (one CTA per stream), same conventions as
// docs_core.cuh (the source also compiles for the host under BMB_HOSTSIM for GPU-less tests).
//
// Replaces (relative to /root/reference/boxmot):
//   trackers/bbox/boosttrack/boosttrack.py:66-207   KalmanBoxTracker (predict, update, update_emb, get_confidence,
//                                                   camera_update)
//   trackers/bbox/boosttrack/boosttrack.py:298-529  BoostTrack._update_impl, filter_outputs, get_iou_matrix,
//                                                   get_mh_dist_matrix, dlo_confidence_boost, duo_confidence_boost
//   trackers/bbox/boosttrack/assoc.py:9-201         shape_similarity v1 / v2, MhDist_similarity, iou_batch,
//                                                   soft_biou_batch, match, linear_assignment, associate
//   motion/kalman_filters/xyhr.py:10-102,159-377    ConstantNoiseXYHR + KalmanFilterXYHR: 8-state [x, y, h, r, vx, vy,
//                                                   vh, vr], Q = diag(1 x4, 0.01 x4), R = diag(1, 1, 10, 0.01)
// Tracks live in the reference's list order (`tracks`: births appended, culls compacted in place); rows are emitted in
// that order.  Every detection row of the frame carries its (boosted) confidence; the rows that survive the
// `conf >= det_thresh` filter are `kdet`, and their appearance rows are picked out of the full per-row embedding matrix.
#pragma once
#include "tracker_core.cuh"
#include "jv_dense.cuh"

namespace bmb {

constexpr double BT_MH_LIMIT = 13.2767;   // chi2inv(0.99, 4): Mahalanobis gate of the boosts and of the softmax

struct BtCfg {
    int cap_tracks, cap_dets, feat_dim, max_age, min_hits, with_reid;
    int use_dlo, use_duo, rich_s, use_sb, use_vt, s_sim_corr;
    int cmc_every_frame;   // an estimator runs: camera_update on every frame (identity when it returns none)
    double det_thresh, iou_threshold, lambda_iou, lambda_mhd, lambda_shape, dlo_coef, min_box_area, ar_thresh;
    const double* conf_pow;   // [n_conf_pow] 0.9 ** k computed by the host with python's float power
    int n_conf_pow;
};

struct BtStream {
    // ---- persistent, slot indexed ----
    double* x;         // [CT][8]
    double* P;         // [CT][64]
    int* age;
    int* hit_streak;
    int* tsu;          // time_since_update
    int* id;
    double* conf;
    double* cls;
    double* det_ind;
    double* emb;       // [CT][F] float64
    int* tracks;       // [CT] ordered slot list (the reference's `trackers`)
    int* scalars;      // [SC_COUNT]
    long long* timers;
    // ---- inputs ----
    const float* dets;   // [CD][6]
    const int* n_dets;
    const float* embs;   // [CD][F] one row per detection row (every row is embedded), may be null
    const double* warp;  // [8] supplied / estimated 2x3 warp, warp[6] != 0 when one is pending; may be null
    // ---- scratch ----
    double* rconf;     // [CD] confidence of every row (boosted in place)
    double* dz;        // [CD][4] convert_bbox_to_z of every row
    double* tbox;      // [CT][5] predicted box + get_confidence by list position
    double* iou;       // [CD][CT] every row x every track
    double* md;        // [CD][CT] Mahalanobis distances
    double* ex;        // [CD][CT] exp(limit - gated distance)
    double* embq;      // [CD][CT] appearance dot product by (raw row, slot): filled by the wide k_bt_embcost
    double* colsum;    // [CT]
    double* ovmax;     // [CD]
    int* kdet;         // [CD] surviving rows
    int* cand;         // [CD] DUO candidates
    int* flag;         // [max(CT, CD)] per-row / per-track scratch flags
    int* mrow;         // [CD] matched track position per surviving row (or -1)
    int* und;          // [CD] unmatched surviving rows, birth order
    int* tmp_a;        // [CT]
    int* tmp_b;        // [CT]
    int* mark;         // [CT]
    int* free_l;       // [MB_COUNT + CT]
    double* cost;      // [MX][MX] assignment cost, lapjv's zero-padded square problem
    int* lap_x; int* lap_y; double* lap_u; double* lap_v; double* lap_spc; int* lap_path; int* lap_insc;
    int* lap_tl; int* lap_sc;
    float* out;        // [CD][8]
    int jv_wide;
};

BMB_FN double bt_iou(double a0, double a1, double a2, double a3, double b0, double b1, double b2, double b3) {
    double w = (a2 < b2 ? a2 : b2) - (a0 > b0 ? a0 : b0);
    double h = (a3 < b3 ? a3 : b3) - (a1 > b1 ? a1 : b1);
    w = 0.0 > w ? 0.0 : w;   // np.maximum(0.0, v): NaN propagates
    h = 0.0 > h ? 0.0 : h;
    const double wh = w * h;
    return wh / ((a2 - a0) * (a3 - a1) + (b2 - b0) * (b3 - b1) - wh);
}

// numpy's maximum / minimum / max-reduction: a NaN operand wins
BMB_FN double np_max(double a, double b) { return (a != a || b != b) ? (a != a ? a : b) : (a > b ? a : b); }
BMB_FN double np_min(double a, double b) { return (a != a || b != b) ? (a != a ? a : b) : (a < b ? a : b); }
// python's max(v, lo) for a float: NaN stays
BMB_FN double py_max(double v, double lo) { return lo > v ? lo : v; }

BMB_FN void bt_box_to_z(const float* r, double* z) {
    const double x1 = r[0], y1 = r[1], x2 = r[2], y2 = r[3];
    const double w = x2 - x1, h = y2 - y1;
    z[0] = x1 + w / 2.0; z[1] = y1 + h / 2.0; z[2] = h; z[3] = w / (h + 1e-6);
}

BMB_FN void bt_x_to_box(const double* x, double* b) {
    const double h = x[2], r = x[3];
    const double w = r <= 0 ? 0.0 : r * h;
    b[0] = x[0] - w / 2.0; b[1] = x[1] - h / 2.0; b[2] = x[0] + w / 2.0; b[3] = x[1] + h / 2.0;
}

BMB_FN void bt_enforce(double* x, double* P) {
    x[2] = py_max(x[2], 1e-4);
    x[3] = py_max(x[3], 1e-4);
    for (int i = 0; i < 8; ++i)
        for (int j = i + 1; j < 8; ++j) {
            const double v = 0.5 * (P[i * 8 + j] + P[j * 8 + i]);
            P[i * 8 + j] = v; P[j * 8 + i] = v;
        }
}

// KalmanFilterXYHR.predict: x <- F x, P <- F P F^T + Q (F = I + shift by 4), then the geometry clamp
BMB_FN void bt_predict(double* x, double* P) {
    for (int i = 0; i < 4; ++i) x[i] = x[i] + x[i + 4];
    double L[64];
    for (int i = 0; i < 8; ++i)
        for (int j = 0; j < 8; ++j) L[i * 8 + j] = i < 4 ? P[i * 8 + j] + P[(i + 4) * 8 + j] : P[i * 8 + j];
    for (int i = 0; i < 8; ++i)
        for (int j = 0; j < 8; ++j) {
            double v = j < 4 ? L[i * 8 + j] + L[i * 8 + j + 4] : L[i * 8 + j];
            if (i == j) v = v + (i < 4 ? 1.0 : 0.01);
            P[i * 8 + j] = v;
        }
    bt_enforce(x, P);
}

// KalmanFilterXYHR.update (xyhr.py:339-377): plain Cholesky of S = H P H^T + R, K = P H^T S^-1,
// x += alpha * (K (z - Hx)), P -= K S K^T, geometry clamp + symmetrise.  alpha is OccluBoost's abnormal-motion gain
// factor; BoostTrack passes 1.0, and x + 1.0 * v is x + v bit for bit.
BMB_FN void bt_kf_update(double* x, double* P, const double* z, double alpha) {
    const double Rd[4] = {1.0, 1.0, 10.0, 0.01};
    double m[4] = {z[0], z[1], py_max(z[2], 1e-4), py_max(z[3], 1e-4)};
    double S[16], Lc[16];
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) S[i * 4 + j] = P[i * 8 + j] + (i == j ? Rd[i] : 0.0);
    for (int i = 0; i < 16; ++i) Lc[i] = 0.0;
    for (int j = 0; j < 4; ++j) {
        double d = S[j * 4 + j];
        for (int k = 0; k < j; ++k) d -= Lc[j * 4 + k] * Lc[j * 4 + k];
        d = sqrt(d);
        Lc[j * 4 + j] = d;
        for (int i = j + 1; i < 4; ++i) {
            double v = S[i * 4 + j];
            for (int k = 0; k < j; ++k) v -= Lc[i * 4 + k] * Lc[j * 4 + k];
            Lc[i * 4 + j] = v / d;
        }
    }
    double K[32];   // [8][4]
    for (int r = 0; r < 8; ++r) {
        double y[4], kt[4];
        for (int i = 0; i < 4; ++i) {
            double v = P[r * 8 + i];
            for (int k = 0; k < i; ++k) v -= Lc[i * 4 + k] * y[k];
            y[i] = v / Lc[i * 4 + i];
        }
        for (int i = 3; i >= 0; --i) {
            double v = y[i];
            for (int k = i + 1; k < 4; ++k) v -= Lc[k * 4 + i] * kt[k];
            kt[i] = v / Lc[i * 4 + i];
        }
        for (int i = 0; i < 4; ++i) K[r * 4 + i] = kt[i];
    }
    double yv[4];
    for (int i = 0; i < 4; ++i) yv[i] = m[i] - x[i];
    for (int r = 0; r < 8; ++r) {
        double acc = 0.0;
        for (int i = 0; i < 4; ++i) acc += yv[i] * K[r * 4 + i];
        x[r] = x[r] + alpha * acc;
    }
    double KS[32];
    for (int r = 0; r < 8; ++r)
        for (int j = 0; j < 4; ++j) {
            double acc = 0.0;
            for (int k = 0; k < 4; ++k) acc += K[r * 4 + k] * S[k * 4 + j];
            KS[r * 4 + j] = acc;
        }
    for (int i = 0; i < 8; ++i)
        for (int j = 0; j < 8; ++j) {
            double acc = 0.0;
            for (int k = 0; k < 4; ++k) acc += KS[i * 4 + k] * K[j * 4 + k];
            P[i * 8 + j] = P[i * 8 + j] - acc;
        }
    bt_enforce(x, P);
}

// KalmanBoxTracker.camera_update (boosttrack.py:132-172), axis-aligned: warp the two corners of get_state() and
// rebuild [cx, cy, h, w / h]; no clamp, covariance and velocities untouched.  fma(W0, x, W1 * y) + W2 is what
// numpy's 3x3 @ 3 product gives on x86 BLAS kernels (as ss_camera_update).
BMB_FN void bt_camera_update(const double* W, double* x) {
    double b[4];
    bt_x_to_box(x, b);
    const double x1 = fma(W[0], b[0], W[1] * b[1]) + W[2], y1 = fma(W[3], b[0], W[4] * b[1]) + W[5];
    const double x2 = fma(W[0], b[2], W[1] * b[3]) + W[2], y2 = fma(W[3], b[2], W[4] * b[3]) + W[5];
    const double w = x2 - x1, h = y2 - y1;
    x[0] = x1 + w / 2; x[1] = y1 + h / 2; x[2] = h; x[3] = w / h;
}

BMB_FN double bt_track_conf(const BtCfg& c, const BtStream& s, int t) {
    int k = s.age[t] < 7 ? 7 - s.age[t] : s.tsu[t] - 1;
    k = k < 0 ? 0 : (k >= c.n_conf_pow ? c.n_conf_pow - 1 : k);
    return c.conf_pow[k];
}

// shape_similarity (assoc.py:15-34) between detection row z-box r and the predicted track box tb
BMB_FN double bt_shape(const BtCfg& c, const float* r, const double* tb) {
    const double dw = (double)r[2] - (double)r[0], dh = (double)r[3] - (double)r[1];
    const double tw = tb[2] - tb[0], th = tb[3] - tb[1];
    const double mw = np_max(dw, tw);
    const double mh = c.s_sim_corr ? np_max(dh, th) : mw;
    return exp(-(fabs(dw - tw) / mw + fabs(dh - th) / mh));
}

// soft_biou_batch (assoc.py:69-103): detection widened by 0.25, track by 0.5, both times (1 - track confidence)
BMB_FN double bt_soft_biou(const float* r, const double* tb) {
    const double d0 = r[0], d1 = r[1], d2 = r[2], d3 = r[3];
    const double sc = 1 - tb[4];
    const double dw = d2 - d0, dh = d3 - d1, tw = tb[2] - tb[0], th = tb[3] - tb[1];
    const double a0 = d0 - dw * sc * 0.25, a1 = d1 - dh * sc * 0.25, a2 = d2 + dw * sc * 0.25, a3 = d3 + dh * sc * 0.25;
    const double b0 = tb[0] - tw * sc * 0.5, b1 = tb[1] - th * sc * 0.5, b2 = tb[2] + tw * sc * 0.5, b3 = tb[3] + th * sc * 0.5;
    return bt_iou(a0, a1, a2, a3, b0, b1, b2, b3);
}

BMB_FN void bt_emb_update(const BtCfg& c, BtStream& s, int t, int d_raw, double alpha) {
    const int F = c.feat_dim;
    const float* e = s.embs + (size_t)d_raw * F;
    double* te = s.emb + (size_t)t * F;
    double acc = 0.0;
    for (int k = BMB_LANE; k < F; k += BMB_NL) {
        const double v = alpha * te[k] + (1 - alpha) * (double)e[k];
        te[k] = v;
        acc += v * v;
    }
#if BMB_DEVICE
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
#endif
    const double nrm = sqrt(acc);
    BMB_SYNCWARP();
    for (int k = BMB_LANE; k < F; k += BMB_NL) te[k] = te[k] / nrm;
    BMB_SYNCWARP();
}

// softmax of (limit - gated distance) down each track column over the rows `rows[0..n)` (numpy sums axis 0 in row
// order); ex / colsum hold the pieces, the similarity of (row i, track k) is bt_mh_sim
template <typename RowOf>
BMB_FN void bt_mh_softmax(BtStream& s, int n, int T, int LD, RowOf row_of) {
    for (int e = BMB_TID; e < n * T; e += BMB_NT) {
        const int i = e / T, k = e - i * T;
        const double m = s.md[(size_t)row_of(i) * LD + k];
        s.ex[(size_t)i * LD + k] = exp(BT_MH_LIMIT - (m > BT_MH_LIMIT ? BT_MH_LIMIT : m));
    }
    BMB_SYNC();
    for (int k = BMB_TID; k < T; k += BMB_NT) {
        double acc = s.ex[k];
        for (int i = 1; i < n; ++i) acc += s.ex[(size_t)i * LD + k];
        s.colsum[k] = acc;
    }
    BMB_SYNC();
}

BMB_FN double bt_mh_sim(const BtStream& s, int i, int row, int k, int LD) {
    return s.md[(size_t)row * LD + k] > BT_MH_LIMIT ? 0.0 : s.ex[(size_t)i * LD + k] / s.colsum[k];
}

// What the phases of one frame hand to each other.  t_prev carries the phase clock (BMB_PHASE) across them.
struct BtFrame {
    int D, T, frame, nk, n_und, n_ufail;
    bool use_emb;
    long long _t_prev;
};

// ---- camera_update on every track, then predict (boosttrack.py:318-331); IoU and Mahalanobis distance of every row
// against every track (get_mh_dist_matrix) ----
BMB_FN BtFrame bt_predict_phase(const BtCfg& c, BtStream& s) {
    const int CD = c.cap_dets;
    const int LD = c.cap_tracks;
    BtFrame f{};
    int D = *s.n_dets;
    if (D > CD) { if (BMB_TID == 0) s.scalars[SC_ERROR] = ERR_DET_CAPACITY; D = CD; }
    f.D = D;
    f.frame = s.scalars[SC_FRAME] + 1;
    const int T = f.T = s.scalars[SC_N_ACTIVE];
    f.use_emb = c.with_reid && s.embs != nullptr;
    long long& _t_prev = f._t_prev;   // phase clocks: 0 camera update + predict, 1 matrices, 2 boosts, 3 cost + match,
    _t_prev = BMB_CLOCK();            // 4 updates, 5 births, 6 emit + cull
    BMB_SYNC();

    const bool warp_pending = s.warp != nullptr && s.warp[6] != 0.0;
    const double ident[6] = {1.0, 0.0, 0.0, 0.0, 1.0, 0.0};
    const double* W = warp_pending ? s.warp : ident;
    for (int k = BMB_TID; k < T; k += BMB_NT) {
        const int t = s.tracks[k];
        double* x = s.x + t * 8;
        if (warp_pending || c.cmc_every_frame) bt_camera_update(W, x);
        bt_predict(x, s.P + t * 64);
        s.age[t] += 1;
        if (s.tsu[t] > 0) s.hit_streak[t] = 0;
        s.tsu[t] += 1;
        bt_x_to_box(x, s.tbox + k * 5);
        s.tbox[k * 5 + 4] = bt_track_conf(c, s, t);
    }
    for (int d = BMB_TID; d < D; d += BMB_NT) {
        s.rconf[d] = (double)s.dets[d * 6 + 4];
        bt_box_to_z(s.dets + d * 6, s.dz + d * 4);
    }
    BMB_SYNC();
    BMB_PHASE(0);

    for (int e = BMB_TID; e < D * T; e += BMB_NT) {
        const int d = e / T, k = e - d * T;
        const float* r = s.dets + d * 6;
        const double* tb = s.tbox + k * 5;
        s.iou[(size_t)d * LD + k] = bt_iou(r[0], r[1], r[2], r[3], tb[0], tb[1], tb[2], tb[3]);
        const int t = s.tracks[k];
        const double* x = s.x + t * 8;
        const double* P = s.P + t * 64;
        const double* z = s.dz + d * 4;
        double acc = 0.0;
        for (int i = 0; i < 4; ++i) {
            const double v = z[i] - x[i];
            const double term = v * v * (1.0 / P[i * 9]);
            acc = i == 0 ? term : acc + term;
        }
        s.md[(size_t)d * LD + k] = acc;
    }
    BMB_SYNC();
    BMB_PHASE(1);
    return f;
}

// ---- DLO boost (boosttrack.py:489-529) over every row, then the DUO boost (boosttrack.py:447-487): far from every
// track and below the threshold, boosted unless a more confident candidate overlaps it; then the survivors
// conf >= det_thresh ----
BMB_FN void bt_boost_phase(const BtCfg& c, BtStream& s, BtFrame& f) {
    const int LD = c.cap_tracks;
    const int D = f.D, T = f.T;
    int* mb = s.free_l;
    long long& _t_prev = f._t_prev;
    if (c.use_dlo && D > 0 && T > 0) {
        if (c.rich_s) bt_mh_softmax(s, D, T, LD, [](int i) { return i; });
        for (int d = BMB_TID; d < D; d += BMB_NT) {
            const float* r = s.dets + d * 6;
            double smax = 0.0;
            bool hit = false;
            for (int k = 0; k < T; ++k) {
                const double* tb = s.tbox + k * 5;
                double S;
                if (c.rich_s) S = ((bt_mh_sim(s, d, d, k, LD) + bt_shape(c, r, tb)) + bt_soft_biou(r, tb)) / 3;
                else S = s.iou[(size_t)d * LD + k];
                smax = k == 0 ? S : np_max(smax, S);
                const double lim = np_max(0.95 - (double)(s.tsu[s.tracks[k]] - 1), 0.8);
                hit = hit || S > lim;
            }
            double cf = s.rconf[d];
            if (!c.use_sb && !c.use_vt) {
                cf = np_max(cf, smax * c.dlo_coef);
            } else {
                if (c.use_sb) cf = np_max(cf, 0.65 * cf + (1 - 0.65) * pow(smax, 1.5));
                if (c.use_vt && hit) cf = np_max(cf, c.det_thresh + 1e-5);
            }
            s.rconf[d] = cf;
        }
        BMB_SYNC();
    }
    if (c.use_duo && D > 0 && T > 0) {
        if (BMB_WARP == 0) {
            const int n = warp_append(D, s.cand, 0, [&](int d) {
                double mn = s.md[(size_t)d * LD];
                for (int k = 1; k < T; ++k) mn = np_min(mn, s.md[(size_t)d * LD + k]);
                return mn > BT_MH_LIMIT && s.rconf[d] < c.det_thresh;
            }, [&](int d) { return d; });
            if (BMB_LANE == 0) mb[0] = n;
        }
        BMB_SYNC();
        const int nc = mb[0];
        auto ov = [&](int i, int j) {
            const float* a = s.dets + s.cand[i] * 6;
            const float* b = s.dets + s.cand[j] * 6;
            return bt_iou(a[0], a[1], a[2], a[3], b[0], b[1], b[2], b[3]) - (i == j ? 1.0 : 0.0);
        };
        for (int i = BMB_TID; i < nc; i += BMB_NT) {
            double m = ov(i, 0);
            for (int j = 1; j < nc; ++j) m = np_max(m, ov(i, j));
            s.ovmax[i] = m;
        }
        BMB_SYNC();
        for (int i = BMB_TID; i < nc; i += BMB_NT) {
            int boost = s.ovmax[i] <= 0.3;
            if (s.ovmax[i] > 0.3) {
                double cm = s.rconf[s.cand[i]];
                for (int j = 0; j < nc; ++j)
                    if (s.ovmax[j] > 0.3 && ov(i, j) > 0.3) cm = np_max(cm, s.rconf[s.cand[j]]);
                boost = s.rconf[s.cand[i]] == cm;
            }
            s.flag[i] = boost;
        }
        BMB_SYNC();
        for (int i = BMB_TID; i < nc; i += BMB_NT)
            if (s.flag[i]) s.rconf[s.cand[i]] = c.det_thresh + 1e-4;
        BMB_SYNC();
    }
    if (BMB_WARP == 0) {
        const int n = warp_append(D, s.kdet, 0, [&](int d) { return s.rconf[d] >= c.det_thresh; }, [&](int d) { return d; });
        if (BMB_LANE == 0) mb[1] = n;
    }
    BMB_SYNC();
    f.nk = mb[1];
    BMB_PHASE(2);
}

// ---- association (assoc.py:156-201, 106-153) with lambda_emb = (1 + l_iou + l_shape + l_mhd) * lambda_emb_mult.
// mrow[i]: matched track position of survivor i or -1; und[0..n_und): unmatched survivors (unmatched ascending, then
// the matches that fail the validity test, in row order); tmp_b[0..n_ufail): the track positions of those failed
// matches, in the same order (the tail of the reference's unmatched_trks) ----
BMB_FN void bt_match_phase(const BtCfg& c, BtStream& s, BtFrame& f, double lambda_emb_mult) {
    const int CT = c.cap_tracks;
    const int LD = CT;
    const int LD2 = CT > c.cap_dets ? CT : c.cap_dets;
    const int T = f.T, nk = f.nk;
    const bool use_emb = f.use_emb;
    int* mb = s.free_l;
    long long& _t_prev = f._t_prev;
    int n_und = 0, n_ufail = 0;
    if (T == 0 || nk == 0) {
        for (int i = BMB_TID; i < nk; i += BMB_NT) { s.mrow[i] = -1; s.und[i] = i; }
        n_und = nk;
        BMB_SYNC();
    } else {
        bt_mh_softmax(s, nk, T, LD, [&](int i) { return s.kdet[i]; });
        const double lambda_emb = (((1 + c.lambda_iou) + c.lambda_shape) + c.lambda_mhd) * lambda_emb_mult;
        auto cost_at = [&](int i, int k) {
            const int d = s.kdet[i];
            const float* r = s.dets + d * 6;
            const double io = s.iou[(size_t)d * LD + k];
            const double cf = io < c.iou_threshold ? 0.0 : s.rconf[d] * s.tbox[k * 5 + 4];
            double v = io + c.lambda_iou * cf * io;
            v = v + c.lambda_mhd * bt_mh_sim(s, i, d, k, LD);
            v = v + c.lambda_shape * cf * bt_shape(c, r, s.tbox + k * 5);
            if (use_emb) v = v + lambda_emb * s.embq[(size_t)d * CT + s.tracks[k]];
            return v;
        };
        // the cost goes straight into the solver's square scratch
        const int n = nk > T ? nk : T;
        for (int e = BMB_TID; e < n * n; e += BMB_NT) {
            const int i = e / n, j = e - i * n;
            s.cost[(size_t)i * LD2 + j] = (i < nk && j < T) ? cost_at(i, j) : 0.0;
        }
        if (BMB_TID == 0) { mb[2] = 0; mb[3] = 0; }
        BMB_SYNC();
        // match(): when no row and no column has more than one entry above the threshold, np.where order
        for (int i = BMB_TID; i < nk; i += BMB_NT) {
            int m = 0;
            for (int k = 0; k < T; ++k) m += s.cost[(size_t)i * LD2 + k] > c.iou_threshold ? 1 : 0;
            BMB_ATOMIC_MAX(&mb[2], m > 1 ? 2 : m);
        }
        for (int k = BMB_TID; k < T; k += BMB_NT) {
            int m = 0;
            for (int i = 0; i < nk; ++i) m += s.cost[(size_t)i * LD2 + k] > c.iou_threshold ? 1 : 0;
            BMB_ATOMIC_MAX(&mb[3], m > 1 ? 2 : m);
        }
        BMB_SYNC();
        const int rmax = mb[2], cmax = mb[3];
        BMB_SYNC();
        if (rmax == 1 && cmax == 1) {
            for (int i = BMB_TID; i < nk; i += BMB_NT) {
                int m = -1;
                for (int k = 0; k < T; ++k)
                    if (s.cost[(size_t)i * LD2 + k] > c.iou_threshold) m = k;
                s.mrow[i] = m;
            }
            BMB_SYNC();
        } else {
            // lap.lapjv(-cost, extend_cost=True): negate in place, solve the zero-padded square problem
            for (int e = BMB_TID; e < n * n; e += BMB_NT) {
                const int i = e / n, j = e - i * n;
                if (i < nk && j < T) s.cost[(size_t)i * LD2 + j] = -s.cost[(size_t)i * LD2 + j];
            }
            BMB_SYNC();
            jv_dense_solve(s, n, LD2, nk, s.jv_wide);
            for (int i = BMB_TID; i < nk; i += BMB_NT) s.mrow[i] = s.lap_x[i] < T ? s.lap_x[i] : -1;
            BMB_SYNC();
        }
        // unmatched rows (ascending), then the matches that fail the validity test, in row order
        if (BMB_TID == 0) {
            for (int i = 0; i < nk; ++i) if (s.mrow[i] < 0) s.und[n_und++] = i;
            for (int i = 0; i < nk; ++i) {
                const int k = s.mrow[i];
                if (k < 0) continue;
                const int d = s.kdet[i];
                const double io = s.iou[(size_t)d * LD + k];
                const bool ok = io >= c.iou_threshold ||
                                (use_emb && io >= c.iou_threshold / 2 && s.embq[(size_t)d * CT + s.tracks[k]] >= 0.75);
                if (!ok) { s.und[n_und++] = i; s.tmp_b[n_ufail++] = k; s.mrow[i] = -1; }
            }
            mb[4] = n_und;
            mb[8] = n_ufail;
        }
        BMB_SYNC();
        n_und = mb[4];
        n_ufail = mb[8];
        BMB_SYNC();
    }
    f.n_und = n_und;
    f.n_ufail = n_ufail;
    BMB_PHASE(3);
}

// ---- BoostTrack's tail: updates of the matched tracks (boosttrack.py:378-387), births in unmatched order
// (389-393), emit in list order with the aspect / area filter (395-421), cull ----
BMB_FN void bt_tail_phase(const BtCfg& c, BtStream& s, BtFrame& f) {
    const int CT = c.cap_tracks, CD = c.cap_dets, F = c.feat_dim;
    const int T = f.T, nk = f.nk, n_und = f.n_und, frame = f.frame;
    const bool use_emb = f.use_emb;
    int* mb = s.free_l;
    int* free_slots = s.free_l + MB_COUNT;
    long long& _t_prev = f._t_prev;
    for (int i = BMB_TID; i < nk; i += BMB_NT) {
        if (s.mrow[i] < 0) continue;
        const int t = s.tracks[s.mrow[i]], d = s.kdet[i];
        s.tsu[t] = 0;
        s.hit_streak[t] += 1;
        bt_kf_update(s.x + t * 8, s.P + t * 64, s.dz + d * 4, 1.0);
        s.conf[t] = s.rconf[d];
        s.cls[t] = (double)s.dets[d * 6 + 5];
        s.det_ind[t] = (double)d;
    }
    if (use_emb)
        for (int i = BMB_WARP; i < nk; i += BMB_NW) {
            if (s.mrow[i] < 0) continue;
            const int d = s.kdet[i];
            const double trust = (s.rconf[d] - c.det_thresh) / (1 - c.det_thresh);
            bt_emb_update(c, s, s.tracks[s.mrow[i]], d, 0.95 + (1 - 0.95) * (1 - trust));
        }
    BMB_SYNC();
    BMB_PHASE(4);

    // ---- births in unmatched order (boosttrack.py:389-393) ----
    for (int k = BMB_TID; k < CT; k += BMB_NT) s.mark[k] = 0;
    BMB_SYNC();
    for (int k = BMB_TID; k < T; k += BMB_NT) s.mark[s.tracks[k]] = 1;
    BMB_SYNC();
    if (BMB_WARP == 0) {
        int nfree = 0;
        for (int k0 = 0; k0 < CT && nfree < n_und; k0 += BMB_NL) {
            const int k = k0 + BMB_LANE;
            const bool p = k < CT && !s.mark[k];
            const unsigned m = BMB_BALLOT(p);
#if BMB_DEVICE
            const int pos = nfree + __popc(m & ((1u << BMB_LANE) - 1u));
#else
            const int pos = nfree;
#endif
            if (p && pos < n_und) free_slots[pos] = k;
            nfree += BMB_POPC(m);
        }
        if (BMB_LANE == 0) {
            if (nfree < n_und) s.scalars[SC_ERROR] = ERR_TRACK_CAPACITY;
            mb[5] = nfree < n_und ? nfree : n_und;
        }
    }
    BMB_SYNC();
    const int n_birth = mb[5];
    {
        const int id0 = s.scalars[SC_NEXT_ID];
        for (int k = BMB_TID; k < n_birth; k += BMB_NT) {
            const int t = free_slots[k], d = s.kdet[s.und[k]];
            double* x = s.x + t * 8;
            double* P = s.P + t * 64;
            const double* z = s.dz + d * 4;
            x[0] = z[0]; x[1] = z[1]; x[2] = py_max(z[2], 1e-4); x[3] = py_max(z[3], 1e-4);
            for (int i = 4; i < 8; ++i) x[i] = 0.0;
            for (int i = 0; i < 64; ++i) P[i] = 0.0;
            for (int i = 0; i < 8; ++i) P[i * 9] = i < 4 ? 10.0 : 10000.0;
            s.age[t] = 0; s.hit_streak[t] = 0; s.tsu[t] = 0;
            s.id[t] = id0 + 1 + k;
            s.conf[t] = s.rconf[d];
            s.cls[t] = (double)s.dets[d * 6 + 5];
            s.det_ind[t] = (double)d;
            s.tracks[T + k] = t;
        }
        if (use_emb)
            for (int k = BMB_WARP; k < n_birth; k += BMB_NW) {
                const int t = free_slots[k], d = s.kdet[s.und[k]];
                const float* e = s.embs + (size_t)d * F;
                for (int q = BMB_LANE; q < F; q += BMB_NL) s.emb[(size_t)t * F + q] = (double)e[q];
            }
    }
    BMB_SYNC();
    const int n_all = T + n_birth;
    BMB_PHASE(5);

    // ---- emit in list order with the aspect / area filter (boosttrack.py:395-421), then cull ----
    for (int k = BMB_TID; k < n_all; k += BMB_NT) {
        const int t = s.tracks[k];
        int keep = s.tsu[t] < 1 && (s.hit_streak[t] >= c.min_hits || frame <= c.min_hits);
        if (keep) {
            double b[4];
            bt_x_to_box(s.x + t * 8, b);
            const double w = b[2] - b[0], h = b[3] - b[1];
            keep = (w / h <= c.ar_thresh) && (w * h > c.min_box_area);
        }
        s.flag[k] = keep;
    }
    BMB_SYNC();
    if (BMB_WARP == 0) {
        int n_out = warp_append(n_all, s.tmp_b, 0, [&](int k) { return s.flag[k] != 0; }, [&](int k) { return s.tracks[k]; });
        if (n_out > CD) { if (BMB_LANE == 0) s.scalars[SC_ERROR] = ERR_DET_CAPACITY; n_out = CD; }
        const int keep = warp_append(n_all, s.tmp_a, 0, [&](int k) { return s.tsu[s.tracks[k]] <= c.max_age; },
                                     [&](int k) { return s.tracks[k]; });
        if (BMB_LANE == 0) { mb[6] = n_out; mb[7] = keep; }
    }
    BMB_SYNC();
    for (int k = BMB_TID; k < mb[6]; k += BMB_NT) {
        const int t = s.tmp_b[k];
        double b[4];
        bt_x_to_box(s.x + t * 8, b);
        float* o = s.out + k * 8;
        o[0] = (float)b[0]; o[1] = (float)b[1]; o[2] = (float)b[2]; o[3] = (float)b[3];
        o[4] = (float)s.id[t]; o[5] = (float)s.conf[t]; o[6] = (float)s.cls[t]; o[7] = (float)s.det_ind[t];
    }
    BMB_SYNC();
    for (int k = BMB_TID; k < mb[7]; k += BMB_NT) s.tracks[k] = s.tmp_a[k];
    if (BMB_TID == 0) {
        s.scalars[SC_N_ACTIVE] = mb[7];
        s.scalars[SC_FRAME] = frame;
        s.scalars[SC_N_OUT] = mb[6];
        s.scalars[SC_NEXT_ID] += n_birth;
    }
    BMB_SYNC();
    BMB_PHASE(6);
}


BMB_FN void bt_frame(const BtCfg& c, BtStream& s) {
    BtFrame f = bt_predict_phase(c, s);
    bt_boost_phase(c, s, f);
    bt_match_phase(c, s, f, 1.5);
    bt_tail_phase(c, s, f);
}

}  // namespace bmb
