// ss_core.cuh -- StrongSORT per-stream, per-frame update (one CTA per stream), same conventions as
// tracker_core.cuh / docs_core.cuh (also compiles for the host under BMB_HOSTSIM for GPU-less tests).
//
// Replaces (relative to /root/reference/boxmot):
//   trackers/bbox/strongsort/strongsort.py:69-123        StrongSort._update_impl
//   trackers/bbox/strongsort/sort/tracker.py:62-169      Tracker.predict / update / _match / _initiate_track
//   trackers/bbox/strongsort/sort/track.py:66-196        Track (camera_update, predict, NSA update, mark_missed)
//   trackers/bbox/strongsort/sort/linear_assignment.py:12-110,145-198   min_cost_matching, matching_cascade,
//                                                        gate_cost_matrix
//   trackers/bbox/strongsort/sort/linear_assignment.py:201-221,266-283,304-344  NN cosine metric + sample gallery
//   trackers/bbox/strongsort/sort/iou_matching.py:9-87   tlwh IoU cost
//   motion/kalman_filters/base.py:253-268,286-355,523-551 + xyah.py:22-68   XYAH filter: single-track predict,
//                                                        project / update with confidence, gating_distance
//   scipy.optimize.linear_sum_assignment                 -> lsa_sap.cuh ;  CPython set order -> pyset.cuh
//
// Work split per frame (tracker_engine.cu): k_ss_prepare (unit detection features) -> k_ss_appearance (nearest-
// neighbour cosine distance of every confirmed track's gallery to every detection: the one GEMM-shaped piece, wide
// grid) -> ss_frame below (one CTA per stream) -> k_ss_features (appearance EMA / births / gallery append).
#pragma once
#include "lsa_sap.cuh"
#include "pyset.cuh"
#include "tracker_core.cuh"

namespace bmb {

enum { SS_TENTATIVE = 1, SS_CONFIRMED = 2, SS_DELETED = 3 };
enum { SS_PEND_NONE = 0, SS_PEND_BIRTH = 1, SS_PEND_EMA = 2 };

struct SsCfg {
    int cap_tracks, cap_dets, feat_dim, n_init, max_age, budget;
    double min_conf, max_cos_dist, max_iou_dist, mc_lambda, ema_alpha;
};

struct SsStream {
    // ---- persistent, slot indexed ----
    int* scalars;      // [SC_COUNT]
    long long* timers; // [16]
    int* state;        // [CT]
    int* id;
    int* hits;
    int* age;
    int* tsu;          // time_since_update
    int* gal_n;        // [CT] gallery entries held (<= budget)
    int* gal_head;     // [CT] next ring position
    int* pend_kind;    // [CT] appearance work left for k_ss_features (SS_PEND_*)
    int* pend_det;     // [CT] raw detection index of that work
    int* tracks;       // [CT] ordered slot list (Tracker.tracks)
    double* conf;      // [CT]
    double* cls;
    double* det_ind;
    double* mean;      // [CT][8]
    double* cov;       // [CT][64]
    float* feat;       // [CT][F]     Track.features[-1] (smoothed, unit norm)
    float* gal;        // [CT][B][F]  metric.samples[id], rows stored as a / |a| (what _cosine_distance uses)
    // ---- inputs ----
    const float* dets;   // [CD][6]
    const int* n_dets;
    const float* embs;   // [CD][F] raw appearance rows by detection index
    const double* warp;  // [8]: 2x3 camera warp, warp[6] != 0 when one is pending (identity otherwise)
    // ---- scratch ----
    float* dfeatn;     // [CD][F] detection rows / |row|
    float* appc;       // [CT][CD] NN cosine distance by (slot, raw detection)
    int* kdet;         // [CD] kept raw detection indices
    double* dtlwh;     // [CD][4] by kept position
    double* dxyah;     // [CD][4]
    double* dconf;     // [CD]
    double* tproj;     // [CT][20] projected mean (4) + Cholesky factor (16) by confirmed row
    double* cost;      // [CT*CD] assignment cost in solver orientation (rows = the smaller side)
    int* conf_pos;     // [CT] confirmed list positions
    int* cand;         // [CT] IoU-stage rows (list positions)
    int* unta;         // [CT] list(set(confirmed) - set(matched))
    int* mdet;         // [CT] matched kept-detection position by list position (-1 none)
    int* rowcol;       // [CT] assigned column of each row of the current stage (-1 none)
    int* colrow;       // [CD] assigned row of each column
    int* und;          // [CD] unmatched kept-detection positions after the appearance stage
    int* und2;         // [CD] ... after the IoU stage
    int* tmp_a;        // [CT + CD]
    int* mark;         // [CT]
    int* free_l;       // [MB_COUNT + CT]
    int* set_buf;      // [4][8*CT + 16] CPython set emulation tables
    double* lsa_u; double* lsa_v; double* lsa_spc;                                  // [MX]
    int* lsa_path; int* lsa_row4col; int* lsa_col4row; int* lsa_rem; int* lsa_sr; int* lsa_sc;  // [MX]
    float* out;        // [CD][8]
};

// ---- XYAH Kalman filter, float64 measurement (StrongSORT's detections are float64 after the det-index hstack) ----
BMB_FN void ss_kf_initiate(const double* z, double* mean, double* cov) {
    const double two_wp = 2 * BMB_W_POS, ten_wv = 10 * BMB_W_VEL;
    double sd[8];
    for (int i = 0; i < 4; ++i) { sd[i] = two_wp * z[3]; sd[4 + i] = ten_wv * z[3]; }
    sd[2] = 1e-2; sd[6] = 1e-5;
    for (int i = 0; i < 64; ++i) cov[i] = 0.0;
    for (int i = 0; i < 8; ++i) cov[i * 8 + i] = sd[i] * sd[i];
    for (int i = 0; i < 4; ++i) { mean[i] = z[i]; mean[4 + i] = 0.0; }
    if (mean[2] < 1e-4) mean[2] = 1e-4;
    if (mean[3] < 1e-4) mean[3] = 1e-4;
}

// base.py:253-268: single-track predict.  np.linalg.multi_dot((F, P, F^T)) evaluates F (P F^T) for equal shapes.
BMB_FN void ss_kf_predict(double* mean, double* cov) {
    double q[8];
    {
        const double sp = BMB_W_POS * mean[3], sv = BMB_W_VEL * mean[3];
        for (int i = 0; i < 4; ++i) { q[i] = sp * sp; q[4 + i] = sv * sv; }
        q[2] = 1e-2 * 1e-2; q[6] = 1e-5 * 1e-5;
    }
    for (int i = 0; i < 4; ++i) mean[i] = mean[i] + mean[4 + i];
    double R[64];
    for (int i = 0; i < 8; ++i)
        for (int j = 0; j < 8; ++j) R[i * 8 + j] = (j < 4) ? (cov[i * 8 + j] + cov[i * 8 + j + 4]) : cov[i * 8 + j];
    for (int i = 0; i < 8; ++i)
        for (int j = 0; j < 8; ++j) {
            double v = (i < 4) ? (R[i * 8 + j] + R[(i + 4) * 8 + j]) : R[i * 8 + j];
            if (i == j) v = v + q[i];
            cov[i * 8 + j] = v;
        }
    if (mean[2] < 1e-4) mean[2] = 1e-4;
    if (mean[3] < 1e-4) mean[3] = 1e-4;
}

// S = H P H^T + diag(((1 - confidence) * std)^2) and its lower Cholesky factor (base.py:286-309)
BMB_FN void ss_kf_project(const double* mean, const double* cov, double confidence, double* S, double* Lc) {
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) S[i * 4 + j] = cov[i * 8 + j];
    for (int i = 0; i < 4; ++i) {
        double sd = (i == 2) ? 1e-1 : BMB_W_POS * mean[3];
        sd = (1 - confidence) * sd;
        S[i * 4 + i] = S[i * 4 + i] + sd * sd;
    }
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
}

// base.py:329-355 with the NSA measurement noise (track.py:174-176)
BMB_FN void ss_kf_update(const double* z, double confidence, double* mean, double* cov) {
    double S[16], Lc[16];
    ss_kf_project(mean, cov, confidence, S, Lc);
    double KT[32];
    for (int r = 0; r < 8; ++r) {
        double y[4];
        for (int i = 0; i < 4; ++i) {
            double v = cov[r * 8 + i];
            for (int k = 0; k < i; ++k) v -= Lc[i * 4 + k] * y[k];
            y[i] = v / Lc[i * 4 + i];
        }
        for (int i = 3; i >= 0; --i) {
            double v = y[i];
            for (int k = i + 1; k < 4; ++k) v -= Lc[k * 4 + i] * KT[k * 8 + r];
            KT[i * 8 + r] = v / Lc[i * 4 + i];
        }
    }
    double inn[4];
    for (int i = 0; i < 4; ++i) inn[i] = z[i] - mean[i];
    for (int r = 0; r < 8; ++r) {
        double acc = 0.0;
        for (int i = 0; i < 4; ++i) acc += inn[i] * KT[i * 8 + r];
        mean[r] = mean[r] + acc;
    }
    double M[32];
    for (int i = 0; i < 4; ++i)
        for (int r = 0; r < 8; ++r) {
            double acc = 0.0;
            for (int k = 0; k < 4; ++k) acc += S[i * 4 + k] * KT[k * 8 + r];
            M[i * 8 + r] = acc;
        }
    for (int a = 0; a < 8; ++a)
        for (int b = 0; b < 8; ++b) {
            double acc = 0.0;
            for (int k = 0; k < 4; ++k) acc += KT[k * 8 + a] * M[k * 8 + b];
            cov[a * 8 + b] = cov[a * 8 + b] - acc;
        }
    if (mean[2] < 1e-4) mean[2] = 1e-4;
    if (mean[3] < 1e-4) mean[3] = 1e-4;
}

BMB_FN void ss_tlwh(const double* mean, double* o) {
    const double w = mean[2] * mean[3];
    o[0] = mean[0] - w / 2;
    o[1] = mean[1] - mean[3] / 2;
    o[2] = w;
    o[3] = mean[3];
}

// track.py:139-148: the box corners go through the 3x3 warp and come back as (cx, cy, a, h)
BMB_FN void ss_camera_update(const double* W, double* mean) {
    double b[4];
    ss_tlwh(mean, b);
    const double x1 = b[0], y1 = b[1], x2 = b[0] + b[2], y2 = b[1] + b[3];
    // `warp_matrix @ np.array([x, y, 1])` (track.py:143-144) goes through numpy's small-matrix product, which rounds as
    // fma(W0, x, W1 * y) + W2 on the x86 BLAS kernels of this image (checked against numpy on 20 000 random triples; the
    // plain left-to-right sum agrees only 75 % of the time).  One ulp matters here: StrongSORT's births follow scipy's
    // tie-breaking among gated pairs, which depends on the dual variables and therefore on the last bit of every cost.
    const double x1w = fma(W[0], x1, W[1] * y1) + W[2], y1w = fma(W[3], x1, W[4] * y1) + W[5];
    const double x2w = fma(W[0], x2, W[1] * y2) + W[2], y2w = fma(W[3], x2, W[4] * y2) + W[5];
    const double w = x2w - x1w, h = y2w - y1w;
    mean[0] = x1w + w / 2;
    mean[1] = y1w + h / 2;
    mean[2] = w / h;
    mean[3] = h;
}

// iou_matching.py:9-47 on (top-left, size) boxes
BMB_FN double ss_tlwh_iou(const double* a, const double* b) {
    const double ax2 = a[0] + a[2], ay2 = a[1] + a[3], bx2 = b[0] + b[2], by2 = b[1] + b[3];
    const double tlx = a[0] > b[0] ? a[0] : b[0], tly = a[1] > b[1] ? a[1] : b[1];
    const double brx = ax2 < bx2 ? ax2 : bx2, bry = ay2 < by2 ? ay2 : by2;
    double w = brx - tlx; w = w > 0.0 ? w : 0.0;
    double h = bry - tly; h = h > 0.0 ? h : 0.0;
    const double inter = w * h;
    return inter / ((a[2] * a[3] + b[2] * b[3]) - inter);
}

// ---- appearance pieces run by the wide kernels (one warp each) ------------------------------------------------
// unit-norm copy of one detection row
BMB_FN void ss_prepare_row(const SsCfg& c, SsStream& s, int d) {
    const int F = c.feat_dim;
    const float* e = s.embs + (size_t)d * F;
    const float nr = vec_norm_f32(e, F);
    for (int q = BMB_LANE; q < F; q += BMB_NL) s.dfeatn[(size_t)d * F + q] = e[q] / nr;
    BMB_SYNCWARP();
}

// reference form of the NN cosine distance of one confirmed track against one detection (host simulation and
// parity checks of the tiled kernel): min over the gallery of float32 (1 - a.b)
BMB_FN float ss_nn_cosine(const SsCfg& c, const SsStream& s, int slot, int d) {
    const int F = c.feat_dim, n = s.gal_n[slot];
    const float* b = s.dfeatn + (size_t)d * F;
    float best = INFINITY;
    for (int g = 0; g < n; ++g) {
        const float* a = s.gal + ((size_t)slot * c.budget + g) * F;
        float acc = 0.0f;
        for (int q = BMB_LANE; q < F; q += BMB_NL) acc = fmaf(a[q], b[q], acc);
        acc = warp_sum_f(acc);
        const float dist = 1.0f - acc;
        best = dist < best ? dist : best;
    }
    return best;
}

// after the frame: appearance of list position k (birth copy / EMA, track.py:98-101,178-184) and the gallery append
// of every confirmed track (tracker.py:96-106, linear_assignment.py:304-326)
BMB_FN void ss_features_pos(const SsCfg& c, SsStream& s, int k) {
    const int F = c.feat_dim;
    const int t = s.tracks[k];
    float* ft = s.feat + (size_t)t * F;
    const int kind = s.pend_kind[t];
    if (kind != SS_PEND_NONE) {
        const float* e = s.embs + (size_t)s.pend_det[t] * F;
        const float nr = vec_norm_f32(e, F);
        if (kind == SS_PEND_BIRTH) {
            for (int q = BMB_LANE; q < F; q += BMB_NL) ft[q] = e[q] / nr;
        } else {
            const float al = (float)c.ema_alpha, be = (float)(1 - c.ema_alpha);
            for (int q = BMB_LANE; q < F; q += BMB_NL) {
                const float f = e[q] / nr;
                const float x = al * ft[q], y = be * f;
                ft[q] = x + y;
            }
            BMB_SYNCWARP();
            const float n2 = vec_norm_f32(ft, F);
            BMB_SYNCWARP();
            for (int q = BMB_LANE; q < F; q += BMB_NL) ft[q] = ft[q] / n2;
        }
        BMB_SYNCWARP();
        if (BMB_LANE == 0) s.pend_kind[t] = SS_PEND_NONE;
    }
    if (s.state[t] == SS_CONFIRMED) {
        const float nr = vec_norm_f32(ft, F);
        const int head = s.gal_head[t];
        float* g = s.gal + ((size_t)t * c.budget + head) * F;
        for (int q = BMB_LANE; q < F; q += BMB_NL) g[q] = ft[q] / nr;
        BMB_SYNCWARP();
        if (BMB_LANE == 0) {
            s.gal_head[t] = head + 1 == c.budget ? 0 : head + 1;
            if (s.gal_n[t] < c.budget) s.gal_n[t] += 1;
        }
    }
    BMB_SYNCWARP();
}

// ---- one min_cost_matching stage (linear_assignment.py:12-70) ----------------------------------------------------
// cost_at(r, c) is the gated cost of row r (0..R) against column c (0..C); entries above max_distance are clipped,
// the matrix is laid out with the smaller side as solver rows (scipy transposes when nc < nr) and solved.
// Results: rowcol[r] / colrow[c] for ACCEPTED pairs only (cost <= max_distance), and the reference's unmatched-
// detection order in und_out (columns never assigned ascending, then clipped assignments in row order).
// col_val(c) maps a column to the value stored in und_out.  Returns the unmatched count through mb_slot.
template <typename CostAt, typename ColVal>
BMB_FN void ss_match_stage(SsStream& s, int R, int C, double max_distance, CostAt cost_at, ColVal col_val,
                           int* und_out, int* mb, int mb_slot) {
    const bool transposed = C < R;
    const int nc = transposed ? R : C;
    const double clipv = max_distance + 1e-5;
    // raw assignment (clipped pairs included) in original orientation
    lsa_rect(s, s.cost, R, C, [&](int r, int cc) {
        const double v = cost_at(r, cc);
        return v > max_distance ? clipv : v;
    }, s.rowcol);
    for (int cc = BMB_TID; cc < C; cc += BMB_NT) s.colrow[cc] = -1;
    BMB_SYNC();
    for (int r = BMB_TID; r < R; r += BMB_NT)
        if (s.rowcol[r] >= 0) s.colrow[s.rowcol[r]] = r;
    BMB_SYNC();
    if (BMB_WARP == 0) {
        int n = warp_append(C, und_out, 0, [&](int cc) { return s.colrow[cc] < 0; }, col_val);
        n = warp_append(R, und_out, n, [&](int r) {
            const int cc = s.rowcol[r];
            return cc >= 0 && s.cost[transposed ? (size_t)cc * nc + r : (size_t)r * nc + cc] > max_distance; },
            [&](int r) { return col_val(s.rowcol[r]); });
        if (BMB_LANE == 0) mb[mb_slot] = n;
    }
    BMB_SYNC();
    // drop the clipped assignments
    for (int r = BMB_TID; r < R; r += BMB_NT) {
        const int cc = s.rowcol[r];
        if (cc >= 0 && s.cost[transposed ? (size_t)cc * nc + r : (size_t)r * nc + cc] > max_distance) {
            s.rowcol[r] = -1;
            s.colrow[cc] = -1;
        }
    }
    BMB_SYNC();
}

// ---- the frame --------------------------------------------------------------------------------------------------
BMB_FN void ss_frame(const SsCfg& c, SsStream& s) {
    const int CT = c.cap_tracks, CD = c.cap_dets;
    long long _t_prev = BMB_CLOCK();
    int* mb = s.free_l;
    int* free_slots = s.free_l + MB_COUNT;
    int D = *s.n_dets;
    if (D > CD) {
        if (BMB_TID == 0) s.scalars[SC_ERROR] = ERR_DET_CAPACITY;
        D = CD;
    }
    const int frame = s.scalars[SC_FRAME] + 1;
    const int T = s.scalars[SC_N_ACTIVE];
    BMB_SYNC();

    // ---- detections: conf >= min_conf in float64 (strongsort.py:74-81), tlwh / xyah in float64 ----
    if (BMB_WARP == 0) {
        const int nk = warp_append(D, s.kdet, 0, [&](int d) { return (double)s.dets[d * 6 + 4] >= c.min_conf; },
                                   [&](int d) { return d; });
        if (BMB_LANE == 0) mb[0] = nk;
    }
    BMB_SYNC();
    const int nk = mb[0];
    for (int k = BMB_TID; k < nk; k += BMB_NT) {
        const float* r = s.dets + s.kdet[k] * 6;
        const double x1 = (double)r[0], y1 = (double)r[1], x2 = (double)r[2], y2 = (double)r[3];
        double* b = s.dtlwh + k * 4;
        b[0] = x1; b[1] = y1; b[2] = x2 - x1; b[3] = y2 - y1;
        double* z = s.dxyah + k * 4;
        z[0] = b[0] + b[2] / 2; z[1] = b[1] + b[3] / 2; z[2] = b[2] / b[3]; z[3] = b[3];
        s.dconf[k] = (double)r[4];
    }
    // ---- camera update (whenever tracks exist, identity included) and predict ----
    {
        double W[6] = {1.0, 0.0, 0.0, 0.0, 1.0, 0.0};
        if (s.warp && s.warp[6] != 0.0)
            for (int i = 0; i < 6; ++i) W[i] = s.warp[i];
        for (int k = BMB_TID; k < T; k += BMB_NT) {
            const int t = s.tracks[k];
            double* m = s.mean + t * 8;
            ss_camera_update(W, m);
            ss_kf_predict(m, s.cov + t * 64);
            s.age[t] += 1;
            s.tsu[t] += 1;
            s.mdet[k] = -1;
        }
    }
    BMB_SYNC();
    BMB_PHASE(0);

    // ---- appearance stage over the confirmed tracks (tracker.py:108-137) ----
    if (BMB_WARP == 0) {
        const int n = warp_append(T, s.conf_pos, 0, [&](int k) { return s.state[s.tracks[k]] == SS_CONFIRMED; },
                                  [&](int k) { return k; });
        if (BMB_LANE == 0) mb[1] = n;
    }
    BMB_SYNC();
    const int nC = mb[1];
    int n_und = nk;
    if (nC > 0 && nk > 0) {
        for (int r = BMB_TID; r < nC; r += BMB_NT) {
            const int t = s.tracks[s.conf_pos[r]];
            double S[16];
            double* p = s.tproj + r * 20;
            ss_kf_project(s.mean + t * 8, s.cov + t * 64, 0.0, S, p + 4);
            for (int i = 0; i < 4; ++i) p[i] = s.mean[t * 8 + i];
        }
        BMB_SYNC();
        const double lam = c.mc_lambda, one_m = 1 - c.mc_lambda;
        ss_match_stage(s, nC, nk, c.max_cos_dist, [&](int r, int k) {
            const double* p = s.tproj + r * 20;
            const double* L = p + 4;
            const double* z = s.dxyah + k * 4;
            double y[4];
            for (int i = 0; i < 4; ++i) {
                double v = z[i] - p[i];
                for (int q = 0; q < i; ++q) v -= L[i * 4 + q] * y[q];
                y[i] = v / L[i * 4 + i];
            }
            const double g = ((y[0] * y[0] + y[1] * y[1]) + y[2] * y[2]) + y[3] * y[3];
            double a = (double)s.appc[(size_t)s.tracks[s.conf_pos[r]] * CD + s.kdet[k]];
            if (g > 9.4877) a = 1e5;
            return lam * a + one_m * g;
        }, [&](int k) { return k; }, s.und, mb, 2);
        n_und = mb[2];
        for (int r = BMB_TID; r < nC; r += BMB_NT) s.mdet[s.conf_pos[r]] = s.rowcol[r];
        BMB_SYNC();
    } else {
        for (int k = BMB_TID; k < nk; k += BMB_NT) s.und[k] = k;
        BMB_SYNC();
    }
    BMB_PHASE(1);

    // ---- list(set(confirmed) - set(matched)) in CPython's order (linear_assignment.py:108) ----
    if (BMB_WARP == 0) {
        const int nu = warp_append(nC, s.unta, 0, [&](int r) { return s.mdet[s.conf_pos[r]] < 0; },
                                   [&](int r) { return s.conf_pos[r]; });
        BMB_SYNCWARP();
        if (BMB_LANE == 0) {
            int n = nu;
            if (nC > 0 && nu > 0 &&
                !pyset_difference_is_ascending(nC, s.conf_pos[nC - 1], nC - nu, s.unta[nu - 1])) {
                const size_t stride = (size_t)8 * CT + 16;
                n = pyset_difference(s.conf_pos, nC, nC - nu, [&](int key) { return s.mdet[key] >= 0; }, s.unta,
                                     s.tmp_a, s.set_buf, s.set_buf + stride, s.set_buf + 2 * stride,
                                     s.set_buf + 3 * stride);
            }
            mb[3] = n;
        }
    }
    BMB_SYNC();
    const int n_unta = mb[3];
    // ---- IoU stage: tentative tracks + confirmed tracks missed for exactly one frame (tracker.py:139-153) ----
    if (BMB_WARP == 0) {
        int n = warp_append(T, s.cand, 0, [&](int k) { return s.state[s.tracks[k]] != SS_CONFIRMED; },
                            [&](int k) { return k; });
        n = warp_append(n_unta, s.cand, n, [&](int q) { return s.tsu[s.tracks[s.unta[q]]] == 1; },
                        [&](int q) { return s.unta[q]; });
        if (BMB_LANE == 0) mb[4] = n;
    }
    BMB_SYNC();
    const int nCand = mb[4];
    int* und_final = s.und;
    int n_birth_req = n_und;
    if (nCand > 0 && n_und > 0) {
        ss_match_stage(s, nCand, n_und, c.max_iou_dist, [&](int r, int q) {
            const int t = s.tracks[s.cand[r]];
            if (s.tsu[t] > 1) return 1e5;
            double b[4];
            ss_tlwh(s.mean + t * 8, b);
            return 1.0 - ss_tlwh_iou(b, s.dtlwh + s.und[q] * 4);
        }, [&](int q) { return s.und[q]; }, s.und2, mb, 5);
        n_birth_req = mb[5];
        und_final = s.und2;
        for (int r = BMB_TID; r < nCand; r += BMB_NT)
            if (s.rowcol[r] >= 0) s.mdet[s.cand[r]] = s.und[s.rowcol[r]];
        BMB_SYNC();
    }
    BMB_PHASE(2);

    // ---- matched: NSA Kalman update + bookkeeping; unmatched: mark_missed (track.py:162-196) ----
    for (int k = BMB_TID; k < T; k += BMB_NT) {
        const int t = s.tracks[k];
        const int kd = s.mdet[k];
        if (kd >= 0) {
            const int d = s.kdet[kd];
            s.conf[t] = s.dconf[kd];
            s.cls[t] = (double)s.dets[d * 6 + 5];
            s.det_ind[t] = (double)d;
            ss_kf_update(s.dxyah + kd * 4, s.dconf[kd], s.mean + t * 8, s.cov + t * 64);
            s.hits[t] += 1;
            s.tsu[t] = 0;
            if (s.state[t] == SS_TENTATIVE && s.hits[t] >= c.n_init) s.state[t] = SS_CONFIRMED;
            s.pend_kind[t] = SS_PEND_EMA;
            s.pend_det[t] = d;
        } else {
            if (s.state[t] == SS_TENTATIVE || s.tsu[t] > c.max_age) s.state[t] = SS_DELETED;
        }
    }
    for (int k = BMB_TID; k < CT; k += BMB_NT) s.mark[k] = 0;
    BMB_SYNC();
    for (int k = BMB_TID; k < T; k += BMB_NT) s.mark[s.tracks[k]] = 1;
    BMB_SYNC();
    // ---- births in unmatched-detection order (tracker.py:91-93,159-169); slots held this frame are not reused ----
    if (BMB_WARP == 0) {
        int nfree = 0;
        for (int k0 = 0; k0 < CT && nfree < n_birth_req; k0 += BMB_NL) {
            const int k = k0 + BMB_LANE;
            const bool p = k < CT && !s.mark[k];
            const unsigned m = BMB_BALLOT(p);
#if BMB_DEVICE
            const int pos = nfree + __popc(m & ((1u << BMB_LANE) - 1u));
#else
            const int pos = nfree;
#endif
            if (p && pos < n_birth_req) free_slots[pos] = k;
            nfree += BMB_POPC(m);
        }
        const int keep = warp_append(T, s.tmp_a, 0, [&](int k) { return s.state[s.tracks[k]] != SS_DELETED; },
                                     [&](int k) { return s.tracks[k]; });
        if (BMB_LANE == 0) {
            if (nfree < n_birth_req) s.scalars[SC_ERROR] = ERR_TRACK_CAPACITY;
            mb[6] = nfree < n_birth_req ? nfree : n_birth_req;
            mb[7] = keep;
        }
    }
    BMB_SYNC();
    const int n_birth = mb[6], n_keep = mb[7];
    {
        const int id0 = s.scalars[SC_NEXT_ID];   // last id handed out; Tracker._next_id starts at 1
        for (int k = BMB_TID; k < n_birth; k += BMB_NT) {
            const int t = free_slots[k], kd = und_final[k], d = s.kdet[kd];
            ss_kf_initiate(s.dxyah + kd * 4, s.mean + t * 8, s.cov + t * 64);
            s.id[t] = id0 + 1 + k;
            s.conf[t] = s.dconf[kd];
            s.cls[t] = (double)s.dets[d * 6 + 5];
            s.det_ind[t] = (double)d;
            s.hits[t] = 1; s.age[t] = 1; s.tsu[t] = 0; s.state[t] = SS_TENTATIVE;
            s.gal_n[t] = 0; s.gal_head[t] = 0;
            s.pend_kind[t] = SS_PEND_BIRTH;
            s.pend_det[t] = d;
            s.tmp_a[n_keep + k] = t;
        }
    }
    BMB_SYNC();
    const int n_all = n_keep + n_birth;
    for (int k = BMB_TID; k < n_all; k += BMB_NT) s.tracks[k] = s.tmp_a[k];
    BMB_SYNC();
    // ---- emit confirmed tracks updated this frame (strongsort.py:104-121) ----
    if (BMB_WARP == 0) {
        int n_out = warp_append(n_all, s.cand, 0, [&](int k) {
            const int t = s.tracks[k];
            return s.state[t] == SS_CONFIRMED && s.tsu[t] < 1; }, [&](int k) { return s.tracks[k]; });
        if (n_out > CD) { if (BMB_LANE == 0) s.scalars[SC_ERROR] = ERR_DET_CAPACITY; n_out = CD; }
        if (BMB_LANE == 0) mb[8] = n_out;
    }
    BMB_SYNC();
    const int n_out = mb[8];
    for (int k = BMB_TID; k < n_out; k += BMB_NT) {
        const int t = s.cand[k];
        double b[4];
        ss_tlwh(s.mean + t * 8, b);
        float* o = s.out + k * 8;
        o[0] = (float)b[0]; o[1] = (float)b[1]; o[2] = (float)(b[0] + b[2]); o[3] = (float)(b[1] + b[3]);
        o[4] = (float)s.id[t]; o[5] = (float)s.conf[t]; o[6] = (float)s.cls[t]; o[7] = (float)s.det_ind[t];
    }
    if (BMB_TID == 0) {
        s.scalars[SC_N_ACTIVE] = n_all;
        s.scalars[SC_FRAME] = frame;
        s.scalars[SC_N_OUT] = n_out;
        s.scalars[SC_NEXT_ID] += n_birth;
    }
    BMB_SYNC();
    BMB_PHASE(3);
}

}  // namespace bmb
