// sf_core.cuh -- SFSORT per-stream, per-frame update (one CTA per stream), same conventions as tracker_core.cuh (the
// source also compiles for the host under BMB_HOSTSIM for GPU-less tests).
//
// Replaces (relative to /root/reference/boxmot):
//   trackers/bbox/sfsort/sfsort.py:239-345   SFSORT._update_impl: density-tuned thresholds, purge of the lost pool,
//                                            the two association passes, births, the lost-pool update, output rows
//   trackers/bbox/sfsort/sfsort.py:523-630   _calculate_cost_aabb + _combine_cost_terms (float32)
//   trackers/association/matching.py:28-43   linear_assignment = lapjv(extend_cost=True, cost_limit), solved on the
//                                            (T + D) square matrix lapjv builds, in lapjv's own order (jv_dense.cuh):
//                                            the float32 costs tie (duplicate boxes) and ties decide ids
// No Kalman filter, no appearance, no camera motion.  Tracks live in the reference's list order: `active_tracks`
// (rows are emitted in that order) and `lost_tracks`.  The CTA's threads build the cost matrices and run the solver;
// thread 0 walks the lists, which are O(tracks + detections) per frame.
#pragma once
#include "tracker_core.cuh"
#include "jv_dense.cuh"

namespace bmb {

enum { SF_ACTIVE = 0, SF_LOST_CENTRAL = 1, SF_LOST_MARGINAL = 2 };
// scalars beyond the shared SC_* slots: margins of the stream are known (from the configuration or the first frame)
enum { SC_SF_MARGINS = 10 };
// mailbox (first ints of `mb`): counts thread 0 hands to the CTA
enum { SF_MB_T = 0, SF_MB_NH, SF_MB_NM, SF_MB_NU, SF_MB_NN, SF_MB_SKIP, SF_MB_COUNT = 8 };

struct SfCfg {
    int cap_tracks, cap_dets;
    int dynamic;                 // density-tuned thresholds (_dynamic_thresholds)
    // comparison precision of `score > hth` / `score < hth` and `score > nth`: 1 = float64 (the reference holds the
    // threshold as np.float64, as the density-tuned ones are), 0 = float32 (a python float, weak under NEP 50).
    // low_th and cth are python floats in the reference: always float32.
    int hth_f64, nth_f64;
    int marginal_timeout, central_timeout;
    int margins_given;           // frame_width and frame_height were given: margins below; else the first frame's size
    float margin[4];             // l, r, t, b
    double h_margin, v_margin;   // horizontal_margin / vertical_margin (None = 0)
    double high_th, new_track_th, match_th_first, low_th, match_th_second, cth;
    double high_th_m, new_track_th_m, match_th_first_m;
    const double* log10_tab;     // [n_log10] np.log10(k) computed by the host
    int n_log10;
};

struct SfStream {
    // ---- persistent, slot indexed ----
    float* box;        // [CT][4] float32 box of the last matched detection
    float* conf;
    float* cls;
    int* det_ind;
    int* last_frame;
    int* id;
    int* state;        // SF_ACTIVE / SF_LOST_CENTRAL / SF_LOST_MARGINAL
    int* active;       // [CT] ordered slot list (active_tracks)
    int* lost;         // [CT] ordered slot list (lost_tracks)
    float* margins;    // [4] l, r, t, b once scalars[SC_SF_MARGINS] is set
    int* scalars;      // [SC_COUNT]
    long long* timers;
    // ---- inputs ----
    const float* dets;   // [CD][6]
    const int* n_dets;
    const float* embs;   // wired like every family's input set; SFSORT reads neither embeddings nor warps
    const double* warp;
    const int* frame_hw; // [2] rows, cols of the stream's frames (0, 0 while unknown): its margins come from the first
    // ---- scratch ----
    int* high;         // [CD] rows with score > hth (definite)
    int* mid;          // [CD] rows with low_th < score < hth (possible)
    int* pool;         // [CT] track_pool = active + lost
    int* unm;          // [CT] pool positions pass 1 left unmatched
    int* nxt;          // [CT] next_active_tracks
    int* nlost;        // [CT]
    int* mark;         // [CT] per-slot flags
    int* next_lost;    // [CT]
    int* mb;           // [SF_MB_COUNT]
    double* th;        // [4] hth, nth, mth of this frame
    int* free_l;       // [MB_COUNT] the dense solver's mailbox
    double* cost;      // [MX][MX], MX = CT + CD: lapjv's extended square problem
    int* lap_x; int* lap_y; double* lap_v; double* lap_spc; int* lap_path; int* lap_insc; int* lap_tl; int* lap_sc;  // [MX]
    float* out;        // [CD][8]
    int jv_wide;       // dense-JV augmentation mode (set per launch, not part of the carved state)
};

// _calculate_cost_aabb (+ _combine_cost_terms unless iou_only) of one (track, detection) pair, float32 in numpy's order
// of operations; eps = float32(1e-7).  The reference's "h_intersection" is the x extent.  (Built with -fmad=false:
// nothing contracts.)
BMB_FN float sf_cost(const float* a, const float* b, bool iou_only) {
    const float eps = 1e-7f;
    float hi = (a[2] < b[2] ? a[2] : b[2]) - (a[0] > b[0] ? a[0] : b[0]);
    float wi = (a[3] < b[3] ? a[3] : b[3]) - (a[1] > b[1] ? a[1] : b[1]);
    hi = hi > 0.f ? hi : 0.f;
    wi = wi > 0.f ? wi : 0.f;
    const float inter = hi * wi;
    const float bh1 = a[2] - a[0], bh2 = b[2] - b[0], bw1 = a[3] - a[1], bw2 = b[3] - b[1];
    const float uni = ((bh2 * bw2 + bh1 * bw1) - inter) + eps;
    const float iou = inter / uni;
    if (iou_only) return 1.0f - iou;
    const float cx1 = (a[0] + a[2]) / 2.0f, cy1 = (a[1] + a[3]) / 2.0f;
    const float cx2 = (b[0] + b[2]) / 2.0f, cy2 = (b[1] + b[3]) / 2.0f;
    const float sw = wi / fabsf((wi + fabsf(bw2 - bw1)) + eps);
    const float sh = hi / fabsf((hi + fabsf(bh2 - bh1)) + eps);
    const float inner = fabsf(cx1 - cx2) + fabsf(cy1 - cy2);
    float outer = fabsf((a[2] > b[2] ? a[2] : b[2]) - (a[0] < b[0] ? a[0] : b[0])) +
                  fabsf((a[3] > b[3] ? a[3] : b[3]) - (a[1] < b[1] ? a[1] : b[1]));
    outer = outer > eps ? outer : eps;
    const float diou = iou - inner / outer;
    return 1.0f - ((diou + sh) + sw) / 3.0f;
}

BMB_FN bool sf_gt(float s, double th, int f64) { return f64 ? (double)s > th : s > (float)th; }
BMB_FN bool sf_lt(float s, double th, int f64) { return f64 ? (double)s < th : s < (float)th; }
// python's max(lo, min(v, hi))
BMB_FN double sf_clamp(double v, double lo, double hi) {
    const double m = hi < v ? hi : v;
    return m > lo ? m : lo;
}

// linear_assignment(cost, limit) for pool rows `rows` (slot = pool[rows[r]], or pool[r] when rows is null) x detection
// rows `cols`: lapjv's (T + D) square matrix (the costs, limit / 2 beside them, 0 in the dummy block) solved in lapjv's
// order.  lap_x[r] >= D / lap_y[k] >= T mean unmatched.
BMB_FN void sf_assign(SfStream& s, const int* rows, int T, const int* cols, int D, bool iou_only, double limit) {
    const int n = T + D;
    const double half = limit / 2.0;
    for (int e = BMB_TID; e < n * n; e += BMB_NT) {
        const int i = e / n, j = e - i * n;
        double v;
        if (i < T && j < D)
            v = (double)sf_cost(s.box + (size_t)s.pool[rows ? rows[i] : i] * 4, s.dets + (size_t)cols[j] * 6, iou_only);
        else
            v = (i >= T && j >= D) ? 0.0 : half;
        s.cost[e] = v;
    }
    BMB_SYNC();
    jv_dense_solve(s, n, n, n, s.jv_wide);
    BMB_SYNC();
}

BMB_FN void sf_set(SfStream& s, int slot, const float* d, int row, int frame) {
    for (int q = 0; q < 4; ++q) s.box[(size_t)slot * 4 + q] = d[q];
    s.conf[slot] = d[4];
    s.cls[slot] = d[5];
    s.det_ind[slot] = row;
    s.last_frame[slot] = frame;
    s.state[slot] = SF_ACTIVE;
}

// log10(k) for k = 0 .. n - 1 with the host's libm: the density table of handles whose creator supplies none (the C ABI).
// numpy's vectorised log10 differs from glibc's in the last bit for some counts (11, 40, 43, ...), so the Python layer
// hands the engine np.log10's own table (BoxMOTB200TrackerConfig.sf_log10_table)
inline void sf_log10_table(int n, double* out) {
    for (int k = 0; k < n; ++k) out[k] = log10((double)k);
}

// one frame of SFSORT._update_impl for one stream
BMB_FN void sf_frame(const SfCfg& c, SfStream& s) {
    int* sc = s.scalars;
    const int CT = c.cap_tracks;
    if (BMB_TID == 0) {
        s.mb[SF_MB_SKIP] = 1;
        if (sc[SC_ERROR] == ERR_NONE && *s.n_dets > c.cap_dets) sc[SC_ERROR] = ERR_DET_CAPACITY;
        if (sc[SC_ERROR] != ERR_NONE) sc[SC_N_OUT] = 0;
        else s.mb[SF_MB_SKIP] = 0;
    }
    BMB_SYNC();
    if (s.mb[SF_MB_SKIP]) return;   // sticky capacity error: nothing runs until reset
    const int D = *s.n_dets;
    if (BMB_TID == 0) {
        const int rows = s.frame_hw[0], cols = s.frame_hw[1];
        if (!sc[SC_SF_MARGINS] && (c.margins_given || (rows > 0 && cols > 0))) {
            if (c.margins_given) {
                for (int q = 0; q < 4; ++q) s.margins[q] = c.margin[q];
            } else {   // _maybe_set_margins(self.w, self.h) on the first frame with an image
                const double W = cols, H = rows;
                s.margins[0] = (float)sf_clamp(c.h_margin, 0.0, W);
                s.margins[1] = (float)sf_clamp(W - c.h_margin, 0.0, W);
                s.margins[2] = (float)sf_clamp(c.v_margin, 0.0, H);
                s.margins[3] = (float)sf_clamp(H - c.v_margin, 0.0, H);
            }
            sc[SC_SF_MARGINS] = 1;
        }
        const int frame = ++sc[SC_FRAME];
        double hth = c.high_th, nth = c.new_track_th, mth = c.match_th_first;
        if (c.dynamic) {
            int count = 0;
            for (int k = 0; k < D; ++k) count += s.dets[(size_t)k * 6 + 4] > (float)c.cth ? 1 : 0;
            const double lnc = c.log10_tab[count < 1 ? 1 : count];
            hth = sf_clamp(hth - c.high_th_m * lnc, 0.0, 1.0);
            nth = sf_clamp(nth + c.new_track_th_m * lnc, hth, 1.0);
            mth = sf_clamp(mth - c.match_th_first_m * lnc, 0.0, 0.67);
        }
        s.th[0] = hth; s.th[1] = nth; s.th[2] = mth;
        // _purge_stale_lost_tracks
        int nl = 0;
        for (int k = 0; k < sc[SC_N_LOST]; ++k) {
            const int t = s.lost[k];
            const int timeout = s.state[t] == SF_LOST_CENTRAL ? c.central_timeout : c.marginal_timeout;
            if (!(frame - s.last_frame[t] > timeout)) s.lost[nl++] = t;
        }
        sc[SC_N_LOST] = nl;
        int T = 0;
        for (int k = 0; k < sc[SC_N_ACTIVE]; ++k) s.pool[T++] = s.active[k];
        for (int k = 0; k < nl; ++k) s.pool[T++] = s.lost[k];
        int nh = 0, nm = 0;
        for (int k = 0; k < D; ++k) {
            const float sc4 = s.dets[(size_t)k * 6 + 4];
            if (sf_gt(sc4, hth, c.hth_f64)) s.high[nh++] = k;
            if ((float)c.low_th < sc4 && sf_lt(sc4, hth, c.hth_f64)) s.mid[nm++] = k;
        }
        s.mb[SF_MB_T] = T; s.mb[SF_MB_NH] = nh; s.mb[SF_MB_NM] = nm;
    }
    BMB_SYNC();
    const int T = s.mb[SF_MB_T], nh = s.mb[SF_MB_NH], nm = s.mb[SF_MB_NM];
    const int frame = sc[SC_FRAME];
    // ---- pass 1: every pool track x the definite detections, cost limit mth ----
    if (nh > 0 && T > 0) {
        sf_assign(s, nullptr, T, s.high, nh, false, s.th[2]);
    }
    if (BMB_TID == 0) {
        const double nth = s.th[1];
        for (int t = 0; t < CT; ++t) s.mark[t] = 0;
        for (int k = 0; k < sc[SC_N_ACTIVE]; ++k) s.mark[s.active[k]] = 1;   // slots in use
        for (int k = 0; k < sc[SC_N_LOST]; ++k) s.mark[s.lost[k]] = 1;
        int nn = 0, nu = 0, free_slot = 0;
        if (nh > 0) {
            if (T > 0)
                for (int r = 0; r < T; ++r) {
                    const int j = s.lap_x[r];
                    if (j < nh) {
                        const int t = s.pool[r];
                        sf_set(s, t, s.dets + (size_t)s.high[j] * 6, s.high[j], frame);   // leaves lost_tracks
                        s.nxt[nn++] = t;
                    } else {
                        s.unm[nu++] = r;
                    }
                }
            for (int k = 0; k < nh; ++k) {
                if (T > 0 && s.lap_y[k] < T) continue;
                const int row = s.high[k];
                const float* d = s.dets + (size_t)row * 6;
                if (!sf_gt(d[4], nth, c.nth_f64)) continue;
                while (free_slot < CT && s.mark[free_slot]) ++free_slot;
                if (free_slot >= CT) { sc[SC_ERROR] = ERR_TRACK_CAPACITY; break; }
                s.mark[free_slot] = 1;
                sf_set(s, free_slot, d, row, frame);
                s.id[free_slot] = sc[SC_NEXT_ID]++;
                s.nxt[nn++] = free_slot;
            }
        }
        s.mb[SF_MB_NU] = nu;
        s.mb[SF_MB_NN] = nn;
    }
    BMB_SYNC();
    // ---- pass 2: the unmatched pool x the possible detections, 1 - IoU, cost limit match_th_second.  The reference
    // tests `len(unmatched_tracks)`, still the initial empty array when no detection was definite ----
    const int nu = s.mb[SF_MB_NU];
    if (nm > 0 && nu > 0) {
        sf_assign(s, s.unm, nu, s.mid, nm, true, c.match_th_second);
    }
    if (BMB_TID == 0) {
        int nn = s.mb[SF_MB_NN];
        // next_lost_tracks: pass 1's unmatched pool minus pass 2's matches, or the whole pool on a frame with neither
        // kind of detection
        int nx = 0;
        int* next_lost = s.next_lost;
        for (int r = 0; r < nu; ++r) {
            const int t = s.pool[s.unm[r]];
            const int j = (nm > 0) ? s.lap_x[r] : nm;
            if (j < nm) {
                sf_set(s, t, s.dets + (size_t)s.mid[j] * 6, s.mid[j], frame);
                s.nxt[nn++] = t;
            } else {
                next_lost[nx++] = t;
            }
        }
        if (nh == 0 && nm == 0)
            for (int r = 0; r < T; ++r) next_lost[nx++] = s.pool[r];
        // lost_tracks: the old ones still lost keep their order and state; newcomers (from the active list) append
        int nl = 0;
        for (int k = 0; k < sc[SC_N_LOST]; ++k) {
            const int t = s.lost[k];
            if (s.state[t] != SF_ACTIVE) s.nlost[nl++] = t;
        }
        const float* m = s.margins;
        const bool ready = sc[SC_SF_MARGINS] != 0;
        for (int k = 0; k < nx; ++k) {
            const int t = next_lost[k];
            if (s.state[t] != SF_ACTIVE) continue;   // already in lost_tracks
            const float* b = s.box + (size_t)t * 4;
            const float u = b[0] + (b[2] - b[0]) / 2.0f, v = b[1] + (b[3] - b[1]) / 2.0f;
            const bool central = ready && (m[0] < u && u < m[1]) && (m[2] < v && v < m[3]);
            s.state[t] = central ? SF_LOST_CENTRAL : SF_LOST_MARGINAL;
            s.nlost[nl++] = t;
        }
        // Tracks matched this frame were marked active again by sf_set; an active track that is neither matched nor
        // in next_lost (pass 2 skipped) is dropped, as in the reference
        for (int k = 0; k < nl; ++k) s.lost[k] = s.nlost[k];
        for (int k = 0; k < nn; ++k) s.active[k] = s.nxt[k];
        sc[SC_N_LOST] = nl;
        sc[SC_N_ACTIVE] = nn;
        sc[SC_N_OUT] = nn;
        for (int k = 0; k < nn; ++k) {
            const int t = s.nxt[k];
            float* o = s.out + (size_t)k * 8;
            for (int q = 0; q < 4; ++q) o[q] = s.box[(size_t)t * 4 + q];
            o[4] = (float)s.id[t];
            o[5] = s.conf[t];
            o[6] = (float)(int)s.cls[t];   // Track.cls = int(cls)
            o[7] = (float)s.det_ind[t];
        }
    }
    BMB_SYNC();
}

}  // namespace bmb
