// ob_core.cuh -- OccluBoost per-stream, per-frame update (one CTA per stream) on top of the BoostTrack phases of
// bt_core.cuh; same conventions (the source also compiles for the host under BMB_HOSTSIM for GPU-less tests).
//
// Replaces (paths in the reference boxmot package), AABB path only:
//   trackers/bbox/occluboost/occluboost.py:185-483  OccluBoost._update_impl: original confidences, associate with a
//                                                   configurable lambda_emb multiplier, abnormal-motion updates, ReID
//                                                   recovery pass, low-confidence second pass, online GTA, tentative
//                                                   births, duplicate suppression, emit, cull + burial
//   trackers/bbox/occluboost/occluboost.py:485-708  _maybe_activate, _gta_appearance_recovery, _gta_bury_dead,
//                                                   _gta_evict_stale, _gta_resurrect (the gap rows are logged as events;
//                                                   the host interpolates and smooths them in flush_gta)
//   trackers/bbox/occluboost/occluboost.py:770-906  _xyxy_to_cxcywh, _compute_ams_alpha, _ams_update,
//                                                   _suppress_duplicate_emissions
// The extra passes read each track's CURRENT state: the reference does not refresh `unmatched_trks` after a pass, so a
// track recovered by one pass can be updated again by the next in the same frame.  Their appearance products are
// recomputed from the current track embedding with k_bt_embcost's arithmetic (float64, feature order).
#pragma once
#include "bt_core.cuh"
#include "lsa_sap.cuh"

namespace bmb {

constexpr int OB_EV = 13;   // event: grave id, death frame, frame, last box [4], new box [4], conf, cls

struct ObCfg {
    BtCfg bt;
    int use_second_pass, recovery_max_age, second_pass_max_age, second_pass_min_hits, confirm_hits, tentative_max_age;
    int ams_on, ams_buffer_size, gta, gta_min_track_length, gta_max_gap;
    double lambda_emb_mult, recovery_appearance_thresh, recovery_iou_thresh, feat_alpha, track_low_thresh,
        second_iou_thresh, second_appearance_thresh, new_track_thresh, instant_confirm_thresh, duplicate_iou_thresh,
        ams_alpha0, ams_threshold, ams_shrink_ratio, gta_appearance_thresh;
};

struct ObStream {
    BtStream b;
    // ---- persistent ----
    int* activated;    // [CT] is_activated
    double* ams;       // [CT][ams_buffer_size][4] ring of observed [cx, cy, w, h]
    int* ams_n;        // [CT] entries in the ring
    int* ams_head;     // [CT] next write position
    int* gv_meta;      // [2] graveyard entries, logged events
    int* gv_order;     // [CT] storage slot of each graveyard entry, insertion order
    int* gv_id;        // [CT] by storage slot
    int* gv_frame;
    double* gv_box;    // [CT][4] get_state() at death
    double* gv_conf;
    double* gv_cls;
    double* gv_emb;    // [CT][F]
    double* ev;        // [CT][OB_EV] resurrection events not yet taken by the host
    // ---- scratch ----
    int* unt;          // [CT] unmatched track positions, the reference's order
    int* elig;         // [CT]
    int* low;          // [CD] second-pass rows
    int* rowcol;       // [CD]
    int* nsrc;         // [CD] rows of the tracks appended this frame
    int* nid;          // [CD] their ids (-1: a fresh id)
    int* emit;         // [CT] emitted track positions
    double* gate;      // [CD][CT] gated similarity / cost of the current pass
    double* lsa_u; double* lsa_v; double* lsa_spc;
    int* scalars; long long* timers;   // b.scalars / b.timers, for lsa_solve and the phase clocks
    int* lsa_path; int* lsa_row4col; int* lsa_col4row; int* lsa_rem; int* lsa_sc; int* lsa_sr;
};

// ||(a, b)||: np.linalg.norm of a 2-vector is sqrt(dot) and the dot of two elements is fma(b, b, a * a)
BMB_FN double ob_norm2(double a, double b) { return sqrt(fma(b, b, a * a)); }

// np.mean of a 1-D float64 vector of n <= 128 entries: numpy's pairwise sum (8 accumulators from 8 entries on) / n
template <typename At>
BMB_FN double ob_np_mean(int n, At at) {
    double res;
    if (n < 8) {
        res = 0.0;
        for (int i = 0; i < n; ++i) res += at(i);
    } else {
        double r[8];
        for (int j = 0; j < 8; ++j) r[j] = at(j);
        int i = 8;
        for (; i < n - (n % 8); i += 8)
            for (int j = 0; j < 8; ++j) r[j] += at(i + j);
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
        for (; i < n; ++i) res += at(i);
    }
    return res / n;
}

// _compute_ams_alpha (occluboost.py:778-844) on the ring `buf` (B entries, n used, next write at head); appends the
// observation and returns alpha.  Python's max() keeps its first argument unless the second is larger.
BMB_FN double ob_ams_alpha(double* buf, int B, int& n, int& head, const double* box, double alpha0, double thr,
                           double shrink) {
    const double x1 = box[0], y1 = box[1], x2 = box[2], y2 = box[3];
    const double w = py_max(x2 - x1, 1e-6), h = py_max(y2 - y1, 1e-6);
    const double cur[4] = {x1 + 0.5 * w, y1 + 0.5 * h, w, h};
    auto push = [&]() {
        for (int q = 0; q < 4; ++q) buf[head * 4 + q] = cur[q];
        head = head + 1 == B ? 0 : head + 1;
        if (n < B) ++n;
    };
    if (n < 2) { push(); return 1.0; }
    const int first = (head - n + B) % B;
    auto at = [&](int i, int q) { return buf[((first + i) % B) * 4 + q]; };
    double cv[4], mv[4];
    for (int q = 0; q < 4; ++q) {
        cv[q] = cur[q] - at(n - 1, q);
        double acc = at(1, q) - at(0, q);
        for (int i = 2; i < n; ++i) acc += at(i, q) - at(i - 1, q);
        mv[q] = acc / (n - 1);
    }
    const double eps = 1e-6;
    const double cur_c = ob_norm2(cv[0], cv[1]), mean_c = ob_norm2(mv[0], mv[1]);
    const double cur_a = ob_norm2(cv[2], cv[3]), mean_a = ob_norm2(mv[2], mv[3]);
    const double ec = cur_c - mean_c, ea = cur_a - mean_a;
    const double d_c = (ec > 0.0 ? ec : 0.0) / (eps > mean_c ? eps : mean_c);
    const double d_a = (ea > 0.0 ? ea : 0.0) / (eps > mean_a ? eps : mean_a);
    const double alpha_c = d_c <= thr ? 1.0 : alpha0;
    const double alpha_a = d_a <= thr ? 1.0 : alpha0;
    double alpha = 0.5 * (alpha_c + alpha_a);
    const double cur_area = cur[2] * cur[3];
    const double mean_area = ob_np_mean(n, [&](int i) { return at(i, 2) * at(i, 3); });
    if (cur_area >= mean_area * shrink) alpha = 1.0;
    push();
    return alpha;
}

// _ams_update (occluboost.py:846-865) of slot t with detection row d; one thread
BMB_FN void ob_ams_update(const ObCfg& c, ObStream& s, int t, int d) {
    BtStream& b = s.b;
    double alpha = 1.0;
    if (c.ams_on) {
        const float* r = b.dets + d * 6;
        const double box[4] = {r[0], r[1], r[2], r[3]};
        alpha = ob_ams_alpha(s.ams + (size_t)t * c.ams_buffer_size * 4, c.ams_buffer_size, s.ams_n[t], s.ams_head[t], box,
                             c.ams_alpha0, c.ams_threshold, c.ams_shrink_ratio);
    }
    b.tsu[t] = 0;
    b.hit_streak[t] += 1;
    bt_kf_update(b.x + t * 8, b.P + t * 64, b.dz + d * 4, alpha);
    b.conf[t] = b.rconf[d];
    b.cls[t] = (double)b.dets[d * 6 + 5];
    b.det_ind[t] = (double)d;
}

BMB_FN void ob_maybe_activate(const ObCfg& c, ObStream& s, int t) {
    if (!s.activated[t] && s.b.hit_streak[t] >= c.confirm_hits) s.activated[t] = 1;
}

// detection row d . a float64 embedding, float64 accumulate in feature order (k_bt_embcost's arithmetic)
BMB_FN double ob_dot(const ObCfg& c, const ObStream& s, int d, const double* e) {
    const int F = c.bt.feat_dim;
    const float* r = s.b.embs + (size_t)d * F;
    double acc = 0.0;
    for (int q = 0; q < F; ++q) acc += (double)r[q] * e[q];
    return acc;
}

// one pass of AMS update + embedding EMA + activation for track slot t and row d, by warp 0
BMB_FN void ob_pass_update(const ObCfg& c, ObStream& s, int t, int d, bool emb) {
    if (BMB_LANE == 0) ob_ams_update(c, s, t, d);
    BMB_SYNCWARP();
    if (emb) bt_emb_update(c.bt, s.b, t, d, c.feat_alpha);
    if (BMB_LANE == 0) ob_maybe_activate(c, s, t);
    BMB_SYNCWARP();
}

// gate[r][j] = gate_at(r, j) for an R x C pass; returns whether any entry passes `pos` (the reference's `.any()`)
template <typename GateAt, typename Pos>
BMB_FN bool ob_fill_gate(ObStream& s, int R, int C, int LD, GateAt gate_at, Pos pos) {
    int* mb = s.b.free_l;
    if (BMB_TID == 0) mb[9] = 0;
    BMB_SYNC();
    for (int e = BMB_TID; e < R * C; e += BMB_NT) {
        const int r = e / C, j = e - r * C;
        const double g = gate_at(r, j);
        s.gate[(size_t)r * LD + j] = g;
        if (pos(g)) mb[9] = 1;
    }
    BMB_SYNC();
    const bool any = mb[9] != 0;
    BMB_SYNC();
    return any;
}

// drop the rows flagged in b.flag[0..n) from und (order kept); returns the new count
BMB_FN int ob_compact_und(ObStream& s, int n) {
    int* mb = s.b.free_l;
    if (BMB_TID == 0) {
        int m = 0;
        for (int r = 0; r < n; ++r)
            if (!s.b.flag[r]) s.b.und[m++] = s.b.und[r];
        mb[10] = m;
    }
    BMB_SYNC();
    const int m = mb[10];
    BMB_SYNC();
    return m;
}

// the two appearance-only passes over unmatched rows and eligible tracks (recovery: IoU-gated too, GTA: appearance
// only): gate, solve linear_sum_assignment(-gated), update the positive pairs in row order, drop their rows from und
BMB_FN int ob_appearance_pass(const ObCfg& c, ObStream& s, int n_und, int n_elig, double app_thresh, bool iou_gate) {
    BtStream& b = s.b;
    const int LD = c.bt.cap_tracks, F = c.bt.feat_dim;
    const bool any = ob_fill_gate(s, n_und, n_elig, LD, [&](int r, int j) {
        const int d = b.kdet[b.und[r]], t = b.tracks[s.elig[j]];
        const double sim = ob_dot(c, s, d, b.emb + (size_t)t * F);
        double g = sim;
        if (iou_gate) {
            double tb[4];
            bt_x_to_box(b.x + t * 8, tb);
            const float* q = b.dets + d * 6;
            if (bt_iou(q[0], q[1], q[2], q[3], tb[0], tb[1], tb[2], tb[3]) < c.recovery_iou_thresh) g = -1.0;
        }
        if (sim < app_thresh) g = -1.0;
        return g;
    }, [](double g) { return g > 0; });
    if (!any) return n_und;
    lsa_rect(s, b.cost, n_und, n_elig, [&](int r, int j) { return -s.gate[(size_t)r * LD + j]; }, s.rowcol);
    for (int r = BMB_TID; r < n_und; r += BMB_NT) b.flag[r] = 0;
    BMB_SYNC();
    if (BMB_WARP == 0)
        for (int r = 0; r < n_und; ++r) {
            const int j = s.rowcol[r];
            if (j < 0 || !(s.gate[(size_t)r * LD + j] > 0)) continue;
            if (BMB_LANE == 0) b.flag[r] = 1;
            ob_pass_update(c, s, b.tracks[s.elig[j]], b.kdet[b.und[r]], true);
        }
    BMB_SYNC();
    return ob_compact_und(s, n_und);
}

// unt filtered by pred into elig; returns the count
template <typename Pred>
BMB_FN int ob_eligible(ObStream& s, int n_unt, Pred pred) {
    int* mb = s.b.free_l;
    if (BMB_TID == 0) {
        int m = 0;
        for (int k = 0; k < n_unt; ++k)
            if (pred(s.b.tracks[s.unt[k]])) s.elig[m++] = s.unt[k];
        mb[11] = m;
    }
    BMB_SYNC();
    const int m = mb[11];
    BMB_SYNC();
    return m;
}

BMB_FN void ob_frame(const ObCfg& c, ObStream& s) {
    const BtCfg& bc = c.bt;
    BtStream& b = s.b;
    const int CT = bc.cap_tracks, CD = bc.cap_dets, F = bc.feat_dim;
    const int LD = CT;
    int* mb = b.free_l;
    int* free_slots = b.free_l + MB_COUNT;

    BtFrame f = bt_predict_phase(bc, b);
    bt_boost_phase(bc, b, f);
    bt_match_phase(bc, b, f, c.lambda_emb_mult);
    long long& _t_prev = f._t_prev;
    const int T = f.T, D = f.D, nk = f.nk, frame = f.frame;
    const bool use_emb = f.use_emb;
    const bool gta = c.gta && use_emb;
    int n_und = f.n_und;

    // ---- unmatched_trks: unmatched positions ascending, then the positions of the matches that failed the validity
    // test; the low-confidence rows of the second pass (original confidence in [track_low_thresh, det_thresh)) ----
    if (BMB_TID == 0) {
        for (int k = 0; k < T; ++k) b.mark[k] = 0;
        for (int i = 0; i < nk; ++i)
            if (b.mrow[i] >= 0) b.mark[b.mrow[i]] = 1;
        for (int i = 0; i < f.n_ufail; ++i) b.mark[b.tmp_b[i]] = 1;
        int m = 0;
        for (int k = 0; k < T; ++k)
            if (!b.mark[k]) s.unt[m++] = k;
        for (int i = 0; i < f.n_ufail; ++i) s.unt[m++] = b.tmp_b[i];
        mb[12] = m;
        int nl = 0;
        if (c.use_second_pass)
            for (int d = 0; d < D; ++d) {
                const double o = (double)b.dets[d * 6 + 4];
                if (!(b.rconf[d] >= bc.det_thresh) && o >= c.track_low_thresh && o < bc.det_thresh) s.low[nl++] = d;
            }
        mb[13] = nl;
    }
    BMB_SYNC();
    const int n_unt = mb[12], n_low = mb[13];
    BMB_SYNC();

    // ---- matched updates: AMS Kalman update, embedding EMA with the trust-based alpha, activation ----
    for (int i = BMB_TID; i < nk; i += BMB_NT)
        if (b.mrow[i] >= 0) ob_ams_update(c, s, b.tracks[b.mrow[i]], b.kdet[i]);
    BMB_SYNC();
    if (use_emb)
        for (int i = BMB_WARP; i < nk; i += BMB_NW) {
            if (b.mrow[i] < 0) continue;
            const int d = b.kdet[i];
            const double trust = (b.rconf[d] - bc.det_thresh) / (1 - bc.det_thresh);
            bt_emb_update(bc, b, b.tracks[b.mrow[i]], d, 0.95 + (1 - 0.95) * (1 - trust));
        }
    BMB_SYNC();
    for (int i = BMB_TID; i < nk; i += BMB_NT)
        if (b.mrow[i] >= 0) ob_maybe_activate(c, s, b.tracks[b.mrow[i]]);
    BMB_SYNC();

    // ---- ReID recovery pass (occluboost.py:291-339) ----
    if (use_emb && n_unt > 0 && n_und > 0) {
        const int ne = ob_eligible(s, n_unt, [&](int t) { return b.tsu[t] <= c.recovery_max_age; });
        if (ne > 0) n_und = ob_appearance_pass(c, s, n_und, ne, c.recovery_appearance_thresh, true);
    }

    // ---- low-confidence second pass (occluboost.py:341-392): cost 1 - IoU, 1 where IoU or appearance fail ----
    if (c.use_second_pass && n_unt > 0 && n_low > 0) {
        const int ne = ob_eligible(s, n_unt, [&](int t) {
            return b.tsu[t] <= c.second_pass_max_age && b.hit_streak[t] >= c.second_pass_min_hits && s.activated[t];
        });
        if (ne > 0) {
            const bool any = ob_fill_gate(s, n_low, ne, LD, [&](int r, int j) {
                const int d = s.low[r], t = b.tracks[s.elig[j]];
                double tb[4];
                bt_x_to_box(b.x + t * 8, tb);
                const float* q = b.dets + d * 6;
                const double io = bt_iou(q[0], q[1], q[2], q[3], tb[0], tb[1], tb[2], tb[3]);
                double v = 1.0 - io;
                if (io < c.second_iou_thresh) v = 1.0;
                if (use_emb && ob_dot(c, s, d, b.emb + (size_t)t * F) < c.second_appearance_thresh) v = 1.0;
                return v;
            }, [](double v) { return v < 1.0; });
            if (any) {
                lsa_rect(s, b.cost, n_low, ne, [&](int r, int j) { return s.gate[(size_t)r * LD + j]; }, s.rowcol);
                if (BMB_WARP == 0)
                    for (int r = 0; r < n_low; ++r) {
                        const int j = s.rowcol[r];
                        if (j < 0 || s.gate[(size_t)r * LD + j] >= 1.0) continue;
                        ob_pass_update(c, s, b.tracks[s.elig[j]], s.low[r], use_emb);
                    }
                BMB_SYNC();
            }
        }
    }

    // ---- online GTA: appearance-only recovery (occluboost.py:499-575) ----
    if (gta && n_und > 0 && n_unt > 0) {
        const int ne = ob_eligible(s, n_unt, [&](int t) {
            return b.tsu[t] <= c.gta_max_gap && b.age[t] >= c.gta_min_track_length;
        });
        if (ne > 0) n_und = ob_appearance_pass(c, s, n_und, ne, c.gta_appearance_thresh, false);
    }

    // ---- new tracks: resurrections from the graveyard (occluboost.py:610-708), then births ----
    int n_new = 0;
    const int n_grave = s.gv_meta[0];
    if (gta && n_und > 0 && n_grave > 0) {
        const bool any = ob_fill_gate(s, n_und, n_grave, LD, [&](int r, int g) {
            const double sim = ob_dot(c, s, b.kdet[b.und[r]], s.gv_emb + (size_t)s.gv_order[g] * F);
            return sim < c.gta_appearance_thresh ? -1.0 : sim;
        }, [](double g) { return g > 0; });
        if (any) {
            lsa_rect(s, b.cost, n_und, n_grave, [&](int r, int g) { return -s.gate[(size_t)r * LD + g]; }, s.rowcol);
            if (BMB_TID == 0) {
                for (int g = 0; g < n_grave; ++g) b.mark[g] = 0;   // graveyard positions resurrected
                for (int r = 0; r < n_und; ++r) {
                    b.flag[r] = 0;
                    const int g = s.rowcol[r];
                    if (g < 0 || !(s.gate[(size_t)r * LD + g] > 0)) continue;
                    const int d = b.kdet[b.und[r]];
                    if (b.rconf[d] < c.new_track_thresh) continue;
                    b.flag[r] = 1;
                    b.mark[g] = 1;
                    const int gs = s.gv_order[g];
                    s.nsrc[n_new] = d;
                    s.nid[n_new] = s.gv_id[gs];
                    ++n_new;
                    const int ne = s.gv_meta[1];
                    if (ne >= CT) { b.scalars[SC_ERROR] = ERR_TRACK_CAPACITY; continue; }
                    double* ev = s.ev + (size_t)ne * OB_EV;
                    const double* z = b.dz + d * 4;
                    const double x0[4] = {z[0], z[1], py_max(z[2], 1e-4), py_max(z[3], 1e-4)};
                    ev[0] = s.gv_id[gs]; ev[1] = s.gv_frame[gs]; ev[2] = frame;
                    for (int q = 0; q < 4; ++q) ev[3 + q] = s.gv_box[gs * 4 + q];
                    bt_x_to_box(x0, ev + 7);
                    ev[11] = s.gv_conf[gs]; ev[12] = s.gv_cls[gs];
                    s.gv_meta[1] = ne + 1;
                }
                int m = 0;
                for (int g = 0; g < n_grave; ++g)
                    if (!b.mark[g]) s.gv_order[m++] = s.gv_order[g];
                s.gv_meta[0] = m;
                mb[14] = n_new;
            }
            BMB_SYNC();
            n_new = mb[14];
            BMB_SYNC();
            n_und = ob_compact_und(s, n_und);
        }
    }
    const int n_res = n_new;
    if (BMB_TID == 0) {
        for (int r = 0; r < n_und; ++r) {
            const int d = b.kdet[b.und[r]];
            if (b.rconf[d] >= c.new_track_thresh) { s.nsrc[n_new] = d; s.nid[n_new] = -1; ++n_new; }
        }
        mb[14] = n_new;
    }
    BMB_SYNC();
    n_new = mb[14];
    BMB_PHASE(4);
    // free slots: not in the list
    for (int k = BMB_TID; k < CT; k += BMB_NT) b.mark[k] = 0;
    BMB_SYNC();
    for (int k = BMB_TID; k < T; k += BMB_NT) b.mark[b.tracks[k]] = 1;
    BMB_SYNC();
    if (BMB_WARP == 0) {
        int nfree = 0;
        for (int k0 = 0; k0 < CT && nfree < n_new; k0 += BMB_NL) {
            const int k = k0 + BMB_LANE;
            const bool p = k < CT && !b.mark[k];
            const unsigned m = BMB_BALLOT(p);
#if BMB_DEVICE
            const int pos = nfree + __popc(m & ((1u << BMB_LANE) - 1u));
#else
            const int pos = nfree;
#endif
            if (p && pos < n_new) free_slots[pos] = k;
            nfree += BMB_POPC(m);
        }
        if (BMB_LANE == 0) {
            if (nfree < n_new) b.scalars[SC_ERROR] = ERR_TRACK_CAPACITY;
            mb[5] = nfree < n_new ? nfree : n_new;
        }
    }
    BMB_SYNC();
    const int n_made = mb[5];
    {
        const int id0 = b.scalars[SC_NEXT_ID];
        for (int k = BMB_TID; k < n_made; k += BMB_NT) {
            const int t = free_slots[k], d = s.nsrc[k];
            double* x = b.x + t * 8;
            double* P = b.P + t * 64;
            const double* z = b.dz + d * 4;
            x[0] = z[0]; x[1] = z[1]; x[2] = py_max(z[2], 1e-4); x[3] = py_max(z[3], 1e-4);
            for (int i = 4; i < 8; ++i) x[i] = 0.0;
            for (int i = 0; i < 64; ++i) P[i] = 0.0;
            for (int i = 0; i < 8; ++i) P[i * 9] = i < 4 ? 10.0 : 10000.0;
            b.age[t] = 0; b.hit_streak[t] = 0; b.tsu[t] = 0;
            b.id[t] = k < n_res ? s.nid[k] : id0 + 1 + (k - n_res);
            b.conf[t] = b.rconf[d];
            b.cls[t] = (double)b.dets[d * 6 + 5];
            b.det_ind[t] = (double)d;
            s.activated[t] = k < n_res || b.rconf[d] >= c.instant_confirm_thresh || c.confirm_hits <= 1;
            s.ams_n[t] = 0; s.ams_head[t] = 0;
            b.tracks[T + k] = t;
        }
        if (use_emb)
            for (int k = BMB_WARP; k < n_made; k += BMB_NW) {
                const int t = free_slots[k];
                const float* e = b.embs + (size_t)s.nsrc[k] * F;
                for (int q = BMB_LANE; q < F; q += BMB_NL) b.emb[(size_t)t * F + q] = (double)e[q];
            }
    }
    BMB_SYNC();
    int n_all = T + n_made;
    BMB_PHASE(5);

    // ---- emit (occluboost.py:432-460): updated this frame, activated, enough hits or warm-up; then duplicate
    // suppression in list order (the younger of a pair above duplicate_iou_thresh leaves the list, unburied), then
    // filter_outputs ----
    if (BMB_TID == 0) {
        int ne = 0;
        for (int k = 0; k < n_all; ++k) {
            const int t = b.tracks[k];
            if (b.tsu[t] < 1 && s.activated[t] && (b.hit_streak[t] >= bc.min_hits || frame <= bc.min_hits)) s.emit[ne++] = k;
        }
        for (int k = 0; k < n_all; ++k) b.flag[k] = 0;   // dropped by duplicate suppression, by list position
        if (ne > 1 && 0.0 < c.duplicate_iou_thresh && c.duplicate_iou_thresh < 1.0) {
            for (int i = 0; i < ne; ++i) {
                if (b.flag[s.emit[i]]) continue;
                double bi[4];
                bt_x_to_box(b.x + b.tracks[s.emit[i]] * 8, bi);
                for (int j = i + 1; j < ne; ++j) {
                    if (b.flag[s.emit[j]]) continue;
                    double bj[4];
                    bt_x_to_box(b.x + b.tracks[s.emit[j]] * 8, bj);
                    if (bt_iou(bi[0], bi[1], bi[2], bi[3], bj[0], bj[1], bj[2], bj[3]) >= c.duplicate_iou_thresh) {
                        const int ai = b.age[b.tracks[s.emit[i]]], aj = b.age[b.tracks[s.emit[j]]];
                        b.flag[ai >= aj ? s.emit[j] : s.emit[i]] = 1;
                    }
                }
            }
        }
        int n_out = 0;
        for (int i = 0; i < ne; ++i) {
            const int t = b.tracks[s.emit[i]];
            if (b.flag[s.emit[i]]) continue;
            double bx[4];
            bt_x_to_box(b.x + t * 8, bx);
            const double w = bx[2] - bx[0], h = bx[3] - bx[1];
            if (!((w / h <= bc.ar_thresh) && (w * h > bc.min_box_area))) continue;
            if (n_out >= CD) { b.scalars[SC_ERROR] = ERR_DET_CAPACITY; break; }
            float* o = b.out + n_out * 8;
            o[0] = (float)bx[0]; o[1] = (float)bx[1]; o[2] = (float)bx[2]; o[3] = (float)bx[3];
            o[4] = (float)b.id[t]; o[5] = (float)b.conf[t]; o[6] = (float)b.cls[t]; o[7] = (float)b.det_ind[t];
            ++n_out;
        }
        // cull (occluboost.py:465-478): confirmed tracks live max_age frames, tentative ones tentative_max_age; the
        // dead that are old enough are buried in list order, then stale graves are evicted
        int keep = 0;
        for (int k = 0; k < n_all; ++k) {
            if (b.flag[k]) continue;
            const int t = b.tracks[k];
            const bool alive = b.tsu[t] <= bc.max_age && (s.activated[t] || b.tsu[t] <= c.tentative_max_age);
            if (alive) { b.tracks[keep++] = t; continue; }
            if (!gta || b.age[t] < c.gta_min_track_length) continue;
            int ng = s.gv_meta[0];
            if (ng >= CT) { b.scalars[SC_ERROR] = ERR_TRACK_CAPACITY; continue; }
            for (int k2 = 0; k2 < CT; ++k2) b.mark[k2] = 0;   // storage slots in use
            for (int g = 0; g < ng; ++g) b.mark[s.gv_order[g]] = 1;
            int gs = 0;
            while (b.mark[gs]) ++gs;
            s.gv_order[ng] = gs;
            s.gv_id[gs] = b.id[t];
            s.gv_frame[gs] = frame;
            bt_x_to_box(b.x + t * 8, s.gv_box + gs * 4);
            s.gv_conf[gs] = b.conf[t];
            s.gv_cls[gs] = b.cls[t];
            for (int q = 0; q < F; ++q) s.gv_emb[(size_t)gs * F + q] = b.emb[(size_t)t * F + q];
            s.gv_meta[0] = ng + 1;
        }
        int m = 0;
        for (int g = 0; g < s.gv_meta[0]; ++g)
            if (!(frame - s.gv_frame[s.gv_order[g]] > c.gta_max_gap)) s.gv_order[m++] = s.gv_order[g];
        s.gv_meta[0] = m;
        b.scalars[SC_N_ACTIVE] = keep;
        b.scalars[SC_FRAME] = frame;
        b.scalars[SC_N_OUT] = n_out;
        b.scalars[SC_NEXT_ID] += n_made > n_res ? n_made - n_res : 0;
    }
    BMB_SYNC();
    BMB_PHASE(6);
}

}  // namespace bmb
