// tests/_obsim/obsim.cpp -- TEST INFRASTRUCTURE ONLY.
// Compiles boxmot_b200/csrc/ob_core.cuh for the host (BMB_HOSTSIM: one "thread") so the OccluBoost device core can be
// checked against the golden vectors without a GPU.  Built by tests/obsim.py with g++ into a temporary directory and
// never linked into libboxmot_b200.so.
#define BMB_HOSTSIM 1
#include <cstring>
#include <vector>

#include "tracker_layout.h"

using namespace bmb;

struct ObSim {
    ObCfg cfg;
    ObStream s;
    std::vector<uint8_t> mem;
    std::vector<float> dets, embs;
    std::vector<double> pow_table;
    int n_dets;
    double warp[8];
};

extern "C" {

int obsim_cfg_size() { return (int)sizeof(ObCfg); }
int obsim_ev_width() { return OB_EV; }

ObSim* obsim_create(const ObCfg* cfg, const double* conf_pow, int n_pow) {
    ObSim* h = new ObSim();
    h->cfg = *cfg;
    h->pow_table.assign(conf_pow, conf_pow + n_pow);
    h->cfg.bt.conf_pow = h->pow_table.data();
    h->cfg.bt.n_conf_pow = n_pow;
    h->mem.assign(carve_ob(h->cfg, nullptr, nullptr, nullptr), 0);
    carve_ob(h->cfg, h->mem.data(), &h->s, nullptr);
    const BtCfg& b = cfg->bt;
    h->dets.assign((size_t)b.cap_dets * 6, 0.f);
    h->embs.assign((size_t)b.cap_dets * (b.feat_dim > 0 ? b.feat_dim : 1), 0.f);
    h->s.b.dets = h->dets.data();
    h->s.b.n_dets = &h->n_dets;
    h->s.b.embs = b.with_reid ? h->embs.data() : nullptr;
    for (double& w : h->warp) w = 0.0;
    h->s.b.warp = h->warp;
    return h;
}

void obsim_destroy(ObSim* h) { delete h; }

void obsim_set_warp(ObSim* h, const double* w6) {
    for (int i = 0; i < 6; ++i) h->warp[i] = w6[i];
    h->warp[6] = 1.0;
}

// returns the number of output rows, or -(error code)
int obsim_update(ObSim* h, const float* dets, int n, const float* embs, float* out) {
    const BtCfg& c = h->cfg.bt;
    BtStream& s = h->s.b;
    if (n > c.cap_dets) return -ERR_DET_CAPACITY;
    h->n_dets = n;
    if (n) memcpy(h->dets.data(), dets, sizeof(float) * 6 * n);
    if (c.with_reid && embs) {
        const int F = c.feat_dim;
        memcpy(h->embs.data(), embs, sizeof(float) * F * n);
        // the wide k_bt_embcost: every row against every live slot, float64 accumulate in feature order
        for (int d = 0; d < n; ++d)
            for (int k = 0; k < s.scalars[SC_N_ACTIVE]; ++k) {
                const int t = s.tracks[k];
                double acc = 0.0;
                for (int q = 0; q < F; ++q) acc += (double)embs[(size_t)d * F + q] * s.emb[(size_t)t * F + q];
                s.embq[(size_t)d * c.cap_tracks + t] = acc;
            }
    }
    ob_frame(h->cfg, h->s);
    h->warp[6] = 0.0;   // a warp applies to one frame
    if (s.scalars[SC_ERROR]) return -s.scalars[SC_ERROR];
    const int m = s.scalars[SC_N_OUT];
    memcpy(out, s.out, sizeof(float) * 8 * m);
    return m;
}

// ids, means, covariances and is_activated of the live tracks in list order
int obsim_snapshot(ObSim* h, int* ids, double* xs, double* Ps, int* act, int cap) {
    const BtStream& s = h->s.b;
    int n = 0;
    for (int k = 0; k < s.scalars[SC_N_ACTIVE] && n < cap; ++k, ++n) {
        const int t = s.tracks[k];
        ids[n] = s.id[t];
        act[n] = h->s.activated[t];
        memcpy(xs + (size_t)n * 8, s.x + (size_t)t * 8, sizeof(double) * 8);
        memcpy(Ps + (size_t)n * 64, s.P + (size_t)t * 64, sizeof(double) * 64);
    }
    return n;
}

// the resurrection events logged since the last call
int obsim_take_events(ObSim* h, double* ev, int cap) {
    const int n = h->s.gv_meta[1] < cap ? h->s.gv_meta[1] : cap;
    memcpy(ev, h->s.ev, sizeof(double) * OB_EV * n);
    h->s.gv_meta[1] = 0;
    return n;
}

// AMS gain factor of a buffer of n observations (oldest first) and a new box, for the numpy comparison
double obsim_ams_alpha(const double* obs, int n, int B, const double* box, double alpha0, double thr, double shrink) {
    std::vector<double> ring((size_t)B * 4);
    int cnt = 0, head = 0;
    for (int i = 0; i < n; ++i) {
        for (int q = 0; q < 4; ++q) ring[head * 4 + q] = obs[i * 4 + q];
        head = head + 1 == B ? 0 : head + 1;
        if (cnt < B) ++cnt;
    }
    return ob_ams_alpha(ring.data(), B, cnt, head, box, alpha0, thr, shrink);
}

}  // extern "C"
