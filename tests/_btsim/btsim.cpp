// tests/_btsim/btsim.cpp -- TEST INFRASTRUCTURE ONLY.
// Compiles boxmot_b200/csrc/bt_core.cuh for the host (BMB_HOSTSIM: one "thread") so the BoostTrack device core can be
// checked against the golden vectors without a GPU.  Built by tests/btsim.py with g++ into a temporary directory and
// never linked into libboxmot_b200.so.
#define BMB_HOSTSIM 1
#include <cstring>
#include <vector>

#include "tracker_layout.h"

using namespace bmb;

struct BtSim {
    BtCfg cfg;
    BtStream s;
    std::vector<uint8_t> mem;
    std::vector<float> dets, embs;
    std::vector<double> pow_table;
    int n_dets;
    double warp[8];
};

extern "C" {

int btsim_cfg_size() { return (int)sizeof(BtCfg); }

BtSim* btsim_create(const BtCfg* cfg, const double* conf_pow, int n_pow) {
    BtSim* h = new BtSim();
    h->cfg = *cfg;
    h->pow_table.assign(conf_pow, conf_pow + n_pow);
    h->cfg.conf_pow = h->pow_table.data();
    h->cfg.n_conf_pow = n_pow;
    h->mem.assign(carve_bt(h->cfg, nullptr, nullptr, nullptr), 0);
    carve_bt(h->cfg, h->mem.data(), &h->s, nullptr);
    h->dets.assign((size_t)cfg->cap_dets * 6, 0.f);
    h->embs.assign((size_t)cfg->cap_dets * (cfg->feat_dim > 0 ? cfg->feat_dim : 1), 0.f);
    h->s.dets = h->dets.data();
    h->s.n_dets = &h->n_dets;
    h->s.embs = cfg->with_reid ? h->embs.data() : nullptr;
    for (double& w : h->warp) w = 0.0;
    h->s.warp = h->warp;
    return h;
}

void btsim_destroy(BtSim* h) { delete h; }

void btsim_set_warp(BtSim* h, const double* w6) {
    for (int i = 0; i < 6; ++i) h->warp[i] = w6[i];
    h->warp[6] = 1.0;
}

// returns the number of output rows, or -(error code)
int btsim_update(BtSim* h, const float* dets, int n, const float* embs, float* out) {
    const BtCfg& c = h->cfg;
    if (n > c.cap_dets) return -ERR_DET_CAPACITY;
    h->n_dets = n;
    if (n) memcpy(h->dets.data(), dets, sizeof(float) * 6 * n);
    if (c.with_reid && embs) {
        const int F = c.feat_dim;
        memcpy(h->embs.data(), embs, sizeof(float) * F * n);
        // the wide k_bt_embcost: every row against every live slot, float64 accumulate in feature order
        for (int d = 0; d < n; ++d)
            for (int k = 0; k < h->s.scalars[SC_N_ACTIVE]; ++k) {
                const int t = h->s.tracks[k];
                double acc = 0.0;
                for (int q = 0; q < F; ++q) acc += (double)embs[(size_t)d * F + q] * h->s.emb[(size_t)t * F + q];
                h->s.embq[(size_t)d * c.cap_tracks + t] = acc;
            }
    }
    bt_frame(c, h->s);
    h->warp[6] = 0.0;   // a warp applies to one frame
    if (h->s.scalars[SC_ERROR]) return -h->s.scalars[SC_ERROR];
    const int m = h->s.scalars[SC_N_OUT];
    memcpy(out, h->s.out, sizeof(float) * 8 * m);
    return m;
}

int btsim_snapshot(BtSim* h, int* ids, double* xs, double* Ps, int cap) {
    int n = 0;
    for (int k = 0; k < h->s.scalars[SC_N_ACTIVE] && n < cap; ++k, ++n) {
        const int t = h->s.tracks[k];
        ids[n] = h->s.id[t];
        memcpy(xs + (size_t)n * 8, h->s.x + (size_t)t * 8, sizeof(double) * 8);
        memcpy(Ps + (size_t)n * 64, h->s.P + (size_t)t * 64, sizeof(double) * 64);
    }
    return n;
}

}  // extern "C"
