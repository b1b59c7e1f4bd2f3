// tests/_sfsim/sfsim.cpp -- TEST INFRASTRUCTURE ONLY.
// Compiles boxmot_b200/csrc/sf_core.cuh for the host (BMB_HOSTSIM: one "thread") so the SFSORT device core can be
// checked against the golden vectors without a GPU.  Built by tests/sfsim.py with g++ into a temporary directory and
// never linked into libboxmot_b200.so.
#define BMB_HOSTSIM 1
#include <cmath>
#include <cstring>
#include <vector>

#include "tracker_layout.h"

using namespace bmb;

struct SfSim {
    SfCfg cfg;
    SfStream s;
    std::vector<uint8_t> mem;
    std::vector<float> dets;
    std::vector<double> log10_tab;
    int n_dets;
    int frame_hw[2];
};

extern "C" {

int sfsim_cfg_size() { return (int)sizeof(SfCfg); }

SfSim* sfsim_create(const SfCfg* cfg) {
    SfSim* h = new SfSim();
    h->cfg = *cfg;
    h->log10_tab.resize((size_t)cfg->cap_dets + 1);
    if (cfg->log10_tab) h->log10_tab.assign(cfg->log10_tab, cfg->log10_tab + cfg->cap_dets + 1);   // the engine's rule
    else sf_log10_table(cfg->cap_dets + 1, h->log10_tab.data());
    h->cfg.log10_tab = h->log10_tab.data();
    h->cfg.n_log10 = (int)h->log10_tab.size();
    h->mem.assign(carve_sf(h->cfg, nullptr, nullptr, nullptr), 0);
    carve_sf(h->cfg, h->mem.data(), &h->s, nullptr);
    h->dets.assign((size_t)cfg->cap_dets * 6, 0.f);
    h->s.dets = h->dets.data();
    h->s.n_dets = &h->n_dets;
    h->frame_hw[0] = h->frame_hw[1] = 0;
    h->s.frame_hw = h->frame_hw;
    return h;
}

void sfsim_destroy(SfSim* h) { delete h; }

// returns the number of output rows, or -(error code)
int sfsim_update(SfSim* h, const float* dets, int n, int rows, int cols, float* out) {
    h->n_dets = n;
    if (rows > 0 && cols > 0) { h->frame_hw[0] = rows; h->frame_hw[1] = cols; }
    if (n && n <= h->cfg.cap_dets) memcpy(h->dets.data(), dets, sizeof(float) * 6 * n);
    sf_frame(h->cfg, h->s);
    if (h->s.scalars[SC_ERROR]) return -h->s.scalars[SC_ERROR];
    const int m = h->s.scalars[SC_N_OUT];
    memcpy(out, h->s.out, sizeof(float) * 8 * m);
    return m;
}

// which = 0: active ids; 1: lost ids; 2: lost states
int sfsim_list(SfSim* h, int which, int* out) {
    const int n = h->s.scalars[which == 0 ? SC_N_ACTIVE : SC_N_LOST];
    const int* l = which == 0 ? h->s.active : h->s.lost;
    for (int k = 0; k < n; ++k) out[k] = which == 2 ? h->s.state[l[k]] : h->s.id[l[k]];
    return n;
}

}  // extern "C"
