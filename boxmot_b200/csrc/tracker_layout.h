// tracker_layout.h -- carve one contiguous allocation into the per-stream SoA views of TrkStream.
// Shared by the CUDA engine (device allocation) and by the host-simulation test harness.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "tracker_core.cuh"

namespace bmb {

struct Carver {
    uint8_t* base;
    size_t off;
    template <typename T>
    T* take(size_t n) {
        off = (off + 255) & ~(size_t)255;
        T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
        off += n * sizeof(T);
        return p;
    }
};

// Fills `s` with pointers into `base` (which may be null to only measure) and returns the bytes needed.
// `persistent_bytes` receives the size of the leading region that must be zeroed on reset.
inline size_t carve_stream(const TrkCfg& c, uint8_t* base, TrkStream* s, size_t* persistent_bytes) {
    const size_t CT = (size_t)c.cap_tracks, CD = (size_t)c.cap_dets, F = (size_t)(c.feat_dim > 0 ? c.feat_dim : 1);
    Carver k{base, 0};
    TrkStream t{};
    t.scalars = k.take<int>(SC_COUNT);
    t.timers = k.take<long long>(16);
    t.state = k.take<int>(CT);
    t.activated = k.take<int>(CT);
    t.id = k.take<int>(CT);
    t.frame_id = k.take<int>(CT);
    t.start_frame = k.take<int>(CT);
    t.tracklet_len = k.take<int>(CT);
    t.hist_n = k.take<int>(CT);
    t.in_removed = k.take<int>(CT);
    t.removed_ring = k.take<int>(c.removed_cap > 0 ? (size_t)c.removed_cap : 1);
    t.active = k.take<int>(CT);
    t.lost = k.take<int>(CT);
    t.conf = k.take<float>(CT);
    t.cls = k.take<float>(CT);
    t.det_ind = k.take<float>(CT);
    t.hist_cls = k.take<float>(CT * HIST_CAP);
    t.hist_sum = k.take<float>(CT * HIST_CAP);
    t.mean = k.take<double>(CT * 8);
    t.cov = k.take<double>(CT * 64);
    t.smooth = k.take<float>(CT * F);
    if (persistent_bytes) *persistent_bytes = k.off;
    // scratch
    t.dxywh = k.take<float>(CD * 4);
    t.dmeas = k.take<float>(CD * 4);
    t.dxyxy = k.take<float>(CD * 4);
    t.dfeat = k.take<float>(CD * F);
    t.embd = k.take<double>(CT * CD);
    t.cost = k.take<double>(CT * CD);
    t.txyxy = k.take<double>(CT * 4);
    t.first = k.take<int>(CD);
    t.second = k.take<int>(CD);
    t.rest = k.take<int>(CD);
    t.pool = k.take<int>(CT);
    t.unconf = k.take<int>(CT);
    t.rtracked = k.take<int>(CT);
    t.act_l = k.take<int>(CT + CD);
    t.refind_l = k.take<int>(CT);
    t.lostnow_l = k.take<int>(CT);
    t.remnow_l = k.take<int>(CT);
    t.tmp_a = k.take<int>(CT);
    t.tmp_b = k.take<int>(CT);
    t.mark = k.take<int>(CT);
    t.free_l = k.take<int>(CT + MB_COUNT);
    t.ema_slot = k.take<int>(CD);
    t.ema_det = k.take<int>(CD);
    t.lap_x = k.take<int>(CT);
    t.lap_y = k.take<int>(CD);
    t.lap_u = k.take<double>(CT);
    t.lap_v = k.take<double>(CD);
    t.lap_spc = k.take<double>(CD);
    t.lap_path = k.take<int>(CD);
    t.lap_insc = k.take<int>(CD);
    t.lap_tl = k.take<int>(CD);
    t.lap_sc = k.take<int>(CD);
    t.csr_ptr = k.take<int>(CT + 1);
    t.csr_col = k.take<int>(CT * CD);
    t.out = k.take<float>(CD * 8);
    if (s) *s = t;
    return (k.off + 255) & ~(size_t)255;
}

}  // namespace bmb

#include "docs_core.cuh"

namespace bmb {

inline size_t carve_docs(const DocsCfg& c, uint8_t* base, DocsStream* s, size_t* persistent_bytes) {
    const size_t CT = (size_t)c.cap_tracks, CD = (size_t)c.cap_dets, F = (size_t)(c.feat_dim > 0 ? c.feat_dim : 1);
    const size_t MX = CT > CD ? CT : CD;
    Carver k{base, 0};
    DocsStream t{};
    t.scalars = k.take<int>(SC_COUNT);
    t.timers = k.take<long long>(16);
    t.gap = k.take<int>(CT); t.has_saved = k.take<int>(CT); t.observed = k.take<int>(CT);
    t.age = k.take<int>(CT); t.hits = k.take<int>(CT); t.hit_streak = k.take<int>(CT); t.tsu = k.take<int>(CT);
    t.id = k.take<int>(CT); t.obs_age = k.take<int>(CT * DOCS_RING); t.obs_n = k.take<int>(CT);
    t.has_vel = k.take<int>(CT); t.tracks = k.take<int>(CT);
    t.x = k.take<double>(CT * 8); t.P = k.take<double>(CT * 56);
    t.xs = k.take<double>(CT * 8); t.Ps = k.take<double>(CT * 56);
    t.zlast = k.take<double>(CT * 4);
    t.conf = k.take<double>(CT); t.cls = k.take<double>(CT); t.det_ind = k.take<double>(CT);
    t.last_obs = k.take<double>(CT * 5); t.obs_box = k.take<double>(CT * DOCS_RING * 5);
    t.vel = k.take<double>(CT * 2);
    t.emb = k.take<double>(CT * F);
    if (persistent_bytes) *persistent_bytes = k.off;
    t.kdet = k.take<int>(CD);
    t.dbox = k.take<double>(CD * 5);
    t.dalpha = k.take<double>(CD);
    t.tbox = k.take<double>(CT * 4);
    t.kobs = k.take<double>(CT * 5);
    t.iou = k.take<double>(CD * CT);
    t.embc = k.take<double>(CD * CT);
    t.embq = k.take<double>(CD * CT);
    t.cost = k.take<double>(MX * MX);   // lapjv's zero-padded square problem
    t.top = k.take<double>(2 * (CD + CT));
    t.mrow = k.take<int>(CD);
    t.und = k.take<int>(CD);
    t.unt = k.take<int>(CT);
    t.tmp_a = k.take<int>(CT + CD);
    t.tmp_b = k.take<int>(MX);
    t.mark = k.take<int>(CT);
    t.free_l = k.take<int>(CT + MB_COUNT);
    t.lap_x = k.take<int>(MX); t.lap_y = k.take<int>(MX);
    t.lap_u = k.take<double>(MX); t.lap_v = k.take<double>(MX); t.lap_spc = k.take<double>(MX);
    t.lap_path = k.take<int>(MX); t.lap_insc = k.take<int>(MX); t.lap_tl = k.take<int>(MX); t.lap_sc = k.take<int>(MX);
    t.csr_ptr = k.take<int>(MX + 1);
    t.csr_col = k.take<int>(CT * CD);
    t.out = k.take<float>(CD * 8);
    if (s) *s = t;
    return (k.off + 255) & ~(size_t)255;
}

}  // namespace bmb

#include "ss_core.cuh"

namespace bmb {

// StrongSORT: the sample gallery ([CT][budget][F] float32) dominates; it sits behind the zero-on-reset region
// (gal_n = 0 is all a reset needs).
inline size_t carve_ss(const SsCfg& c, uint8_t* base, SsStream* s, size_t* persistent_bytes) {
    const size_t CT = (size_t)c.cap_tracks, CD = (size_t)c.cap_dets, F = (size_t)(c.feat_dim > 0 ? c.feat_dim : 1);
    const size_t B = (size_t)(c.budget > 0 ? c.budget : 1);
    const size_t MX = CT > CD ? CT : CD;
    Carver k{base, 0};
    SsStream t{};
    t.scalars = k.take<int>(SC_COUNT);
    t.timers = k.take<long long>(16);
    t.state = k.take<int>(CT); t.id = k.take<int>(CT); t.hits = k.take<int>(CT); t.age = k.take<int>(CT);
    t.tsu = k.take<int>(CT); t.gal_n = k.take<int>(CT); t.gal_head = k.take<int>(CT);
    t.pend_kind = k.take<int>(CT); t.pend_det = k.take<int>(CT); t.tracks = k.take<int>(CT);
    t.conf = k.take<double>(CT); t.cls = k.take<double>(CT); t.det_ind = k.take<double>(CT);
    t.mean = k.take<double>(CT * 8); t.cov = k.take<double>(CT * 64);
    if (persistent_bytes) *persistent_bytes = k.off;
    t.feat = k.take<float>(CT * F);
    t.gal = k.take<float>(CT * B * F);
    t.dfeatn = k.take<float>(CD * F);
    t.appc = k.take<float>(CT * CD);
    t.kdet = k.take<int>(CD);
    t.dtlwh = k.take<double>(CD * 4); t.dxyah = k.take<double>(CD * 4); t.dconf = k.take<double>(CD);
    t.tproj = k.take<double>(CT * 20);
    t.cost = k.take<double>(CT * CD);
    t.conf_pos = k.take<int>(CT); t.cand = k.take<int>(CT); t.unta = k.take<int>(CT); t.mdet = k.take<int>(CT);
    t.rowcol = k.take<int>(CT); t.colrow = k.take<int>(CD); t.und = k.take<int>(CD); t.und2 = k.take<int>(CD);
    t.tmp_a = k.take<int>(CT + CD); t.mark = k.take<int>(CT); t.free_l = k.take<int>(CT + MB_COUNT);
    t.set_buf = k.take<int>(4 * (8 * CT + 16));
    t.lsa_u = k.take<double>(MX); t.lsa_v = k.take<double>(MX); t.lsa_spc = k.take<double>(MX);
    t.lsa_path = k.take<int>(MX); t.lsa_row4col = k.take<int>(MX); t.lsa_col4row = k.take<int>(MX);
    t.lsa_rem = k.take<int>(MX); t.lsa_sr = k.take<int>(MX); t.lsa_sc = k.take<int>(MX);
    t.out = k.take<float>(CD * 8);
    if (s) *s = t;
    return (k.off + 255) & ~(size_t)255;
}

}  // namespace bmb

#include "bt_core.cuh"

namespace bmb {

// BoostTrack: the (row, track) matrices dominate the scratch
inline size_t carve_bt(const BtCfg& c, uint8_t* base, BtStream* s, size_t* persistent_bytes) {
    const size_t CT = (size_t)c.cap_tracks, CD = (size_t)c.cap_dets, F = (size_t)(c.feat_dim > 0 ? c.feat_dim : 1);
    const size_t MX = CT > CD ? CT : CD;
    Carver k{base, 0};
    BtStream t{};
    t.scalars = k.take<int>(SC_COUNT);
    t.timers = k.take<long long>(16);
    t.age = k.take<int>(CT); t.hit_streak = k.take<int>(CT); t.tsu = k.take<int>(CT); t.id = k.take<int>(CT);
    t.tracks = k.take<int>(CT);
    t.x = k.take<double>(CT * 8); t.P = k.take<double>(CT * 64);
    t.conf = k.take<double>(CT); t.cls = k.take<double>(CT); t.det_ind = k.take<double>(CT);
    t.emb = k.take<double>(CT * F);
    if (persistent_bytes) *persistent_bytes = k.off;
    t.rconf = k.take<double>(CD); t.dz = k.take<double>(CD * 4); t.tbox = k.take<double>(CT * 5);
    t.iou = k.take<double>(CD * CT); t.md = k.take<double>(CD * CT); t.ex = k.take<double>(CD * CT);
    t.embq = k.take<double>(CD * CT);
    t.colsum = k.take<double>(CT); t.ovmax = k.take<double>(CD);
    t.kdet = k.take<int>(CD); t.cand = k.take<int>(CD); t.flag = k.take<int>(MX); t.mrow = k.take<int>(CD);
    t.und = k.take<int>(CD); t.tmp_a = k.take<int>(CT); t.tmp_b = k.take<int>(CT); t.mark = k.take<int>(CT);
    t.free_l = k.take<int>(CT + MB_COUNT);
    t.cost = k.take<double>(MX * MX);
    t.lap_x = k.take<int>(MX); t.lap_y = k.take<int>(MX);
    t.lap_u = k.take<double>(MX); t.lap_v = k.take<double>(MX); t.lap_spc = k.take<double>(MX);
    t.lap_path = k.take<int>(MX); t.lap_insc = k.take<int>(MX); t.lap_tl = k.take<int>(MX); t.lap_sc = k.take<int>(MX);
    t.out = k.take<float>(CD * 8);
    if (s) *s = t;
    return (k.off + 255) & ~(size_t)255;
}

}  // namespace bmb

#include "ob_core.cuh"

namespace bmb {

// OccluBoost: BoostTrack's stream, then its own state.  The persistent part is the whole stream (reset clears it all):
// the graveyard and the event log sit after BoostTrack's scratch.
inline size_t carve_ob(const ObCfg& c, uint8_t* base, ObStream* s, size_t* persistent_bytes) {
    const size_t CT = (size_t)c.bt.cap_tracks, CD = (size_t)c.bt.cap_dets;
    const size_t F = (size_t)(c.bt.feat_dim > 0 ? c.bt.feat_dim : 1), B = (size_t)(c.ams_buffer_size > 0 ? c.ams_buffer_size : 1);
    const size_t MX = CT > CD ? CT : CD;
    ObStream t{};
    const size_t nb = carve_bt(c.bt, base, s ? &t.b : nullptr, nullptr);
    Carver k{base, nb};
    t.activated = k.take<int>(CT); t.ams = k.take<double>(CT * B * 4); t.ams_n = k.take<int>(CT); t.ams_head = k.take<int>(CT);
    t.gv_meta = k.take<int>(2); t.gv_order = k.take<int>(CT); t.gv_id = k.take<int>(CT); t.gv_frame = k.take<int>(CT);
    t.gv_box = k.take<double>(CT * 4); t.gv_conf = k.take<double>(CT); t.gv_cls = k.take<double>(CT);
    t.gv_emb = k.take<double>(CT * F); t.ev = k.take<double>(CT * OB_EV);
    t.unt = k.take<int>(CT); t.elig = k.take<int>(CT); t.low = k.take<int>(CD); t.rowcol = k.take<int>(CD);
    t.nsrc = k.take<int>(CD); t.nid = k.take<int>(CD); t.emit = k.take<int>(CT);
    t.gate = t.b.ex;
    t.scalars = t.b.scalars; t.timers = t.b.timers;   // BoostTrack's softmax scratch is free once the association is done
    t.lsa_u = k.take<double>(MX); t.lsa_v = k.take<double>(MX); t.lsa_spc = k.take<double>(MX);
    t.lsa_path = k.take<int>(MX); t.lsa_row4col = k.take<int>(MX); t.lsa_col4row = k.take<int>(MX);
    t.lsa_rem = k.take<int>(MX); t.lsa_sc = k.take<int>(MX); t.lsa_sr = k.take<int>(MX);
    const size_t total = (k.off + 255) & ~(size_t)255;
    if (persistent_bytes) *persistent_bytes = total;
    if (s) *s = t;
    return total;
}

}  // namespace bmb


#include "sf_core.cuh"

namespace bmb {

// SFSORT: boxes and the two ordered lists persist; lapjv's (CT + CD) square problem dominates the scratch
inline size_t carve_sf(const SfCfg& c, uint8_t* base, SfStream* s, size_t* persistent_bytes) {
    const size_t CT = (size_t)c.cap_tracks, CD = (size_t)c.cap_dets, MX = CT + CD;
    Carver k{base, 0};
    SfStream t{};
    t.scalars = k.take<int>(SC_COUNT);
    t.timers = k.take<long long>(16);
    t.box = k.take<float>(CT * 4); t.conf = k.take<float>(CT); t.cls = k.take<float>(CT);
    t.det_ind = k.take<int>(CT); t.last_frame = k.take<int>(CT); t.id = k.take<int>(CT); t.state = k.take<int>(CT);
    t.active = k.take<int>(CT); t.lost = k.take<int>(CT); t.margins = k.take<float>(4);
    if (persistent_bytes) *persistent_bytes = k.off;
    t.high = k.take<int>(CD); t.mid = k.take<int>(CD);
    t.pool = k.take<int>(CT); t.unm = k.take<int>(CT); t.nxt = k.take<int>(CT); t.nlost = k.take<int>(CT);
    t.mark = k.take<int>(CT); t.next_lost = k.take<int>(CT); t.mb = k.take<int>(SF_MB_COUNT); t.th = k.take<double>(4);
    t.free_l = k.take<int>(MB_COUNT);
    t.cost = k.take<double>(MX * MX);
    t.lap_x = k.take<int>(MX); t.lap_y = k.take<int>(MX); t.lap_v = k.take<double>(MX); t.lap_spc = k.take<double>(MX);
    t.lap_path = k.take<int>(MX); t.lap_insc = k.take<int>(MX); t.lap_tl = k.take<int>(MX); t.lap_sc = k.take<int>(MX);
    t.out = k.take<float>(CD * 8);
    if (s) *s = t;
    return (k.off + 255) & ~(size_t)255;
}

}  // namespace bmb
