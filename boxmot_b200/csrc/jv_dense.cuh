// jv_dense.cuh -- dense Jonker-Volgenant linear assignment with the SAME tie-breaking as lap.lapjv
// (restated for the oracle in oracle/lapjv.c): column reduction + reduction transfer, two passes of augmenting row
// reduction, shortest-augmenting-path augmentation with lapjv's column-list bookkeeping.
//
// DeepOCSORT's association (association/association.py:20-24, 105-123; deepocsort.py:433) calls
// lapjv(extend_cost=True) WITHOUT a cost limit on matrices full of exact zeros (no overlap, no velocity, gated
// appearance): many optima tie, lapjv's choice among them decides the ORDER in which unmatched detections become
// tracks and therefore the track ids.  Bit-exact ids need the same algorithm, not just an exact optimum.
//
// One warp runs the solver.  Control flow is lapjv's sequential control flow; the O(n) inner scans are spread
// over the lanes with reductions that reproduce the sequential result exactly: minima are combined as
// (value, lowest index), the two-smallest search of the row reduction as lexicographic (value, index) pairs, and
// the relaxation loop of the path search updates all columns in parallel and then replays the rare
// "distance equals the band minimum" events in ascending position order.
#pragma once
#include "tracker_core.cuh"

namespace bmb {

#if BMB_DEVICE
#define BMB_SYNC_OR(p) __syncthreads_or(p)
#define BMB_PREFETCH_L1(ptr) asm volatile("prefetch.global.L1 [%0];" ::"l"(ptr))
#define BMB_FFS(m) (__ffs(m) - 1)
#else
#define BMB_SYNC_OR(p) (p)
#define BMB_PREFETCH_L1(ptr) ((void)0)
#define BMB_FFS(m) 0
#endif

// CTA-wide augmentation phase of the dense JV solver (same results as the one-warp loop in jv_dense_solve).
//
// BASELINE config 3 (512 detections against ~1500 live tracks, 3/4 of them unobserved) spends its time in lapjv's
// _scan_dense: ~7e5 band columns per frame, each relaxing the ~600 columns not yet in the ready band (4.4e8 relaxed
// entries, profiled on the oracle).  Here every thread of the CTA owns the positions hi + tid, hi + tid + NT, ... of
// the column list, so one band column costs one pass over shared-memory state plus one barrier:
//   * relax all positions >= hi at once; "distance equals the band minimum" events (1 % of the steps) are recorded
//     as ballot masks per (chunk, warp) and replayed by thread 0 in ascending position order -- the order in which
//     the sequential scan meets them, which is what lapjv's tie-breaking is made of (a position is never rewritten
//     before its own replay: swaps only write hit positions and positions < every later hit);
//   * a final hit ends the search exactly as in lapjv; entries relaxed beyond it only touch d/pred of columns that
//     are not on the augmenting path and are re-initialised by the next search;
//   * rows >= zrow are the zero padding of extend_cost: their entries are not loaded; for real rows the next band
//     column's row is prefetched into L1 while the current one is relaxed.
// find_dense stays on warp 0 (its hits are inherently sequential), everything else is thread-strided.
template <typename S>
BMB_FN void jv_augment_wide(S& s, int n, int ld, int zrow, int n_free, int* mbx) {
    int* x = s.lap_x; int* y = s.lap_y; double* v = s.lap_v; double* d = s.lap_spc;
    int* pred = s.lap_path; int* cols = s.lap_tl; const int* free_rows = s.lap_sc;
    unsigned* hitm = reinterpret_cast<unsigned*>(s.lap_insc);   // `once` flags are dead after the reduction transfer
    const double* c = s.cost;
    const double BIG = 1.7976931348623157e308;
    const int lane = BMB_LANE;
    long long n_steps = 0;   // band columns scanned (diagnostic counter 13)
    long long c_find = 0, c_replay = 0, c_edge = 0;   // cycles: _find_dense (11), hit replays (14), init + prices + path (15)
    for (int f = 0; f < n_free; ++f) {
        const int start = free_rows[f];
        int lo = 0, hi = 0, n_ready = 0, band = 0, final_j = -1;
        long long c0 = BMB_CLOCK();
        {
            const bool zr = start >= zrow;
            const double* cs = c + (size_t)start * ld;
            for (int j = BMB_TID; j < n; j += BMB_NT) { cols[j] = j; pred[j] = start; d[j] = (zr ? 0.0 : cs[j]) - v[j]; }
        }
        BMB_SYNC();
        c_edge += BMB_CLOCK() - c0;
        while (final_j == -1) {
            if (lo == hi) {
                c0 = BMB_CLOCK();
                if (BMB_WARP == 0) {   // _find_dense, as in jv_dense_solve
                    int h2 = lo + 1;
                    double mind = d[cols[lo]];
                    for (int k0 = lo + 1; k0 < n; k0 += BMB_NL) {
                        const int k = k0 + lane;
                        const int j = k < n ? cols[k] : -1;
                        const double dj = k < n ? d[j] : BIG;
#if BMB_DEVICE
                        double pm = dj;
                        for (int o = 1; o < 32; o <<= 1) {
                            const double t = __shfl_up_sync(0xffffffffu, pm, o);
                            if (lane >= o && t < pm) pm = t;
                        }
                        const double excl = __shfl_up_sync(0xffffffffu, pm, 1);
                        const double before = lane == 0 ? mind : (excl < mind ? excl : mind);
                        unsigned hits = __ballot_sync(0xffffffffu, k < n && dj <= before);
                        // degenerate blocks (thousands of equal distances): when no column of the chunk is strictly
                        // below the minimum and the hits are exactly the positions h2, h2+1, ... every swap of the
                        // sequential scan is a self-swap -- advance h2 without touching the list
                        if (hits && k0 == h2 && (hits & (hits + 1u)) == 0u &&
                            !__any_sync(0xffffffffu, k < n && dj < mind)) {
                            h2 += __popc(hits);
                            hits = 0u;
                        }
                        while (hits) {
                            const int src = __ffs(hits) - 1;
                            hits &= hits - 1;
                            const double dh = __shfl_sync(0xffffffffu, dj, src);
                            const int jh = __shfl_sync(0xffffffffu, j, src);
                            if (dh < mind) { h2 = lo; mind = dh; }
                            if (lane == 0) { cols[k0 + src] = cols[h2]; cols[h2] = jh; }
                            ++h2;
                            __syncwarp();
                        }
#else
                        if (dj <= mind) {
                            if (dj < mind) { h2 = lo; mind = dj; }
                            cols[k] = cols[h2];
                            cols[h2++] = j;
                        }
#endif
                    }
                    BMB_SYNCWARP();
                    int last = -1;   // lapjv keeps the LAST free column of the band
                    for (int k = lo + lane; k < h2; k += BMB_NL)
                        if (y[cols[k]] < 0) last = k;
#if BMB_DEVICE
                    for (int o = 16; o > 0; o >>= 1) { const int t = __shfl_xor_sync(0xffffffffu, last, o); if (t > last) last = t; }
#endif
                    if (lane == 0) {
                        mbx[0] = h2;
                        mbx[1] = last >= 0 ? cols[last] : -1;
                    }
                }
                BMB_SYNC();
                n_ready = lo;
                band = lo;
                hi = mbx[0];
                final_j = mbx[1];
                BMB_SYNC();
                c_find += BMB_CLOCK() - c0;
            }
            // _scan_dense over the ready band, one barrier per band column
            while (lo != hi && final_j == -1) {
                ++n_steps;
                const int j = cols[lo++];
                const int i = y[j];
                const double mind = d[j];
                const bool zr = i >= zrow;
                const double* ci = c + (size_t)i * ld;
                const double h = (zr ? 0.0 : ci[j]) - v[j] - mind;
                const double* cn = nullptr;   // row of the next band column (prefetch target)
                if (lo != hi) {
                    const int jn = cols[lo];
                    const int in = y[jn];
                    if (in < zrow) { cn = c + (size_t)in * ld; if (BMB_TID == 0) BMB_PREFETCH_L1(cn + jn); }
                }
                const int hi0 = hi;
                int any = 0;
                int slot = BMB_WARP;
                for (int k0 = hi0; k0 < n; k0 += BMB_NT, slot += BMB_NW) {
                    const int k = k0 + BMB_TID;
                    bool hit = false;
                    if (k < n) {
                        const int jj = cols[k];
                        const double r = (zr ? 0.0 : ci[jj]) - v[jj] - h;
                        if (cn) BMB_PREFETCH_L1(cn + jj);
                        if (r < d[jj]) {
                            d[jj] = r;
                            pred[jj] = i;
                            hit = (r == mind);
                        }
                    }
                    const unsigned m = BMB_BALLOT(hit);
                    if (lane == 0) hitm[slot] = m;
                    any |= (m != 0u);
                }
                any = BMB_SYNC_OR(any);
                if (any) {
                    c0 = BMB_CLOCK();
                    if (BMB_TID == 0) {
                        // replay the "equals the band minimum" events in ascending position order
                        int h2 = hi0, fj = -1;
                        const int n_slots = ((n - hi0 + BMB_NT - 1) / BMB_NT) * BMB_NW;
                        for (int q = 0; q < n_slots && fj < 0; ++q) {
                            unsigned m = hitm[q];
                            const int base = hi0 + (q / BMB_NW) * BMB_NT + (q % BMB_NW) * BMB_NL;
                            while (m) {
                                const int kq = base + BMB_FFS(m);
                                m &= m - 1;
                                const int jq = cols[kq];
                                if (y[jq] < 0) { fj = jq; break; }
                                cols[kq] = cols[h2];
                                cols[h2] = jq;
                                ++h2;
                            }
                        }
                        mbx[0] = h2;
                        mbx[1] = fj;
                    }
                    BMB_SYNC();
                    hi = mbx[0];
                    final_j = mbx[1];
                    BMB_SYNC();
                    c_replay += BMB_CLOCK() - c0;
                }
            }
        }
        c0 = BMB_CLOCK();
        // price update for the columns scanned before the last band, then augment along the path
        {
            const double mind = d[cols[band]];
            for (int k = BMB_TID; k < n_ready; k += BMB_NT) { const int j = cols[k]; v[j] += d[j] - mind; }
        }
        if (BMB_TID == 0) {
            int j = final_j, i = -1;
            while (i != start) {
                i = pred[j];
                y[j] = i;
                const int prev = x[i];
                x[i] = j;
                j = prev;
            }
        }
        BMB_SYNC();
        c_edge += BMB_CLOCK() - c0;
    }
    if (BMB_TID == 0) { s.timers[13] += n_steps; s.timers[11] += c_find; s.timers[14] += c_replay; s.timers[15] += c_edge; }
}

// ---- column-owned CTA-wide augmentation (wide == 2) --------------------------------------------------------------
// jv_augment_wide walks the open part of the column LIST, so every relaxed entry costs a chain of shared-memory reads
// (cols[k] -> v[jj], d[jj]) per band column.  Here every thread OWNS the columns
// tid, tid + NT, ... and keeps their distance d and the negated price (0.0 - v) in registers; "open" (position >= hi)
// is a bit per owned column refreshed from the inverse permutation pos[] whenever the band changes.  A band column
// then costs one pass of register arithmetic and one barrier.  The band-minimum hits are recovered in POSITION order
// (lapjv's order) by the same mask-and-replay pass as in jv_augment_wide: an open column's distance equals the band
// minimum iff it was a hit of this step (shared-memory copies of d are refreshed at every _find_dense and on hits).
// _find_dense is split into a parallel part (chunk minima -> running minimum at every chunk start -> hit masks, all
// warps) and the inherently sequential replay of the hits by one thread.
#if BMB_DEVICE
#define JV_OWN 12        // owned columns per thread: n <= JV_OWN * blockDim
#define JV_CHUNKS 128    // 32-position chunks _find_dense can hold: n <= 4096
#else
#define JV_OWN 4096
#define JV_CHUNKS 4104
#endif

//
// Mode 3 (the default) adds exact shortcuts selected by the bits of `feat` (all on by default; the bits exist so that a
// hardware run can bisect them), found by counting on the BASELINE config-3 frames (oracle instrumented: 5.5e5 band
// columns and 1.3e6 list swaps per frame):
//   * NO-OP BAND COLUMNS.  In a search that starts from a zero-padding row every open column has
//     d <= (0.0 - v) (its initial value; d only decreases).  A band column owned by another zero-padding row whose own
//     distance never improved has h = ((0.0 - v[j]) - d[j]) == 0.0, so its relaxation value is r = (0.0 - v[jj]) - 0.0
//     >= d[jj] for every open column: nothing changes, bit for bit.  91 % of the band columns of those frames are of
//     this kind; the warps walk over runs of them (32 positions per ballot, no barrier, nothing is written).
//   * PARALLEL _find_dense TAIL.  After the last strict decrease of the running minimum (position k*, found with the
//     chunk minima) lapjv's swaps are a queue rotation: the m-th column at the minimum goes to cell lo + m and the
//     element it displaces goes to that column's old position k_m, possibly to be displaced again by swap k_m - lo.
//     The final cell of a displaced element is therefore the first iterate >= H of q -> k_q - lo (H = columns at the
//     minimum), computed by pointer jumping over all cells at once; the columns at the minimum go to lo + rank.
//     93-99 % of the swaps of those frames sit in such tails (570-740 swaps each); thread 0 still replays the part
//     before k* and short tails.
//   * HIT LIST.  A band-minimum hit of the relaxation is usually alone: the owning thread appends its list position
//     (pos[]) to a short shared list; thread 0 sorts and replays it instead of the CTA scanning every open position
//     for "distance == band minimum" (the mask pass remains the overflow path).
#define JV_F_SKIP 1
#define JV_F_PARFIND 2
#define JV_F_HITLIST 4
#define JV_F_ARRWIDE 8  // CTA-wide augmenting row reduction (jv_arr_wide)
#define JV_PAR_MIN 48   // shortest tail (columns at the minimum) handled by the parallel pass
#define JV_HITCAP 32    // hit list capacity
template <typename S>
BMB_FN void jv_augment_owned(S& s, int n, int ld, int zrow, int n_free, int* mbx, const int feat) {
    const bool fast = (feat & JV_F_PARFIND) != 0;
    const bool skip_noop = (feat & JV_F_SKIP) != 0;
    const bool hitlist = (feat & JV_F_HITLIST) != 0;
    int* x = s.lap_x; int* y = s.lap_y; double* v = s.lap_v; double* d = s.lap_spc;
    int* pred = s.lap_path; int* cols = s.lap_tl; const int* free_rows = s.lap_sc;
    int* pos = s.lap_insc;   // inverse of cols (the `once` flags are dead after the reduction transfer)
    const double* c = s.cost;
    const double BIG = 1.7976931348623157e308;
    const int lane = BMB_LANE;
#if BMB_DEVICE
    __shared__ double cmin[JV_CHUNKS];
    __shared__ unsigned hmask[JV_CHUNKS];
    __shared__ unsigned smask[JV_CHUNKS];
    __shared__ unsigned emask[JV_CHUNKS];   // positions at the global minimum (fast mode)
    __shared__ int erank[JV_CHUNKS];        // exclusive prefix count of emask
    __shared__ double sh_min;
    __shared__ int sh_aux[2];               // [0] k*: first position at the global minimum, [1] number of emask bits
    __shared__ int sh_nhit;
    __shared__ int hitpos[JV_HITCAP];
#else
    static double cmin[JV_CHUNKS];
    static unsigned hmask[JV_CHUNKS];
    static unsigned smask[JV_CHUNKS];
    static unsigned emask[JV_CHUNKS];
    static int erank[JV_CHUNKS];
    static double sh_min;
    static int sh_aux[2];
    static int sh_nhit;
    static int hitpos[JV_HITCAP];
#endif
    if (BMB_TID == 0) sh_nhit = 0;   // ordered before the first relaxation by the barrier after the first init
    long long n_skip = 0;   // no-op band columns walked over (diagnostic counter 7)
    double dq[JV_OWN];    // distance of the owned columns (registers on the device)
    double nvq[JV_OWN];   // 0.0 - v[jj]: a zero-padding row relaxes with r = (0.0 - v) - h, the same two operations
    long long n_steps = 0, c_find = 0, c_replay = 0, c_edge = 0;
    for (int f = 0; f < n_free; ++f) {
        const int start = free_rows[f];
        int lo = 0, hi = 0, n_ready = 0, band = 0, final_j = -1;
        unsigned open = 0u;   // bit q: owned column q is still outside the band (position >= hi)
#if !BMB_DEVICE
        unsigned char open_h[JV_OWN];
#endif
        long long c0 = BMB_CLOCK();
        const bool start_zr = start >= zrow;
        {
            const bool zr = start_zr;
            const double* cs = c + (size_t)start * ld;
#pragma unroll
            for (int q = 0; q < JV_OWN; ++q) {
                const int jj = BMB_TID + q * BMB_NT;
                if (jj < n) {
                    const double vj = v[jj];
                    const double dj = (zr ? 0.0 : cs[jj]) - vj;
                    dq[q] = dj;
                    nvq[q] = 0.0 - vj;
                    d[jj] = dj;
                    cols[jj] = jj;
                    pos[jj] = jj;
                    pred[jj] = start;
#if BMB_DEVICE
                    open |= 1u << q;
#else
                    open_h[q] = 1;
#endif
                }
#if BMB_DEVICE
                else { dq[q] = -BIG; nvq[q] = 0.0; }   // a closed column carries -BIG: `r < dq` never holds
#else
                else break;
#endif
            }
        }
        BMB_SYNC();
        c_edge += BMB_CLOCK() - c0;
        while (final_j == -1) {
            if (lo == hi) {
                // ---- _find_dense over positions [lo, n): distances of the open columns go back to shared memory ----
                c0 = BMB_CLOCK();
#pragma unroll
                for (int q = 0; q < JV_OWN; ++q) {
                    const int jj = BMB_TID + q * BMB_NT;
#if BMB_DEVICE
                    if ((open >> q) & 1u) d[jj] = dq[q];
#else
                    if (jj >= n) break;
                    if (open_h[q]) d[jj] = dq[q];
#endif
                }
                BMB_SYNC();
                const int base = lo + 1;
                const int C = (n - base + BMB_NL - 1) / BMB_NL;   // chunks of one warp width
                // (1) chunk minima
                for (int cc = BMB_WARP; cc < C; cc += BMB_NW) {
                    const int k = base + cc * BMB_NL + lane;
                    double m = k < n ? d[cols[k]] : BIG;
#if BMB_DEVICE
                    for (int o = 16; o > 0; o >>= 1) { const double t = __shfl_xor_sync(0xffffffffu, m, o); if (t < m) m = t; }
#endif
                    if (lane == 0) cmin[cc] = m;
                }
                BMB_SYNC();
                // (2) running minimum at the start of every chunk (exclusive prefix minimum, seeded with position lo)
                if (BMB_WARP == 0) {
                    double run = d[cols[lo]];
                    for (int c0i = 0; c0i < C; c0i += BMB_NL) {
                        const int cc = c0i + lane;
                        const double mc = cc < C ? cmin[cc] : BIG;
#if BMB_DEVICE
                        double pm = mc;
                        for (int o = 1; o < 32; o <<= 1) {
                            const double t = __shfl_up_sync(0xffffffffu, pm, o);
                            if (lane >= o && t < pm) pm = t;
                        }
                        const double excl = __shfl_up_sync(0xffffffffu, pm, 1);
                        const double before = lane == 0 ? run : (excl < run ? excl : run);
                        const double tot = __shfl_sync(0xffffffffu, pm, 31);
#else
                        const double before = run;
                        const double tot = mc;
#endif
                        if (cc < C) cmin[cc] = before;
                        if (tot < run) run = tot;
                    }
                    if (lane == 0) {   // global minimum; k* = lo when the first column of the list already holds it
                        sh_min = run;
                        sh_aux[0] = d[cols[lo]] == run ? lo : 0x7fffffff;
                        sh_aux[1] = 0;
                    }
                }
                BMB_SYNC();
                // (3) hit masks: a position is a hit when its distance is at or below the running minimum before it
                for (int cc = BMB_WARP; cc < C; cc += BMB_NW) {
                    const int k = base + cc * BMB_NL + lane;
                    const double dj = k < n ? d[cols[k]] : BIG;
                    const double at_start = cmin[cc];
#if BMB_DEVICE
                    double pm = dj;
                    for (int o = 1; o < 32; o <<= 1) {
                        const double t = __shfl_up_sync(0xffffffffu, pm, o);
                        if (lane >= o && t < pm) pm = t;
                    }
                    const double excl = __shfl_up_sync(0xffffffffu, pm, 1);
                    const double before = lane == 0 ? at_start : (excl < at_start ? excl : at_start);
#else
                    const double before = at_start;
#endif
                    const unsigned hm = BMB_BALLOT(k < n && dj <= before);
                    const unsigned sm = BMB_BALLOT(k < n && dj < at_start);   // the minimum moves inside this chunk
                    if (lane == 0) { hmask[cc] = hm; smask[cc] = sm; }
                    if (fast) {
                        const unsigned em = BMB_BALLOT(k < n && dj == sh_min);
                        if (lane == 0) {
                            emask[cc] = em;
                            if (em) BMB_ATOMIC_MIN(&sh_aux[0], base + cc * BMB_NL + BMB_FFS(em));
                        }
                    }
                }
                BMB_SYNC();
                if (fast) {
                    // (4') thread 0 replays the hits BEFORE k* (earlier running minima), one warp counts the columns at
                    // the global minimum per chunk; the tail from k* on is a queue rotation (see the header comment)
                    const int kstar = sh_aux[0];
                    const int off = kstar == lo ? 1 : 0;   // position lo itself is column 0 of the band, in place
                    if (BMB_WARP == (BMB_NW > 1 ? 1 : 0)) {
                        int carry = 0;
                        for (int c0i = 0; c0i < C; c0i += BMB_NL) {
                            const int cc = c0i + lane;
                            const int cnt = cc < C ? BMB_POPC(emask[cc]) : 0;
#if BMB_DEVICE
                            int inc = cnt;
                            for (int o = 1; o < 32; o <<= 1) {
                                const int t = __shfl_up_sync(0xffffffffu, inc, o);
                                if (lane >= o) inc += t;
                            }
                            const int tot = __shfl_sync(0xffffffffu, inc, 31);
#else
                            const int inc = cnt;
                            const int tot = cnt;
#endif
                            if (cc < C) erank[cc] = carry + inc - cnt;
                            carry += tot;
                        }
                        if (lane == 0) sh_aux[1] = carry;
                    }
                    if (BMB_TID == 0 && kstar > lo + 1) {
                        int h2 = lo + 1;
                        double mind = d[cols[lo]];
                        for (int cc = 0; cc < C; ++cc) {
                            const int kb = base + cc * BMB_NL;
                            if (kb >= kstar) break;
                            unsigned m = hmask[cc];
                            if (kstar - kb < BMB_NL) m &= (1u << (kstar - kb)) - 1u;   // positions below k* only
                            if (!m) continue;
                            if (smask[cc] == 0u && kb == h2 && (m & (m + 1u)) == 0u) { h2 += BMB_POPC(m); continue; }
                            while (m) {
                                const int k = kb + BMB_FFS(m);
                                m &= m - 1;
                                const int j = cols[k];
                                const double dj = d[j];
                                if (dj < mind) { h2 = lo; mind = dj; }
                                cols[k] = cols[h2];
                                cols[h2] = j;
                                ++h2;
                            }
                        }
                    }
                    BMB_SYNC();
                    const int H = off + sh_aux[1];   // columns at the minimum: the new band is [lo, lo + H)
                    if (H < JV_PAR_MIN) {
                        if (BMB_TID == 0) {
                            int h2 = lo + off;
                            for (int cc = 0; cc < C; ++cc) {
                                unsigned m = emask[cc];
                                const int kb = base + cc * BMB_NL;
                                while (m) {
                                    const int k = kb + BMB_FFS(m);
                                    m &= m - 1;
                                    const int j = cols[k];
                                    const int other = cols[h2];
                                    cols[k] = other;
                                    cols[h2] = j;
                                    ++h2;
                                }
                            }
                        }
                    } else {
                        int* J = pos;   // J[q] = k_q - lo: where swap q sends the element of cell lo + q (pos is rebuilt in (5))
                        for (int cc = BMB_WARP; cc < C; cc += BMB_NW) {
                            const unsigned em = emask[cc];
                            if ((em >> lane) & 1u)
                                J[off + erank[cc] + BMB_POPC(em & ((1u << lane) - 1u))] = base + cc * BMB_NL + lane - lo;
                        }
                        if (off && BMB_TID == 0) J[0] = 0;
                        BMB_SYNC();
                        int rounds = 1;
                        while ((1 << rounds) < H) ++rounds;
                        for (int r = 0; r <= rounds; ++r) {   // pointer jumping: first iterate >= H (in place: any value
                            int ch = 0;                       // read is an iterate of its cell); chains are short in
                            for (int q = BMB_TID; q < H; q += BMB_NT) {   // practice, so stop when nothing moved
                                const int t = J[q];
                                if (t < H) {
                                    const int t2 = J[t];
                                    if (t2 != t) { J[q] = t2; ch = 1; }   // t2 == t: cell t is a column at the minimum in place
                                }
                            }
                            if (!BMB_SYNC_OR(ch)) break;
                        }
                        int val[JV_OWN], dst[JV_OWN];
#pragma unroll
                        for (int q = 0; q < JV_OWN; ++q) {
                            const int P = lo + BMB_TID + q * BMB_NT;
                            dst[q] = -1;
#if !BMB_DEVICE
                            if (P >= n) break;
#endif
                            if (P < n) {
                                val[q] = cols[P];
                                if (P == lo) {
                                    if (off) dst[q] = lo; else if (H > 0) dst[q] = lo + J[0];
                                } else {
                                    const int cc = (P - base) / BMB_NL, b = (P - base) % BMB_NL;
                                    const unsigned em = emask[cc];
                                    if ((em >> b) & 1u) dst[q] = lo + off + erank[cc] + BMB_POPC(em & ((1u << b) - 1u));
                                    else if (P - lo < H) dst[q] = lo + J[P - lo];
                                }
                            }
                        }
                        BMB_SYNC();
#pragma unroll
                        for (int q = 0; q < JV_OWN; ++q) {
#if !BMB_DEVICE
                            if (lo + BMB_TID + q * BMB_NT >= n) break;
#endif
                            if (dst[q] >= 0) cols[dst[q]] = val[q];
                        }
                    }
                    if (BMB_TID == 0) { mbx[0] = lo + H; mbx[1] = -1; }
                } else
                // (4) the swaps are sequential by nature: one thread replays the hits in position order
                if (BMB_TID == 0) {
                    int h2 = lo + 1;
                    double mind = d[cols[lo]];
                    for (int cc = 0; cc < C; ++cc) {
                        unsigned m = hmask[cc];
                        if (!m) continue;
                        const int kb = base + cc * BMB_NL;
                        if (smask[cc] == 0u && kb == h2 && (m & (m + 1u)) == 0u) {   // ties at h2, h2+1, ...: self-swaps
                            h2 += BMB_POPC(m);
                            continue;
                        }
                        while (m) {
                            const int k = kb + BMB_FFS(m);
                            m &= m - 1;
                            const int j = cols[k];
                            const double dj = d[j];
                            if (dj < mind) { h2 = lo; mind = dj; }
                            cols[k] = cols[h2];
                            cols[h2] = j;
                            ++h2;
                        }
                    }
                    mbx[0] = h2;
                    mbx[1] = -1;
                }
                BMB_SYNC();
                hi = mbx[0];
                // (5) inverse permutation, and lapjv's choice among free columns of the band: the LAST one
                {
                    int last = -1;
                    for (int k = BMB_TID; k < n; k += BMB_NT) {
                        const int j = cols[k];
                        pos[j] = k;
                        if (k >= lo && k < hi && y[j] < 0) last = k;
                    }
                    if (last >= 0) BMB_ATOMIC_MAX(&mbx[1], last);
                }
                BMB_SYNC();
                n_ready = lo;
                band = lo;
                final_j = mbx[1] >= 0 ? cols[mbx[1]] : -1;
#pragma unroll
                for (int q = 0; q < JV_OWN; ++q) {
                    const int jj = BMB_TID + q * BMB_NT;
#if BMB_DEVICE
                    if (jj < n && pos[jj] < hi) { open &= ~(1u << q); dq[q] = -BIG; }
#else
                    if (jj >= n) break;
                    if (pos[jj] < hi) open_h[q] = 0;
#endif
                }
                BMB_SYNC();   // mbx is rewritten by the next replay / find only after everyone has read it
                c_find += BMB_CLOCK() - c0;
            }
            // ---- _scan_dense over the ready band: register arithmetic and one barrier per band column ----
            // no-op band columns: zero-padding owner whose distance never improved (h == 0.0 exactly).  Every warp walks
            // on its own over 32 positions per ballot; nothing is written, and later steps only write open columns.
            auto walk = [&](int from, int to) {
                while (from != to) {
                    const int k = from + lane;
                    bool stop = false;
                    if (k < to) {
                        const int jb = cols[k];
                        stop = !(y[jb] >= zrow && ((0.0 - v[jb]) - d[jb]) == 0.0);
                    }
                    const unsigned m = BMB_BALLOT(stop);
                    if (m) { from += BMB_FFS(m); break; }
                    from += to - from < BMB_NL ? to - from : BMB_NL;
                }
                return from;
            };
            const bool walking = skip_noop && start_zr;
            bool known = false;   // cols[lo] was already found to need a relaxation by the previous step's look-ahead
            while (lo != hi && final_j == -1) {
                if (walking && !known) {
                    const int nl = walk(lo, hi);
                    n_skip += nl - lo;
                    lo = nl;
                    if (lo == hi) break;
                }
                ++n_steps;
                const int j = cols[lo++];
                const int i = y[j];
                const double mind = d[j];
                const bool zr = i >= zrow;
                const double* ci = c + (size_t)i * ld;
                const double h = (zr ? 0.0 : ci[j]) - v[j] - mind;
                // look ahead to the next band column that needs a relaxation: its cost row is prefetched while this one
                // is relaxed (with the no-op columns skipped the next list entry is usually not the next row to load,
                // so without this every relaxed column waits for its row).  [lo, la) stays no-op whatever this step
                // appends to the band: hits only write list positions >= hi.
                const int la = walking ? walk(lo, hi) : lo;
                known = walking && la != hi;
                const double* cn = nullptr;   // row of the next relaxed band column (prefetch target)
                if (la != hi) {
                    const int jn = cols[la];
                    const int in = y[jn];
                    if (in < zrow) { cn = c + (size_t)in * ld; if (BMB_TID == 0) BMB_PREFETCH_L1(cn + jn); }
                }
                if (walking) { n_skip += la - lo; lo = la; }
                int any = 0;
#if BMB_DEVICE
                // straight-line relax: no per-column branch (closed columns hold -BIG), improvements and band-minimum
                // hits are collected as bit masks and written back afterwards (they are rare)
                unsigned imp = 0u, hitq = 0u;
                if (zr) {
#pragma unroll
                    for (int q = 0; q < JV_OWN; ++q) {
                        const double r = nvq[q] - h;
                        const bool better = r < dq[q];
                        dq[q] = better ? r : dq[q];
                        imp |= (better ? 1u : 0u) << q;
                        hitq |= ((better && r == mind) ? 1u : 0u) << q;
                    }
                } else {
                    // the row entries first, all loads in flight together (inside the branchy loop below each load waited
                    // for the previous column), then the
                    // prefetch of the next row, then the arithmetic
                    double cq[JV_OWN];
#pragma unroll
                    for (int q = 0; q < JV_OWN; ++q) cq[q] = ((open >> q) & 1u) ? ci[BMB_TID + q * BMB_NT] : 0.0;
                    if (cn) {
#pragma unroll
                        for (int q = 0; q < JV_OWN; ++q)
                            if ((open >> q) & 1u) BMB_PREFETCH_L1(cn + BMB_TID + q * BMB_NT);
                    }
#pragma unroll
                    for (int q = 0; q < JV_OWN; ++q) {
                        const int jj = BMB_TID + q * BMB_NT;
                        if ((open >> q) & 1u) {
                            const double r = (cq[q] - v[jj]) - h;
                            const bool better = r < dq[q];
                            dq[q] = better ? r : dq[q];
                            imp |= (better ? 1u : 0u) << q;
                            hitq |= ((better && r == mind) ? 1u : 0u) << q;
                        }
                    }
                }
                while (imp) {
                    const int q = __ffs(imp) - 1;
                    imp &= imp - 1u;
                    const int jj = BMB_TID + q * BMB_NT;
                    pred[jj] = i;
                    if ((hitq >> q) & 1u) {
                        d[jj] = mind;
                        any = 1;
                        if (hitlist) { const int sl = atomicAdd(&sh_nhit, 1); if (sl < JV_HITCAP) hitpos[sl] = pos[jj]; }
                    }
                }
#else
                for (int q = 0; q < JV_OWN; ++q) {
                    const int jj = BMB_TID + q * BMB_NT;
                    if (jj >= n) break;
                    if (open_h[q]) {
                        const double r = zr ? nvq[q] - h : (ci[jj] - v[jj]) - h;
                        if (r < dq[q]) {
                            dq[q] = r;
                            pred[jj] = i;
                            if (r == mind) {
                                d[jj] = r;
                                any = 1;
                                if (hitlist) { const int sl = sh_nhit++; if (sl < JV_HITCAP) hitpos[sl] = pos[jj]; }
                            }
                        }
                    }
                }
#endif
                any = BMB_SYNC_OR(any);
                if (any) {
                    c0 = BMB_CLOCK();
                    // the hits, in position order: open positions whose distance now equals the band minimum
                    const int hi0 = hi;
                    const int nh = hitlist ? sh_nhit : JV_HITCAP + 1;   // reset by thread 0 after the next barrier
                    if (nh <= JV_HITCAP) {
                        if (BMB_TID == 0) {
                            for (int a = 1; a < nh; ++a) {   // the list is short: insertion sort by position
                                const int pa = hitpos[a];
                                int b = a - 1;
                                while (b >= 0 && hitpos[b] > pa) { hitpos[b + 1] = hitpos[b]; --b; }
                                hitpos[b + 1] = pa;
                            }
                            int h2 = hi0, fj = -1;
                            for (int a = 0; a < nh; ++a) {
                                const int kq = hitpos[a];
                                const int jq = cols[kq];
                                if (y[jq] < 0) { fj = jq; break; }
                                const int other = cols[h2];
                                cols[kq] = other;
                                pos[other] = kq;
                                cols[h2] = jq;
                                pos[jq] = h2;
                                ++h2;
                            }
                            mbx[0] = h2;
                            mbx[1] = fj;
                        }
                    } else {
                    int slot = BMB_WARP;
                    for (int k0 = hi0; k0 < n; k0 += BMB_NT, slot += BMB_NW) {
                        const int k = k0 + BMB_TID;
                        const unsigned m = BMB_BALLOT(k < n && d[cols[k]] == mind);
                        if (lane == 0) hmask[slot] = m;
                    }
                    BMB_SYNC();
                    if (BMB_TID == 0) {
                        int h2 = hi0, fj = -1;
                        const int n_slots = ((n - hi0 + BMB_NT - 1) / BMB_NT) * BMB_NW;
                        for (int qq = 0; qq < n_slots && fj < 0; ++qq) {
                            unsigned m = hmask[qq];
                            const int kb = hi0 + (qq / BMB_NW) * BMB_NT + (qq % BMB_NW) * BMB_NL;
                            while (m) {
                                const int kq = kb + BMB_FFS(m);
                                m &= m - 1;
                                const int jq = cols[kq];
                                if (y[jq] < 0) { fj = jq; break; }
                                const int other = cols[h2];
                                cols[kq] = other;
                                pos[other] = kq;
                                cols[h2] = jq;
                                pos[jq] = h2;
                                ++h2;
                            }
                        }
                        mbx[0] = h2;
                        mbx[1] = fj;
                    }
                    }
                    BMB_SYNC();
                    hi = mbx[0];
                    final_j = mbx[1];
                    if (hitlist && BMB_TID == 0) sh_nhit = 0;   // everyone has read it; next push is after the barrier below
#pragma unroll
                    for (int q = 0; q < JV_OWN; ++q) {
                        const int jj = BMB_TID + q * BMB_NT;
#if BMB_DEVICE
                        if (((open >> q) & 1u) && pos[jj] < hi) { open &= ~(1u << q); dq[q] = -BIG; }
#else
                        if (jj >= n) break;
                        if (open_h[q] && pos[jj] < hi) open_h[q] = 0;
#endif
                    }
                    BMB_SYNC();
                    c_replay += BMB_CLOCK() - c0;
                }
            }
        }
        c0 = BMB_CLOCK();
        // price update for the columns scanned before the last band, then augment along the path
        {
            const double mind = d[cols[band]];
            for (int k = BMB_TID; k < n_ready; k += BMB_NT) { const int j = cols[k]; v[j] += d[j] - mind; }
        }
        if (BMB_TID == 0) {
            int j = final_j, i = -1;
            while (i != start) {
                i = pred[j];
                y[j] = i;
                const int prev = x[i];
                x[i] = j;
                j = prev;
            }
        }
        BMB_SYNC();
        c_edge += BMB_CLOCK() - c0;
    }
    if (BMB_TID == 0) {
        s.timers[13] += n_steps; s.timers[11] += c_find; s.timers[14] += c_replay; s.timers[15] += c_edge;
        s.timers[7] += n_skip;
    }
}

// CTA-wide augmenting row reduction (feature JV_F_ARRWIDE): the same sequential rounds as the one-warp loop in
// jv_dense_solve, but the lexicographic two-smallest search of a round runs on every thread (the one-warp loop waits for
// one dependent global load per 32 columns), per-warp results are merged
// through shared memory by every thread alike (top-2 under the strict order (value, index) is associative), and thread 0
// applies the round's writes between two barriers.
struct JvTop2 { double a1, a2; int i1, i2; };
BMB_FN bool jv_less(double va, int ia, double vb, int ib) {
    if (ib < 0) return ia >= 0;
    if (ia < 0) return false;
    return va < vb || (va == vb && ia < ib);
}
BMB_FN JvTop2 jv_merge(const JvTop2& p, const JvTop2& q) {   // both sorted pairs; missing entries have index -1
    JvTop2 r;
    if (jv_less(p.a1, p.i1, q.a1, q.i1)) {
        r.a1 = p.a1; r.i1 = p.i1;
        if (jv_less(p.a2, p.i2, q.a1, q.i1)) { r.a2 = p.a2; r.i2 = p.i2; } else { r.a2 = q.a1; r.i2 = q.i1; }
    } else {
        r.a1 = q.a1; r.i1 = q.i1;
        if (jv_less(q.a2, q.i2, p.a1, p.i1)) { r.a2 = q.a2; r.i2 = q.i2; } else { r.a2 = p.a1; r.i2 = p.i1; }
    }
    return r;
}

template <typename S>
BMB_FN int jv_arr_wide(S& s, int n, int ld, int zrow, int n_free) {
    int* x = s.lap_x; int* y = s.lap_y; double* v = s.lap_v; int* free_rows = s.lap_sc;
    const double* c = s.cost;
    const double BIG = 1.7976931348623157e308;
    const int lane = BMB_LANE;
#if BMB_DEVICE
    __shared__ JvTop2 part[32];
#else
    static JvTop2 part[1];
#endif
    for (int pass = 0; pass < 2 && n_free > 0; ++pass) {
        int cur = 0, kept = 0;
        long long rounds = 0;
        while (cur < n_free) {
            ++rounds;
            const int fi = free_rows[cur++];
            const double* ci = c + (size_t)fi * ld;
            const bool zr = fi >= zrow;
            JvTop2 t;
            t.a1 = BIG; t.a2 = BIG; t.i1 = -1; t.i2 = -1;
            for (int j = BMB_TID; j < n; j += BMB_NT) {
                const double r = (zr ? 0.0 : ci[j]) - v[j];
                if (t.i1 < 0 || r < t.a1) { t.a2 = t.a1; t.i2 = t.i1; t.a1 = r; t.i1 = j; }
                else if (t.i2 < 0 || r < t.a2) { t.a2 = r; t.i2 = j; }
            }
#if BMB_DEVICE
            for (int o = 16; o > 0; o >>= 1) {
                JvTop2 u;
                u.a1 = __shfl_xor_sync(0xffffffffu, t.a1, o); u.a2 = __shfl_xor_sync(0xffffffffu, t.a2, o);
                u.i1 = __shfl_xor_sync(0xffffffffu, t.i1, o); u.i2 = __shfl_xor_sync(0xffffffffu, t.i2, o);
                t = jv_merge(t, u);
            }
#endif
            if (lane == 0) part[BMB_WARP] = t;
            BMB_SYNC();   // (1) per-warp results published; the prices read above are final for this round
            t = part[0];
            for (int w = 1; w < BMB_NW; ++w) t = jv_merge(t, part[w]);
            int j1 = t.i1;
            const int j2 = t.i2;
            const double v1 = t.a1, v2 = (j2 >= 0) ? t.a2 : BIG;
            int i0 = y[j1];
            const int y2 = j2 >= 0 ? y[j2] : -1;
            const double vj1 = v[j1];
            const double lowered = vj1 - (v2 - v1);
            const int moves = lowered < vj1;
            BMB_SYNC();   // (2) everyone has read y / v of this round before thread 0 rewrites them
            if (rounds < (long long)cur * n) {
                if (moves) { if (BMB_TID == 0) v[j1] = lowered; }
                else if (i0 >= 0 && j2 >= 0) { j1 = j2; i0 = y2; }
                if (i0 >= 0) {
                    if (moves) { --cur; if (BMB_TID == 0) free_rows[cur] = i0; }
                    else { if (BMB_TID == 0) free_rows[kept] = i0; ++kept; }
                }
            } else {
                if (i0 >= 0) { if (BMB_TID == 0) free_rows[kept] = i0; ++kept; }
            }
            if (BMB_TID == 0) { x[fi] = j1; y[j1] = fi; }
            BMB_SYNC();   // (3) the round's writes are visible to the next round
        }
        n_free = kept;
    }
    return n_free;
}

// S provides: cost (n x n, leading dimension ld), lap_x, lap_y, lap_v, lap_spc (d), lap_path (pred),
// lap_tl (cols), lap_sc (free rows), lap_insc (once flags).  Called by the whole CTA.
//
// zrow: rows >= zrow of the cost matrix are known to be all +0.0 (the extend_cost padding) -- the CTA-wide search
// does not load them.  wide != 0 selects the CTA-wide augmentation (jv_augment_wide) for n >= 64.
template <typename S>
BMB_FN void jv_dense_solve(S& s, int n, int ld, int zrow = 0x7fffffff, int wide = 0) {
    if (n <= 0) return;
    // wide = mode | (feature bits << 2): mode 0 one warp, 1 CTA-wide over list positions, 2 column-owned, 3 column-owned
    // with the shortcuts of `feat` (JV_F_*)
    const int mode = wide & 3;
    const int feat = mode == 3 ? (wide >> 2) : 0;
    const bool wide_eff = mode && n >= 64;
    // column-owned variant: every thread keeps JV_OWN columns in registers, _find_dense holds JV_CHUNKS chunks
    const bool owned_eff = wide_eff && mode >= 2 && n <= JV_OWN * BMB_NT && n <= (JV_CHUNKS - 8) * BMB_NL;
    const bool arr_wide = owned_eff && (feat & JV_F_ARRWIDE) != 0 && BMB_NW <= 32;
#if BMB_DEVICE
    __shared__ int jv_mbx[2];
#else
    int jv_mbx[2];
#endif
    const double BIG = 1.7976931348623157e308;
    int* x = s.lap_x; int* y = s.lap_y; double* v = s.lap_v; double* d = s.lap_spc;
    int* pred = s.lap_path; int* cols = s.lap_tl; int* free_rows = s.lap_sc; int* once = s.lap_insc;
    const double* c = s.cost;
    // ---- column reduction: every column elects its cheapest row (first minimal row) ----
    for (int i = BMB_TID; i < n; i += BMB_NT) { x[i] = -1; once[i] = 1; }
    for (int j = BMB_TID; j < n; j += BMB_NT) {
        double vj = BIG; int yj = 0;
        for (int i = 0; i < n; ++i) {
            const double cij = c[(size_t)i * ld + j];
            if (cij < vj) { vj = cij; yj = i; }
        }
        v[j] = vj; y[j] = yj;
    }
    BMB_SYNC();
    if (BMB_WARP == 0) {
        const int lane = BMB_LANE;
        long long _jt = BMB_CLOCK();   // solver phase clocks (timers 8..11) and work counters (12..13), diagnostics
        auto tick = [&](int slot) {
            if (lane == 0) { const long long now = BMB_CLOCK(); s.timers[slot] += now - _jt; _jt = now; }
        };
        if (lane == 0) {
            for (int j = n - 1; j >= 0; --j) {
                const int i = y[j];
                if (x[i] < 0) x[i] = j;
                else { once[i] = 0; y[j] = -1; }
            }
        }
        BMB_SYNCWARP();
        // reduction transfer (sequential over rows: prices change as we go), free rows collected in order
        int n_free = 0;
        for (int i = 0; i < n; ++i) {
            const int xi = x[i];
            if (xi < 0) { if (lane == 0) free_rows[n_free] = i; ++n_free; continue; }
            if (!once[i]) continue;
            const double* ci = c + (size_t)i * ld;
            const bool zr = i >= zrow;   // zero padding row: nothing to load
            double m = BIG;
            for (int k = lane; k < n; k += BMB_NL)
                if (k != xi) { const double r = (zr ? 0.0 : ci[k]) - v[k]; if (r < m) m = r; }
#if BMB_DEVICE
            for (int o = 16; o > 0; o >>= 1) { const double t = __shfl_xor_sync(0xffffffffu, m, o); if (t < m) m = t; }
#endif
            if (lane == 0) v[xi] -= m;
            BMB_SYNCWARP();
        }
        tick(8);
        // ---- augmenting row reduction, two passes ----
        for (int pass = 0; pass < 2 && n_free > 0 && !arr_wide; ++pass) {
            int cur = 0, kept = 0;
            long long rounds = 0;
            while (cur < n_free) {
                ++rounds;
                const int fi = free_rows[cur++];
                const double* ci = c + (size_t)fi * ld;
                const bool zr = fi >= zrow;
                // lexicographic (value, index) minimum and the minimum over the remaining indices
                double a1 = BIG, a2 = BIG; int i1 = -1, i2 = -1;
                for (int j = lane; j < n; j += BMB_NL) {
                    const double r = (zr ? 0.0 : ci[j]) - v[j];
                    if (i1 < 0 || r < a1) { a2 = a1; i2 = i1; a1 = r; i1 = j; }
                    else if (i2 < 0 || r < a2) { a2 = r; i2 = j; }
                }
#if BMB_DEVICE
                for (int o = 16; o > 0; o >>= 1) {
                    const double b1 = __shfl_xor_sync(0xffffffffu, a1, o), b2 = __shfl_xor_sync(0xffffffffu, a2, o);
                    const int k1 = __shfl_xor_sync(0xffffffffu, i1, o), k2 = __shfl_xor_sync(0xffffffffu, i2, o);
                    // merge two sorted pairs {(a1,i1),(a2,i2)} and {(b1,k1),(b2,k2)}; missing entries have index -1
                    auto less = [](double va, int ia, double vb, int ib) {
                        if (ib < 0) return ia >= 0;
                        if (ia < 0) return false;
                        return va < vb || (va == vb && ia < ib);
                    };
                    double n1, n2; int m1, m2;
                    if (less(a1, i1, b1, k1)) {
                        n1 = a1; m1 = i1;
                        if (less(a2, i2, b1, k1)) { n2 = a2; m2 = i2; } else { n2 = b1; m2 = k1; }
                    } else {
                        n1 = b1; m1 = k1;
                        if (less(b2, k2, a1, i1)) { n2 = b2; m2 = k2; } else { n2 = a1; m2 = i1; }
                    }
                    a1 = n1; i1 = m1; a2 = n2; i2 = m2;
                }
#endif
                int j1 = i1, j2 = i2;
                const double v1 = a1, v2 = (i2 >= 0) ? a2 : BIG;
                int i0 = y[j1];
                const double lowered = v[j1] - (v2 - v1);
                const int moves = lowered < v[j1];
                BMB_SYNCWARP();
                if (rounds < (long long)cur * n) {
                    if (moves) { if (lane == 0) v[j1] = lowered; }
                    else if (i0 >= 0 && j2 >= 0) { j1 = j2; i0 = y[j2]; }
                    if (i0 >= 0) {
                        if (moves) { --cur; if (lane == 0) free_rows[cur] = i0; }
                        else { if (lane == 0) free_rows[kept] = i0; ++kept; }
                    }
                } else {
                    if (i0 >= 0) { if (lane == 0) free_rows[kept] = i0; ++kept; }
                }
                if (lane == 0) { x[fi] = j1; y[j1] = fi; }
                BMB_SYNCWARP();
            }
            n_free = kept;
        }
        if (!arr_wide) tick(9);
        if (lane == 0) { if (!arr_wide) s.timers[12] += n_free; jv_mbx[0] = n_free; }
        // ---- augmentation (one warp; the CTA-wide variant follows the barrier below) ----
        for (int f = 0; f < (wide_eff ? 0 : n_free); ++f) {
            const int start = free_rows[f];
            int lo = 0, hi = 0, n_ready = 0, band = 0, final_j = -1;
            {
                const double* cs = c + (size_t)start * ld;
                for (int j = lane; j < n; j += BMB_NL) { cols[j] = j; pred[j] = start; d[j] = cs[j] - v[j]; }
            }
            BMB_SYNCWARP();
            while (final_j == -1) {
                if (lo == hi) {
                    // _find_dense.  lapjv scans cols[lo+1..n) once, keeping the running minimum: a column at or below
                    // it is a "hit" (strictly below: the tie list restarts at lo) and is swapped to the front; the
                    // swaps define the scan order of later ties, so they are replayed exactly -- but only the hits are
                    // sequential.  The lanes find them with a warp prefix-minimum per 32 columns (a hit at position k
                    // only rewrites positions <= k, so the columns of a chunk can be read before its hits are applied).
                    {
                        int h2 = lo + 1;
                        double mind = d[cols[lo]];
                        for (int k0 = lo + 1; k0 < n; k0 += BMB_NL) {
                            const int k = k0 + lane;
                            const int j = k < n ? cols[k] : -1;
                            const double dj = k < n ? d[j] : BIG;
#if BMB_DEVICE
                            double pm = dj;   // inclusive prefix minimum over the lanes of this chunk
                            for (int o = 1; o < 32; o <<= 1) {
                                const double t = __shfl_up_sync(0xffffffffu, pm, o);
                                if (lane >= o && t < pm) pm = t;
                            }
                            const double excl = __shfl_up_sync(0xffffffffu, pm, 1);
                            const double before = lane == 0 ? mind : (excl < mind ? excl : mind);   // running minimum
                            unsigned hits = __ballot_sync(0xffffffffu, k < n && dj <= before);
                            while (hits) {
                                const int src = __ffs(hits) - 1;
                                hits &= hits - 1;
                                const double dh = __shfl_sync(0xffffffffu, dj, src);
                                const int jh = __shfl_sync(0xffffffffu, j, src);
                                if (dh < mind) { h2 = lo; mind = dh; }
                                if (lane == 0) { cols[k0 + src] = cols[h2]; cols[h2] = jh; }
                                ++h2;
                                __syncwarp();
                            }
#else
                            if (dj <= mind) {
                                if (dj < mind) { h2 = lo; mind = dj; }
                                cols[k] = cols[h2];
                                cols[h2++] = j;
                            }
#endif
                        }
                        BMB_SYNCWARP();
                        if (lane == 0) {
                            int fj = -1;
                            for (int k = lo; k < h2; ++k)
                                if (y[cols[k]] < 0) fj = cols[k];
                            s.free_l[MB_COUNT - 1] = h2;
                            s.free_l[MB_COUNT - 2] = fj;
                        }
                    }
                    BMB_SYNCWARP();
                    n_ready = lo;
                    band = lo;
                    hi = s.free_l[MB_COUNT - 1];
                    final_j = s.free_l[MB_COUNT - 2];
                    BMB_SYNCWARP();
                }
                if (final_j == -1) {
                    // _scan_dense over the ready band
                    while (lo != hi && final_j == -1) {
                        if (lane == 0) s.timers[13] += 1;
                        const int j = cols[lo++];
                        const int i = y[j];
                        const double mind = d[j];
                        const double* ci = c + (size_t)i * ld;
                        const double h = ci[j] - v[j] - mind;
                        const int hi0 = hi;
                        for (int k0 = hi0; k0 < n && final_j == -1; k0 += BMB_NL) {
                            const int k = k0 + lane;
                            int jj = -1;
                            bool hit = false;
                            if (k < n) {
                                jj = cols[k];
                                const double r = ci[jj] - v[jj] - h;
                                if (r < d[jj]) {
                                    d[jj] = r;
                                    pred[jj] = i;
                                    hit = (r == mind);
                                }
                            }
                            unsigned m = BMB_BALLOT(hit);
                            // replay the "equals the band minimum" events in ascending position order
                            while (m) {
#if BMB_DEVICE
                                const int src = __ffs(m) - 1;
                                const int kq = k0 + src;
                                const int jq = __shfl_sync(0xffffffffu, jj, src);
#else
                                const int src = 0;
                                const int kq = k0;
                                const int jq = jj;
#endif
                                m &= m - 1;
                                if (y[jq] < 0) { final_j = jq; break; }
                                if (lane == 0) { cols[kq] = cols[hi]; cols[hi] = jq; }
                                ++hi;
                                BMB_SYNCWARP();
                                (void)src;
                            }
                            BMB_SYNCWARP();
                        }
                    }
                }
            }
            // price update for the columns scanned before the last band, then augment along the path
            {
                const double mind = d[cols[band]];
                BMB_SYNCWARP();
                for (int k = lane; k < n_ready; k += BMB_NL) { const int j = cols[k]; v[j] += d[j] - mind; }
            }
            BMB_SYNCWARP();
            if (lane == 0) {
                int j = final_j, i = -1;
                while (i != start) {
                    i = pred[j];
                    y[j] = i;
                    const int prev = x[i];
                    x[i] = j;
                    j = prev;
                }
            }
            BMB_SYNCWARP();
        }
        if (!wide_eff) tick(10);
    }
    BMB_SYNC();
    if (arr_wide) {
        const long long t0 = BMB_CLOCK();
        const int nf0 = jv_mbx[0];
        BMB_SYNC();
        const int nf = jv_arr_wide(s, n, ld, zrow, nf0);
        if (BMB_TID == 0) { jv_mbx[0] = nf; s.timers[12] += nf; s.timers[9] += BMB_CLOCK() - t0; }
        BMB_SYNC();
    }
    if (wide_eff) {
        const long long t0 = BMB_CLOCK();
        if (owned_eff) jv_augment_owned(s, n, ld, zrow, jv_mbx[0], jv_mbx, feat);
        else jv_augment_wide(s, n, ld, zrow, jv_mbx[0], jv_mbx);
        if (BMB_TID == 0) s.timers[10] += BMB_CLOCK() - t0;
    }
}

}  // namespace bmb
