// lsa_sap.cuh -- rectangular linear sum assignment with the SAME tie-breaking as scipy.optimize.linear_sum_assignment
// (scipy 1.18: the modified Jonker-Volgenant shortest-augmenting-path solver of Crouse, "On implementing 2D
// rectangular assignment algorithms", IEEE TAES 2016).  StrongSORT's min_cost_matching
// (trackers/bbox/strongsort/sort/linear_assignment.py:59-70) clips every cost above the gate to
// `max_distance + 1e-5`, so its matrices tie by construction, and the solution scipy picks among the optima decides
// the order of the unmatched detections -- i.e. the ids of the tracks born this frame.  A different exact solver
// is not enough; this one reproduces scipy's choices:
//   * rows are augmented in order 0..nr-1 (the caller passes the matrix with nr <= nc, transposing like scipy);
//   * the column scan runs over scipy's `remaining` list (initialised in reverse, swap-with-last removal);
//   * the next column is the lowest shortest-path cost, ties going to the LAST unassigned column scanned, or to the
//     FIRST column scanned when no tied column is unassigned;
//   * dual updates and the path flip are scipy's.
// The whole CTA runs the solver: the O(nc) scans are thread-strided, combined per warp with shuffles and across warps
// through shared memory with exactly that rule (two barriers per augmentation step).
#pragma once
#include "tracker_core.cuh"

namespace bmb {

template <typename S>
BMB_FN void lsa_solve(S& s, const double* cost, int nr, int nc, int ld);

// scipy.optimize.linear_sum_assignment(cost) of an R x C matrix given by cost_at(r, c): scipy solves the transpose when
// C < R.  buf receives the laid-out problem (min(R, C) x max(R, C), leading dimension max(R, C)); rowcol[r] is the
// column assigned to row r, or -1.  Called by the whole CTA.
template <typename S, typename CostAt>
BMB_FN void lsa_rect(S& s, double* buf, int R, int C, CostAt cost_at, int* rowcol) {
    const bool transposed = C < R;
    const int nr = transposed ? C : R, nc = transposed ? R : C;
    for (int e = BMB_TID; e < R * C; e += BMB_NT) {
        const int r = e / C, cc = e - r * C;
        buf[transposed ? (size_t)cc * nc + r : (size_t)r * nc + cc] = cost_at(r, cc);
    }
    BMB_SYNC();
    lsa_solve(s, buf, nr, nc, nc);
    for (int r = BMB_TID; r < R; r += BMB_NT) rowcol[r] = -1;
    BMB_SYNC();
    for (int i = BMB_TID; i < nr; i += BMB_NT) {
        const int j = s.lsa_col4row[i];
        if (j < 0) continue;
        if (transposed) rowcol[j] = i;
        else rowcol[i] = j;
    }
    BMB_SYNC();
}

// S provides lsa_u [>=nr], lsa_v, lsa_spc [>=nc] (double) and lsa_path, lsa_row4col, lsa_rem, lsa_sc [>=nc],
// lsa_col4row, lsa_sr [>=nr] (int).  cost is row-major (nr x nc, leading dimension ld), nr <= nc, finite.
// Result: lsa_col4row[i] for every row.  Called by the whole CTA.
template <typename S>
BMB_FN void lsa_solve(S& s, const double* cost, int nr, int nc, int ld) {
    double* u = s.lsa_u; double* v = s.lsa_v; double* spc = s.lsa_spc;
    int* path = s.lsa_path; int* row4col = s.lsa_row4col; int* col4row = s.lsa_col4row;
    int* rem = s.lsa_rem; int* SR = s.lsa_sr; int* SC = s.lsa_sc;
#if BMB_DEVICE
    __shared__ double red_m[32];
    __shared__ int red_f[32], red_l[32];
#endif
    for (int i = BMB_TID; i < nr; i += BMB_NT) { u[i] = 0.0; col4row[i] = -1; }
    for (int j = BMB_TID; j < nc; j += BMB_NT) { v[j] = 0.0; row4col[j] = -1; }
    BMB_SYNC();
    bool failed = false;
    for (int cur = 0; cur < nr && !failed; ++cur) {
        for (int j = BMB_TID; j < nc; j += BMB_NT) { spc[j] = INFINITY; rem[j] = nc - 1 - j; SC[j] = 0; }
        for (int i = BMB_TID; i < nr; i += BMB_NT) SR[i] = 0;
        BMB_SYNC();
        int num_rem = nc, i = cur, sink = -1;
        double min_val = 0.0;
        while (sink == -1) {
            if (BMB_TID == 0) SR[i] = 1;
            const double* ci = cost + (size_t)i * ld;
            const double ui = u[i];
            double lm = INFINITY;
            int lfirst = 0x7fffffff, llast = -1;
            // the whole CTA scans scipy's `remaining` list; position order is kept by reducing (value, positions)
            for (int it = BMB_TID; it < num_rem; it += BMB_NT) {
                const int j = rem[it];
                const double r = ((min_val + ci[j]) - ui) - v[j];
                double sj = spc[j];
                if (r < sj) { path[j] = i; spc[j] = r; sj = r; }
                const bool un = row4col[j] == -1;
                if (sj < lm) { lm = sj; lfirst = it; llast = un ? it : -1; }
                else if (sj == lm && un) llast = it;
            }
#if BMB_DEVICE
            double m = lm;
            for (int o = 16; o > 0; o >>= 1) { const double t = __shfl_xor_sync(0xffffffffu, m, o); if (t < m) m = t; }
            int f = (lm == m) ? lfirst : 0x7fffffff, l = (lm == m) ? llast : -1;
            for (int o = 16; o > 0; o >>= 1) {
                const int tf = __shfl_xor_sync(0xffffffffu, f, o), tl = __shfl_xor_sync(0xffffffffu, l, o);
                f = tf < f ? tf : f;
                l = tl > l ? tl : l;
            }
            if (BMB_LANE == 0) { red_m[BMB_WARP] = m; red_f[BMB_WARP] = f; red_l[BMB_WARP] = l; }
            __syncthreads();
            m = red_m[0];
            for (int w = 1; w < BMB_NW; ++w) m = red_m[w] < m ? red_m[w] : m;
            f = 0x7fffffff; l = -1;
            for (int w = 0; w < BMB_NW; ++w)
                if (red_m[w] == m) { f = red_f[w] < f ? red_f[w] : f; l = red_l[w] > l ? red_l[w] : l; }
#else
            const double m = lm;
            const int f = lfirst, l = llast;
#endif
            if (!(m < INFINITY)) {  // infeasible / NaN costs: scipy raises; report through the error scalar
                if (BMB_TID == 0) s.scalars[SC_ERROR] = ERR_LSA_INFEASIBLE;
                failed = true;
                break;
            }
            const int index = l >= 0 ? l : f;
            min_val = m;
            const int j = rem[index];
            const int r4 = row4col[j];
            const int last = rem[num_rem - 1];
            BMB_SYNC();   // every thread has read rem[] / the partials before they change
            if (BMB_TID == 0) { SC[j] = 1; rem[index] = last; }
            --num_rem;
            if (r4 == -1) sink = j; else i = r4;
            BMB_SYNC();
        }
        if (failed) break;
        // dual updates (scipy: u[cur] += minVal; visited rows / columns shifted by their slack)
        for (int r = BMB_TID; r < nr; r += BMB_NT) {
            if (r == cur) u[r] = u[r] + min_val;
            else if (SR[r]) u[r] = u[r] + (min_val - spc[col4row[r]]);
        }
        for (int j = BMB_TID; j < nc; j += BMB_NT)
            if (SC[j]) v[j] = v[j] - (min_val - spc[j]);
        BMB_SYNC();
        if (BMB_TID == 0) {
            int j = sink;
            while (true) {
                const int r = path[j];
                row4col[j] = r;
                const int t = col4row[r];
                col4row[r] = j;
                j = t;
                if (r == cur) break;
            }
        }
        BMB_SYNC();
    }
    BMB_SYNC();
}

}  // namespace bmb
