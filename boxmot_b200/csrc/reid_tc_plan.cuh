// reid_tc_plan.cuh -- builds and replays the launch plan of the tensor-core OSNet path (included at the end of
// reid_model.cu; needs ReidModel / BlockW).  Network graph: reid/backbones/osnet.py:380-405, blocks :212-260.
#pragma once

namespace bmb {
namespace tcx {

// stage geometry of the chain kernel instances (osnet_x0_25: mid 16 / 24 / 32 at 64x32 / 32x16 / 16x8)
struct ChainShape { int CP, CR, W, H, R, kind; };
static const ChainShape kChainShapes[3] = {{16, 16, 32, 64, chain_rows<BMB_CHAIN_S2>(), LK_CHAIN_S2}, {32, 24, 16, 32, chain_rows<BMB_CHAIN_S3>(), LK_CHAIN_S3},
                                           {32, 32, 8, 16, chain_rows<BMB_CHAIN_S4>(), LK_CHAIN_S4}};

inline bool plan_supported(const ReidModel* m) {
    return m->arch == ARCH_OSNET && m->c[0] == 16 && m->c[1] == 64 && m->c[2] == 96 && m->c[3] == 128;
}

Plan* plan_build(ReidModel* m, const float* hw) {
    Plan* P = new Plan();
    try {
        P->chunk = m->chunk;
        const size_t CH = (size_t)m->chunk;
        int dev = 0;
        RCUDA_OK(cudaGetDevice(&dev));
        RCUDA_OK(cudaDeviceGetAttribute(&P->smem_limit, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
        P->smem_limit -= 1024;   // static shared memory (barriers) comes out of the same budget
        // ---- workspace: split planes (hi, lo), sized for the widest use of each buffer ----
        alloc_planes(P->P, CH * 2048 * 16);
        alloc_planes(P->X1, CH * 2048 * 16);
        alloc_planes(P->Y, CH * 2048 * 64);
        alloc_planes(P->XA, CH * 2048 * 64);
        alloc_planes(P->XB, CH * 2048 * 64);
        RCUDA_OK(cudaMalloc(&P->c5, sizeof(float) * CH * 128 * m->c[3]));
        for (int b = 0; b < 4; ++b) RCUDA_OK(cudaMalloc(&P->sums[b], sizeof(float) * CH * 8 * 32));
        RCUDA_OK(cudaMalloc(&P->gates, sizeof(float) * CH * 4 * 32));
        RCUDA_OK(cudaMalloc(&P->arrivals, sizeof(int) * CH));
        RCUDA_OK(cudaMemset(P->arrivals, 0, sizeof(int) * CH));
        RCUDA_OK(cudaMalloc(&P->bfold, (size_t)CH * 16 * 2 * 128 * 16));   // [crops][<= 16 planes][2 * NP <= 256][8] BF16
        RCUDA_OK(cudaMalloc(&P->dbg, sizeof(float) * CH * 2048 * 64));

        // ---- weights ----
        std::vector<uint16_t> wb;
        std::vector<float> wf;
        struct BlkOff { size_t pw[10], dw[10], lb[10], c1, c1b, cx, cxb; } bo[6];
        for (int bi = 0; bi < 6; ++bi) {
            const BlockW& b = m->blocks[bi];
            const int midp = pad16(b.mid);
            for (int l = 0; l < 10; ++l) {
                bo[bi].pw[l] = pack_b(wb, hw + b.light[l].pw, b.mid, b.mid, b.mid, midp / 8, midp);
                // depthwise taps [9][mid] -> [9][midp]
                size_t at = (wf.size() + 3) / 4 * 4;
                wf.resize(at + 9 * midp, 0.f);
                for (int t = 0; t < 9; ++t)
                    for (int c = 0; c < b.mid; ++c) wf[at + t * midp + c] = hw[b.light[l].dw + (size_t)t * b.mid + c];
                bo[bi].dw[l] = at;
                bo[bi].lb[l] = pack_f(wf, hw + b.light[l].b, b.mid, midp);
                // k_chain_tc fetches taps + bias with one bulk copy
                if (bo[bi].lb[l] != at + (size_t)9 * midp) throw std::runtime_error("chain weights: taps and bias are not contiguous");
            }
            bo[bi].c1 = pack_b(wb, hw + b.c1w, b.cin, b.mid, b.mid, b.cin / 8, midp);
            bo[bi].c1b = pack_f(wf, hw + b.c1b, b.mid, midp);
            // combine: K rows = [4 * midp gate-folded conv3 rows (built in the kernel)] ++ [cin rows: downsample or identity]
            const int K8 = 4 * midp / 8 + b.cin / 8;
            if (b.has_ds)
                bo[bi].cx = pack_b(wb, hw + b.cw + (size_t)b.mid * b.cout, b.cin, b.cout, b.cout, K8, b.cout, 4 * midp);
            else
                bo[bi].cx = pack_b(wb, nullptr, b.cin, b.cout, b.cout, K8, b.cout, 4 * midp, true);
            bo[bi].cxb = pack_f(wf, hw + b.cb, b.cout, b.cout);
        }
        size_t tr[2], trb[2];
        for (int s = 0; s < 2; ++s) {
            const int C = m->c[s + 1];
            tr[s] = pack_b(wb, hw + m->trans_w[s], C, C, C, C / 8, C);
            trb[s] = pack_f(wf, hw + m->trans_b[s], C, C);
        }
        const size_t c5 = pack_b(wb, hw + m->c5w, m->c[3], m->c[3], m->c[3], m->c[3] / 8, m->c[3]);
        const size_t c5b = pack_f(wf, hw + m->c5b, m->c[3], m->c[3]);
        // fused front kernel: stem weights with the input normalisation folded in, W' = w / (255 std), as
        // [7 kx][4 k8][32 n' = hi | lo][8 k] with k = ky * 4 + ci (tap 7 and channel 3 are zero), and the bias table
        // b - sum over the taps inside the image of w mean / std per (row class, column class)
        size_t fw, fb;
        {
            const double mean[3] = {0.485, 0.456, 0.406}, stdv[3] = {0.229, 0.224, 0.225};
            const int C0 = m->c[0];
            fw = (wb.size() + 63) / 64 * 64;
            wb.resize(fw + 7 * 4 * 32 * 8, 0);
            for (int kx = 0; kx < 7; ++kx)
                for (int ky = 0; ky < 7; ++ky)
                    for (int ci = 0; ci < 3; ++ci)
                        for (int co = 0; co < C0; ++co) {
                            const float v = (float)((double)hw[m->stem_w + (size_t)((ky * 7 + kx) * 3 + ci) * C0 + co] / (255.0 * stdv[ci]));
                            const int k = ky * 4 + ci;
                            uint16_t* plane = wb.data() + fw + ((size_t)(kx * 4 + k / 8) * 32) * 8;
                            const uint16_t h = f2bf(v);
                            plane[(size_t)co * 8 + k % 8] = h;
                            plane[(size_t)(16 + co) * 8 + k % 8] = f2bf(v - bf2f(h));
                        }
            fb = (wf.size() + 3) / 4 * 4;
            wf.resize(fb + 4 * 4 * 16, 0.f);
            const int lo_[4] = {3, 1, 0, 0}, hi_[4] = {6, 6, 6, 4};       // valid taps per class: first/second/interior/last
            for (int rc = 0; rc < 4; ++rc)
                for (int cc = 0; cc < 4; ++cc)
                    for (int co = 0; co < C0; ++co) {
                        double acc = hw[m->stem_b + co];
                        for (int ky = lo_[rc]; ky <= hi_[rc]; ++ky)
                            for (int kx = lo_[cc]; kx <= hi_[cc]; ++kx)
                                for (int ci = 0; ci < 3; ++ci)
                                    acc -= (double)hw[m->stem_w + (size_t)((ky * 7 + kx) * 3 + ci) * C0 + co] * mean[ci] / stdv[ci];
                        wf[fb + (rc * 4 + cc) * 16 + co] = (float)acc;
                    }
        }
        RCUDA_OK(cudaMalloc(&P->d_wb, wb.size() * 2 + 256));
        RCUDA_OK(cudaMemcpy(P->d_wb, wb.data(), wb.size() * 2, cudaMemcpyHostToDevice));
        RCUDA_OK(cudaMalloc(&P->d_wf, wf.size() * 4 + 256));
        RCUDA_OK(cudaMemcpy(P->d_wf, wf.data(), wf.size() * 4, cudaMemcpyHostToDevice));
        const bf16* WB = P->d_wb;
        const float* WF = P->d_wf;
        const float* W32 = m->d_w;

        // ---- kernel attributes ----
        RCUDA_OK(chain_prepare<BMB_CHAIN_S2>());
        RCUDA_OK(chain_prepare<BMB_CHAIN_S3>());
        RCUDA_OK(chain_prepare<BMB_CHAIN_S4>());
        for (const GemmInstance& gi : kGemmInstances)
            RCUDA_OK(cudaFuncSetAttribute(gi.fn, cudaFuncAttributeMaxDynamicSharedMemorySize, P->smem_limit));
        RCUDA_OK(cudaFuncSetAttribute(k_front_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FR_SMEM));

        // ---- launches ----
        struct Src { Planes* buf; int C8; };
        auto gemm = [&](int H, int Wd, std::vector<Src> srcs, size_t b_off, int N, size_t bias_off, bool relu) -> Launch {
            Launch L{};
            L.kind = LK_GEMM;
            L.cls = CLS_POINTWISE;
            GemmTcArgs& g = L.gemm;
            g.n_src = (int)srcs.size();
            g.rows_per_tile = 128 / Wd;
            g.tiles_per_crop = H * Wd / 128;
            g.tiles_per_cta = g.tiles_per_crop >= 16 ? 4 : (g.tiles_per_crop >= 4 ? 2 : 1);
            g.K8 = 0;
            for (int s = 0; s < g.n_src; ++s) {
                const int C8 = srcs[s].C8;
                const int kc = C8 % 4 == 0 ? 4 : 2;
                g.src_planes[s] = C8;
                g.src_kc[s] = kc;
                g.K8 += C8;
                L.src_hi[s] = srcs[s].buf->hi;
                L.src_lo[s] = srcs[s].buf->lo;
            }
            g.b_packed = WB + b_off;
            g.N = N;
            g.NP = pad16(N);
            g.bias = WF + bias_off;
            g.relu = relu ? 1 : 0;
            g.HW = H * Wd;
            g.W = Wd;
            return L;
        };
        auto finish_into = [&](Launch& L, std::vector<Launch>* out) {
            GemmTcArgs& g = L.gemm;
            const bool tail = g.b2_packed != nullptr;
            if (g.NP > 128 || (tail && g.NP2 > 128)) throw std::runtime_error("tensor-core GEMM: more than 128 output channels");
            const int mode = g.head_w ? GM_HEAD : g.pool ? GM_POOL : !tail ? GM_PLAIN : g.pool2 ? GM_TAIL_POOL2 : GM_TAIL;
            L.gemm_fn = gemm_instance(g.NP, tail ? g.NP2 : 0, mode);
            if (!L.gemm_fn)
                throw std::runtime_error("tensor-core GEMM: no kernel instance for NP = " + std::to_string(g.NP) + ", NP2 = " +
                                         std::to_string(tail ? g.NP2 : 0) + ", epilogue mode " + std::to_string(mode));
            auto layout = [&](int ns) { return gemm_smem_layout(g.K8, g.NP, g.NP2, ns, tail, g.pool != 0, g.slot_bytes, g.pool2 != 0); };
            auto ctas = [&](int ns) {     // CTAs per SM of the instance at this layout (registers, shared memory, threads)
                const size_t bytes = layout(ns).total;
                int c = 0;
                if ((int)bytes <= P->smem_limit)
                    RCUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&c, L.gemm_fn, GEMM_THREADS, bytes));
                return c;
            };
            // two CTAs per SM (they overlap each other's MMA / epilogue / load latencies) when the occupancy calculator
            // places two with a >= 2-deep ring -- with smaller ring chunks (2 planes) if that is what it takes; otherwise
            // one CTA with the deepest ring that fits
            int ns = 0;
            for (int pass = 0; pass < 2 && !ns; ++pass) {
                int kc_max = 2;
                for (int s = 0; s < g.n_src; ++s) {
                    if (pass == 1) g.src_kc[s] = 2;
                    kc_max = std::max(kc_max, g.src_kc[s]);
                }
                g.slot_bytes = kc_max * 128 * 16 * 2;
                for (int cand = 4; cand >= 2 && !ns; --cand)
                    if (ctas(cand) >= 2) ns = cand;
            }
            if (!ns) {
                int kc_max = 2;
                for (int s = 0; s < g.n_src; ++s) {
                    g.src_kc[s] = g.src_planes[s] % 4 == 0 ? 4 : 2;
                    kc_max = std::max(kc_max, g.src_kc[s]);
                }
                g.slot_bytes = kc_max * 128 * 16 * 2;
                for (int cand = 4; cand >= 2 && !ns; --cand)
                    if (ctas(cand) >= 1) ns = cand;
            }
            if (!ns) throw std::runtime_error("tensor-core GEMM does not fit shared memory");
            L.gemm_ctas = ctas(ns);
            for (int s = 0; s < g.n_src; ++s) {   // the boxes follow the chunk size
                make_tile_map(&g.map_hi[s], L.src_hi[s], P->chunk, g.src_planes[s], g.HW, g.src_kc[s]);
                make_tile_map(&g.map_lo[s], L.src_lo[s], P->chunk, g.src_planes[s], g.HW, g.src_kc[s]);
            }
            L.gl = layout(ns);
            g.n_stage = ns;
            L.gemm_groups = (g.tiles_per_crop + g.tiles_per_cta - 1) / g.tiles_per_cta;
            out->push_back(L);
        };
        auto dbg = [&](Launch& L, int stage, const Planes& buf, int C8, int HW, int C) {
            L.stage_after = stage;
            L.dbg_hi = buf.hi; L.dbg_lo = buf.lo; L.dbg_C8 = C8; L.dbg_HW = HW; L.dbg_C = C;
        };

        auto build_launches = [&](bool fuse_trans, std::vector<Launch>* out) {
            auto finish = [&](Launch& L) { finish_into(L, out); };
        {   // crop + resize + stem + max pool -> planes P (one fused tensor-core kernel); launches[1] is the float32-stem
            // fallback entry used when a diagnostic stop asks for the blob / stem tensors of the round-1 kernels
            Launch L{};
            L.kind = LK_FRONT;
            L.cls = CLS_STEM;
            L.front.w = WB + fw;
            L.front.bias_tab = WF + fb;
            L.front.p_hi = P->P.hi; L.front.p_lo = P->P.lo;
            dbg(L, 2, P->P, 2, 2048, 16);
            out->push_back(L);
        }
        Planes* X = &P->P;          // block input
        Planes* Xo = &P->XA;
        Planes* Xspare = &P->XB;
        int xC8 = 2;
        int H = 64, Wd = 32;
        int stage = 3;
        {   // conv1 of the first block
            const BlockW& b = m->blocks[0];
            Launch L = gemm(H, Wd, {{X, xC8}}, bo[0].c1, b.mid, bo[0].c1b, true);
            L.gemm.out_hi = P->X1.hi; L.gemm.out_lo = P->X1.lo;
            dbg(L, 100, P->X1, pad16(b.mid) / 8, H * Wd, pad16(b.mid));
            finish(L);
        }
        for (int s = 0; s < 3; ++s) {
            const ChainShape& cs = kChainShapes[s];
            bool trans_done = false;
            for (int j = 0; j < 2; ++j) {
                const int bi = s * 2 + j;
                const BlockW& b = m->blocks[bi];
                const int midp = pad16(b.mid);
                {   // the four LightConv branches
                    Launch L{};
                    L.kind = cs.kind;
                    L.cls = CLS_LIGHTCONV;
                    ChainTcArgs& c = L.chain;
                    make_rows_map(&c.map_hi, P->X1.hi, P->chunk, midp / 8, H, Wd, cs.R + 8);
                    make_rows_map(&c.map_lo, P->X1.lo, P->chunk, midp / 8, H, Wd, cs.R + 8);
                    for (int l = 0; l < 10; ++l) {
                        c.wpw[l] = WB + bo[bi].pw[l];
                        c.wdw[l] = WF + bo[bi].dw[l];
                        c.bias[l] = WF + bo[bi].lb[l];
                    }
                    c.y_hi = P->Y.hi; c.y_lo = P->Y.lo;
                    for (int br = 0; br < 4; ++br) c.sums[br] = P->sums[br];
                    c.H = H;
                    GatesTcArgs& ga = c.gate;     // ChannelGate + conv3 fold: the last CTA of each crop does it
                    for (int br = 0; br < 4; ++br) ga.sums[br] = P->sums[br];
                    ga.g1w = W32 + b.g1w; ga.g1b = W32 + b.g1b; ga.g2w = W32 + b.g2w; ga.g2b = W32 + b.g2b;
                    ga.gates = P->gates;
                    ga.mid = b.mid; ga.midp = midp; ga.hid = b.hid; ga.tiles = H / cs.R; ga.HW = H * Wd;
                    ga.w3 = W32 + b.cw; ga.bfold = P->bfold; ga.N = b.cout; ga.NP = pad16(b.cout);
                    ga.arrivals = P->arrivals;
                    L.chain_tiles = H / cs.R;
                    dbg(L, 200 + bi, P->Y, 4 * midp / 8, H * Wd, 4 * midp);
                    out->push_back(L);
                }
                {   // gate (x) conv3 (+ downsample / identity) + ReLU, and the next block's conv1 on the fresh tile
                    Launch L = gemm(H, Wd, {{&P->Y, 4 * midp / 8}, {X, xC8}}, bo[bi].cx, b.cout, bo[bi].cxb, true);
                    GemmTcArgs& g = L.gemm;
                    g.bfold = P->bfold;
                    g.midp = midp;
                    g.out_hi = Xo->hi; g.out_lo = Xo->lo;
                    bool fused_trans = false;
                    if (j == 0) {
                        const BlockW& nb = m->blocks[bi + 1];
                        const int nmidp = pad16(nb.mid);
                        const GemmSmem probe = gemm_smem_layout(g.K8, g.NP, nmidp, 2, true, false, 4 * 128 * 16 * 2);
                        if ((int)probe.total <= P->smem_limit) {
                            g.b2_packed = WB + bo[bi + 1].c1;
                            g.bias2 = WF + bo[bi + 1].c1b;
                            g.N2 = nb.mid; g.NP2 = nmidp;
                            g.out2_hi = P->X1.hi; g.out2_lo = P->X1.lo;
                        }
                    } else if (s < 2 && fuse_trans) {
                        // second block of a stage: the transition (1x1 + ReLU, 2x2 average pool) runs on the fresh tile, the
                        // block's own output never goes to HBM (nothing else reads it); diagnostic stops keep the two launches
                        const int C = m->c[s + 1];
                        const GemmSmem probe = gemm_smem_layout(g.K8, g.NP, C, 2, true, false, 2 * 128 * 16 * 2, true);
                        if ((int)probe.total <= P->smem_limit && g.NP + C <= 512) {
                            g.b2_packed = WB + tr[s];
                            g.bias2 = WF + trb[s];
                            g.N2 = C; g.NP2 = C;
                            g.pool2 = 1;
                            g.out_hi = nullptr; g.out_lo = nullptr;
                            g.out2_hi = Xo->hi; g.out2_lo = Xo->lo;      // pooled transition output
                            fused_trans = true;
                        }
                    }
                    if (fused_trans) {
                        ++stage;                                         // the block output itself is not materialised
                        dbg(L, stage++, *Xo, m->c[s + 1] / 8, H * Wd / 4, m->c[s + 1]);
                    } else {
                        dbg(L, stage++, *Xo, b.cout / 8, H * Wd, b.cout);
                    }
                    const bool fused_next = g.b2_packed != nullptr && !fused_trans;
                    finish(L);
                    Planes* t = X == &P->P ? Xspare : X;
                    X = Xo; Xo = t; xC8 = b.cout / 8;
                    trans_done = fused_trans;
                    if (j == 0 && !fused_next) {
                        const BlockW& nb = m->blocks[bi + 1];
                        Launch L2 = gemm(H, Wd, {{X, xC8}}, bo[bi + 1].c1, nb.mid, bo[bi + 1].c1b, true);
                        L2.gemm.out_hi = P->X1.hi; L2.gemm.out_lo = P->X1.lo;
                        dbg(L2, 100 + bi + 1, P->X1, pad16(nb.mid) / 8, H * Wd, pad16(nb.mid));
                        finish(L2);
                    }
                }
            }
            if (s < 2) {
                const int C = m->c[s + 1];
                if (!trans_done) {   // transition: 1x1 + ReLU, 2x2 average pool in the epilogue
                    Launch L = gemm(H, Wd, {{X, xC8}}, tr[s], C, trb[s], true);
                    L.gemm.pool = 1;
                    L.gemm.out_hi = Xo->hi; L.gemm.out_lo = Xo->lo;
                    dbg(L, stage++, *Xo, C / 8, H * Wd / 4, C);
                    finish(L);
                    Planes* t = X; X = Xo; Xo = t;
                }
                H /= 2; Wd /= 2;
                const BlockW& nb = m->blocks[(s + 1) * 2];
                Launch L = gemm(H, Wd, {{X, xC8}}, bo[(s + 1) * 2].c1, nb.mid, bo[(s + 1) * 2].c1b, true);
                L.gemm.out_hi = P->X1.hi; L.gemm.out_lo = P->X1.lo;
                dbg(L, 100 + (s + 1) * 2, P->X1, pad16(nb.mid) / 8, H * Wd, pad16(nb.mid));
                finish(L);
            }
        }
        {   // conv5: with the head (global average pool, fc, L2 norm) in its epilogue, or -- in the diagnostic list -- as
            // float32 NHWC for k_head
            Launch L = gemm(H, Wd, {{X, xC8}}, c5, m->c[3], c5b, true);
            if (fuse_trans && H * Wd == 128) {
                L.gemm.head_w = W32 + m->fcw;
                L.gemm.head_b = W32 + m->fcb;
                L.gemm.head_feat = m->feat;
                L.cls = CLS_HEAD;
                P->head_fused = true;
            } else {
                L.gemm.out_f32 = P->c5;
            }
            L.stage_after = 11;
            finish(L);
        }
        };
        build_launches(true, &P->launches);
        build_launches(false, &P->launches_dbg);   // diagnostic stops at block outputs need the unfused transition
    } catch (...) {
        plan_free(P);
        throw;
    }
    return P;
}

// Replays the plan for one chunk of crops (the stem output of that chunk is in m->bufA).  Returns true when a debug tap
// stopped the chunk.
struct FrontInput { const uint8_t* images; size_t image_stride; int rows, cols; const CropDesc* crops; float* out; int out_ld; };

template <class Prof>
bool plan_run(ReidModel* m, const FrontInput& fi, const int* d_n, int off, int upper, cudaStream_t st, Prof& prof) {
    Plan* P = m->tc;
    for (const Launch& L : (m->debug_stop >= 0 ? P->launches_dbg : P->launches)) {
        prof.begin(L.cls);
        switch (L.kind) {
            case LK_FRONT: {
                FrontTcArgs fa = L.front;
                fa.images = fi.images; fa.image_stride = fi.image_stride; fa.rows = fi.rows; fa.cols = fi.cols; fa.crops = fi.crops;
                fa.pad_mode = m->preprocess;
                if (m->debug_stop == 50) {
                    if (!P->dbg_crop) RCUDA_OK(cudaMalloc(&P->dbg_crop, sizeof(float) * (size_t)P->chunk * 256 * 128 * 3));
                    fa.dbg_crop = P->dbg_crop;
                }
                k_front_tc<<<dim3(4, upper), 256, FR_SMEM, st>>>(fa, d_n, off, upper);
                break;
            }
            case LK_MAXPOOL_PLANES:
                k_maxpool_planes<<<m->sms * 4, 256, 0, st>>>(m->bufA, 128, 64, m->c[0], d_n, off, upper, P->P.hi, P->P.lo);
                break;
            case LK_CHAIN_S2:
                chain_launch<BMB_CHAIN_S2>(L.chain, L.chain_tiles, upper, d_n, off, st);
                break;
            case LK_CHAIN_S3:
                chain_launch<BMB_CHAIN_S3>(L.chain, L.chain_tiles, upper, d_n, off, st);
                break;
            case LK_CHAIN_S4:
                chain_launch<BMB_CHAIN_S4>(L.chain, L.chain_tiles, upper, d_n, off, st);
                break;
            case LK_GEMM:
                L.gemm_fn<<<dim3(L.gemm_groups, upper), GEMM_THREADS, L.gl.total, st>>>(L.gemm, d_n, off, upper, L.gl, GemmHeadIO{fi.crops, fi.out, fi.out_ld});
                break;
        }
        prof.end();
        if (m->debug_stop == 50 && L.kind == LK_FRONT) {
            m->debug_ptr = P->dbg_crop;
            m->debug_floats_per_crop = (size_t)256 * 128 * 3;
            return true;
        }
        if (m->debug_stop >= 0 && L.stage_after == m->debug_stop) {
            if (L.stage_after == 11) {
                m->debug_ptr = P->c5;
                m->debug_floats_per_crop = (size_t)128 * m->c[3];
            } else {
                k_planes_to_nhwc<<<m->sms * 4, 256, 0, st>>>(L.dbg_hi, L.dbg_lo, L.dbg_C8, L.dbg_HW, L.dbg_C, d_n, off, upper, P->dbg);
                m->debug_ptr = P->dbg;
                m->debug_floats_per_crop = (size_t)L.dbg_HW * L.dbg_C;
            }
            return true;
        }
    }
    return false;
}

}  // namespace tcx
}  // namespace bmb
