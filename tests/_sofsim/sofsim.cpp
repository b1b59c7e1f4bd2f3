// tests/_sofsim/sofsim.cpp -- TEST INFRASTRUCTURE ONLY.
// Compiles boxmot_b200/csrc/cmc_sof.cuh for the host (BMB_HOSTSIM: one "thread") and composes its functions serially
// into SOF.apply, so the CPU tests can pin the arithmetic on the installed OpenCV and the GPU tests can pin the kernels
// on this build bit for bit.  Built by tests/sofsim.py with g++; never linked into libboxmot_b200.so.
#define BMB_HOSTSIM 1
#include <algorithm>
#include <cstring>
#include <vector>

#include "cmc_sof.cuh"

using namespace bmb;

namespace {

void host_pyramid(const uint8_t* gray, const SofGeom& g, std::vector<uint8_t>& pyr, std::vector<int16_t>& der) {
    pyr.assign(g.npx, 0);
    der.assign(2 * (size_t)g.npx, 0);
    std::memcpy(pyr.data(), gray, (size_t)g.h * g.w);
    for (int l = 1; l < g.nlev; ++l)
        for (int y = 0; y < g.lh[l]; ++y)
            for (int x = 0; x < g.lw[l]; ++x)
                pyr[g.off[l] + y * g.lw[l] + x] = sof_pyrdown_pixel(pyr.data() + g.off[l - 1], g.lh[l - 1], g.lw[l - 1], y, x);
    for (int l = 0; l < g.nlev; ++l)
        for (int y = 0; y < g.lh[l]; ++y)
            for (int x = 0; x < g.lw[l]; ++x)
                sof_scharr_pixel(pyr.data() + g.off[l], g.lh[l], g.lw[l], y, x,
                                 der.data() + 2 * ((size_t)g.off[l] + y * g.lw[l] + x));
}

void host_eig(const uint8_t* gray, int h, int w, std::vector<float>& E) {
    std::vector<float> DX((size_t)h * w), DY((size_t)h * w);
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) sof_sobel(gray, h, w, y, x, DX[(size_t)y * w + x], DY[(size_t)y * w + x]);
    E.resize((size_t)h * w);
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) E[(size_t)y * w + x] = sof_eig_pixel(DX.data(), DY.data(), h, w, y, x);
}

int host_corners(const uint8_t* gray, int h, int w, const uint8_t* mask, float* xy) {
    std::vector<float> E;
    host_eig(gray, h, w, E);
    bool any = false;
    float mx = 0.f;
    for (size_t p = 0; p < E.size(); ++p)
        if (mask[p] && (!any || E[p] > mx)) { mx = E[p]; any = true; }
    const float thr = (float)((double)mx * 0.01);
    std::vector<uint64_t> keys;
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
            const uint64_t k = sof_candidate(E.data(), mask, h, w, y, x, thr);
            if (k) keys.push_back(k);
        }
    std::sort(keys.begin(), keys.end(), [](uint64_t a, uint64_t b) { return a > b; });
    const int n = (int)std::min<size_t>(keys.size(), SOF_MAX_CORNERS);
    for (int i = 0; i < n; ++i) sof_key_point(keys[i], w, xy + 2 * i);
    return n;
}

// RANSAC + refine on point pairs; returns 1 and M when a model was found (inlier mask in `inl`)
int host_ransac(const float* src, const float* dst, int n, float thr, double* M, uint8_t* inl, int* n_inl) {
    std::vector<int> pairs(2 * SOF_RANSAC_ITERS), good(SOF_RANSAC_ITERS);
    sof_draw_pairs(n, SOF_RANSAC_ITERS, pairs.data());
    const float thr2 = (float)((double)thr * (double)thr);
    std::vector<double> models(6 * (size_t)SOF_RANSAC_ITERS);
    for (int it = 0; it < SOF_RANSAC_ITERS; ++it) {
        double* m = models.data() + 6 * it;
        const int a = pairs[2 * it], b = pairs[2 * it + 1];
        sof_model(src + 2 * a, src + 2 * b, dst + 2 * a, dst + 2 * b, m);
        int c = 0;
        for (int i = 0; i < n; ++i) c += sof_inlier(m, src + 2 * i, dst + 2 * i, thr2);
        good[it] = c;
    }
    int best_good = 0;
    const int best = sof_ransac_pick(good.data(), n, &best_good);
    *n_inl = 0;
    if (best < 0) {
        std::memset(inl, 0, n);
        return 0;
    }
    std::memcpy(M, models.data() + 6 * best, 6 * sizeof(double));
    std::vector<float> s, d;
    for (int i = 0; i < n; ++i) {
        inl[i] = (uint8_t)sof_inlier(M, src + 2 * i, dst + 2 * i, thr2);
        if (inl[i]) {
            s.push_back(src[2 * i]); s.push_back(src[2 * i + 1]);
            d.push_back(dst[2 * i]); d.push_back(dst[2 * i + 1]);
        }
    }
    *n_inl = (int)(s.size() / 2);
    std::vector<double> red(6 * SOF_RED);
    sof_refine(s.data(), d.data(), *n_inl, M, red.data());
    return 1;
}

struct SofHost {
    double scale;
    float thr;
    int min_inliers;
    double min_ratio;
    int h = 0, w = 0, initialized = 0;
    SofGeom g;
    std::vector<uint8_t> pyr;
    std::vector<int16_t> der;
    std::vector<float> kps;   // previous keypoints, 2 per point
};

}  // namespace

extern "C" {

void sofsim_eig(const uint8_t* gray, int h, int w, float* out) {
    std::vector<float> E;
    host_eig(gray, h, w, E);
    std::memcpy(out, E.data(), E.size() * sizeof(float));
}

void sofsim_mask(int h, int w, const float* dets, int n, int stride, float scale, uint8_t* out) {
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) out[(size_t)y * w + x] = sof_mask_pixel(h, w, y, x, dets, n, stride, scale);
}

int sofsim_corners(const uint8_t* gray, int h, int w, const uint8_t* mask, float* xy) {
    return host_corners(gray, h, w, mask, xy);
}

void sofsim_subpix(const uint8_t* gray, int h, int w, float* xy, int n) {
    for (int i = 0; i < n; ++i) sof_subpix_point(gray, h, w, xy + 2 * i);
}

int sofsim_levels(int h, int w) { return sof_geom(h, w).nlev; }

void sofsim_lk(const uint8_t* prev, const uint8_t* cur, int h, int w, const float* pts, int n, float* out, int* status) {
    const SofGeom g = sof_geom(h, w);
    std::vector<uint8_t> P, C;
    std::vector<int16_t> DP, DC;
    host_pyramid(prev, g, P, DP);
    host_pyramid(cur, g, C, DC);
    for (int i = 0; i < n; ++i) sof_lk_point(g, P.data(), DP.data(), C.data(), pts[2 * i], pts[2 * i + 1], out + 2 * i, status + i);
}

int sofsim_ransac(const float* src, const float* dst, int n, float thr, double* M, uint8_t* inl, int* n_inl) {
    return host_ransac(src, dst, n, thr, M, inl, n_inl);
}

void* sofsim_create(double scale, int min_inliers, double min_ratio, float thr) {
    SofHost* s = new SofHost();
    s->scale = scale; s->min_inliers = min_inliers; s->min_ratio = min_ratio; s->thr = thr;
    return s;
}

void sofsim_destroy(void* p) { delete (SofHost*)p; }

// SOF.apply on one BGR frame: warp6 (float32, row major), status SOF_INIT / SOF_ESTIMATED / SOF_REJECTED,
// `reg` (optional) receives the registration image
void sofsim_apply(void* p, const uint8_t* bgr, int rows, int cols, const float* dets, int n_dets, int det_stride,
                  float* warp6, int* status, uint8_t* reg) {
    SofHost& s = *(SofHost*)p;
    int h, w;
    h = (int)nearbyint(rows * s.scale);
    w = (int)nearbyint(cols * s.scale);
    std::vector<uint8_t> gray((size_t)h * w), mask((size_t)h * w);
    const double inv = 1.0 / s.scale;
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) {
            gray[(size_t)y * w + x] = cmc_prepare_pixel(bgr, rows, cols, inv, y, x);
            mask[(size_t)y * w + x] = sof_mask_pixel(h, w, y, x, dets, n_dets, det_stride, (float)s.scale);
        }
    if (reg) std::memcpy(reg, gray.data(), gray.size());
    if (h != s.h || w != s.w) { s.h = h; s.w = w; s.initialized = 0; s.kps.clear(); }
    const SofGeom g = sof_geom(h, w);
    std::vector<uint8_t> pyr;
    std::vector<int16_t> der;
    host_pyramid(gray.data(), g, pyr, der);
    std::vector<float> corners(2 * SOF_MAX_CORNERS);
    const int nc = host_corners(gray.data(), h, w, mask.data(), corners.data());
    corners.resize(2 * nc);
    const float eye[6] = {1.f, 0.f, 0.f, 0.f, 1.f, 0.f};
    std::memcpy(warp6, eye, sizeof(eye));
    int st = SOF_REJECTED;
    if (!s.initialized) {
        st = SOF_INIT;
        if (nc >= 4) sofsim_subpix(gray.data(), h, w, corners.data(), nc);
        s.kps = corners;
        s.initialized = nc >= 4;
    } else {
        const int np = (int)s.kps.size() / 2;
        std::vector<float> nxt(2 * np), pv, nv;
        std::vector<int> ok(np);
        for (int i = 0; i < np; ++i)
            sof_lk_point(g, s.pyr.data(), s.der.data(), pyr.data(), s.kps[2 * i], s.kps[2 * i + 1], nxt.data() + 2 * i, &ok[i]);
        for (int i = 0; i < np; ++i)
            if (ok[i]) {
                pv.push_back(s.kps[2 * i]); pv.push_back(s.kps[2 * i + 1]);
                nv.push_back(nxt[2 * i]); nv.push_back(nxt[2 * i + 1]);
            }
        const int nvalid = (int)pv.size() / 2;
        if (nvalid < 4) {   // SOF._reset
            s.kps = corners;
            s.initialized = nc >= 4;
        } else {
            double M[6];
            std::vector<uint8_t> inl(nvalid);
            int n_inl = 0;
            const int found = host_ransac(pv.data(), nv.data(), nvalid, s.thr, M, inl.data(), &n_inl);
            if (found && sof_accept(n_inl, nvalid, s.min_inliers, s.min_ratio)) {
                sof_warp_out(M, (float)s.scale, warp6);
                st = SOF_ESTIMATED;
            }
            s.kps = nc >= 4 ? corners : nv;
            s.initialized = 1;
        }
    }
    s.pyr.swap(pyr);
    s.der.swap(der);
    *status = st;
}

}  // extern "C"
