// cmc_sof.cuh -- camera-motion estimation on the device: the reference's sparse-optical-flow estimator (SOF).
//
// Replaces boxmot/motion/cmc/sof.py (`SOF.apply` with its defaults: scale 0.15, goodFeaturesToTrack(maxCorners 1000,
// qualityLevel 0.01, minDistance 1, blockSize 3, min-eigenvalue response), cornerSubPix(5x5 half window) on the
// initialising frame, calcOpticalFlowPyrLK(21x21, maxLevel 3, 30 iterations, eps 0.01), estimateAffinePartial2D(RANSAC,
// threshold 3, 2000 iterations, confidence 0.99, 10 refine iterations), then the inlier gate (>= 8 inliers, ratio
// >= 0.2)) and base_cmc.py (`preprocess`, `generate_mask`).
//
// The arithmetic restates the OpenCV calls (third party) in float32 image arithmetic and their operation order, with
// three deliberate changes that make every reduction independent of how the device splits it:
//   * the LK window sums (441 integer products per iteration) are accumulated exactly in int64 (OpenCV sums the same
//     integers in float, so the two differ by float rounding only);
//   * the 3x3 box sums of cornerMinEigenVal are taken in float64 in a fixed order and rounded once;
//   * the Levenberg-Marquardt sums over the inliers are lane-strided partials over SOF_RED slots reduced by a fixed
//     tree (sof_lm_eval); the 4x4 normal equations are solved by Gaussian elimination instead of DECOMP_EIG.
// Every other value is computed per pixel / per point by the same expression on the host and on the device, so the
// host build (tests/_sofsim) and the kernels (cmc_sof_kernels.cu, -fmad=false) give bit-identical results.  The one
// transcendental on the path is RANSAC's log() in sof_update_iters (see there).
//
// Data per stream: the registration image (rint(rows*0.15) x rint(cols*0.15), 162 x 288 at 1080p) and its pyramid
// (OpenCV's level count: a level is added while both halved sides stay > 21), int16 Scharr derivatives of every level,
// at most SOF_MAX_CORNERS keypoints.
#pragma once
#include <float.h>
#include <stdint.h>
#include <string.h>

#include "cmc_ecc.cuh"

namespace bmb {

constexpr int SOF_MAX_CORNERS = 1000;
constexpr int SOF_WIN = 21;             // LK window side
constexpr int SOF_WIN_AREA = SOF_WIN * SOF_WIN;
constexpr int SOF_MAX_LEVELS = 4;       // maxLevel 3
constexpr int SOF_LK_ITERS = 30;
constexpr int SOF_SUBPIX_HALF = 5;      // cornerSubPix winSize (5, 5): an 11 x 11 window
constexpr int SOF_SUBPIX_ITERS = 30;
constexpr int SOF_RANSAC_ITERS = 2000;
constexpr int SOF_LM_ITERS = 10;
constexpr int SOF_RED = 256;            // slots of the fixed-order LM reduction (= threads of the refine CTA)
enum { SOF_INIT = 0, SOF_ESTIMATED = 1, SOF_REJECTED = 2 };

BMB_FN int sof_reflect(int i, int n) {   // BORDER_REFLECT_101
    if (n == 1) return 0;
    while (i < 0 || i >= n) i = i < 0 ? -i : 2 * n - 2 - i;
    return i;
}

// pyramid geometry (buildOpticalFlowPyramid's level count for winSize 21) and offsets of each level in the packed
// per-stream buffers
struct SofGeom {
    int h, w, nlev;
    int lh[SOF_MAX_LEVELS], lw[SOF_MAX_LEVELS];
    int off[SOF_MAX_LEVELS];   // pixel offset of each level; total pixels in `npx`
    int npx;
};

#if BMB_DEVICE
__host__ __device__ inline
#else
static inline
#endif
SofGeom sof_geom(int h, int w) {   // also called by the host code that sizes the buffers
    SofGeom g;
    g.h = h; g.w = w;
    g.lh[0] = h; g.lw[0] = w; g.off[0] = 0;
    int L = 0;
    while (L + 1 < SOF_MAX_LEVELS) {
        const int nh = (g.lh[L] + 1) / 2, nw = (g.lw[L] + 1) / 2;
        if (nw <= SOF_WIN || nh <= SOF_WIN) break;
        g.off[L + 1] = g.off[L] + g.lh[L] * g.lw[L];
        ++L;
        g.lh[L] = nh; g.lw[L] = nw;
    }
    g.nlev = L + 1;
    g.npx = g.off[L] + g.lh[L] * g.lw[L];
    for (int k = g.nlev; k < SOF_MAX_LEVELS; ++k) { g.lh[k] = 0; g.lw[k] = 0; g.off[k] = g.npx; }
    return g;
}

// ---- BaseCMC.generate_mask ---------------------------------------------------------------------------------------
// one detection box in registration pixels: float32(coord) * float32(scale), truncated toward zero, clamped
BMB_FN int sof_box_coord(float c, float scale, int lim) {
    float v = c * scale;
    if (!(v == v)) v = 0.f;
    v = v < -1e9f ? -1e9f : (v > 1e9f ? 1e9f : v);
    int i = (int)v;
    return i < 0 ? 0 : (i > lim ? lim : i);
}

// `conf_col` >= 0 keeps only the rows with d[conf_col] > conf_thr (float32): DeepOCSORT passes the detections it
// keeps (deepocsort.py:330-347), BoT-SORT every row (conf_col -1)
BMB_FN uint8_t sof_mask_pixel(int h, int w, int y, int x, const float* dets, int n_dets, int det_stride, float scale,
                              int conf_col = -1, float conf_thr = 0.f) {
    const int y1 = (int)(0.02 * h), y2 = (int)(0.98 * h), x1 = (int)(0.02 * w), x2 = (int)(0.98 * w);
    if (y < y1 || y >= y2 || x < x1 || x >= x2) return 0;
    for (int i = 0; i < n_dets; ++i) {
        const float* d = dets + (size_t)i * det_stride;
        if (conf_col >= 0 && !(d[conf_col] > conf_thr)) continue;
        const int bx1 = sof_box_coord(d[0], scale, w), by1 = sof_box_coord(d[1], scale, h);
        const int bx2 = sof_box_coord(d[2], scale, w), by2 = sof_box_coord(d[3], scale, h);
        if (bx2 > bx1 && by2 > by1 && x >= bx1 && x < bx2 && y >= by1 && y < by2) return 0;
    }
    return 255;
}

// ---- cornerMinEigenVal(blockSize 3, ksize 3) -----------------------------------------------------------------------
// Sobel dx and dy of the uint8 image at (y, x), CV_32F, scale 1 / (4 * 3 * 255) applied to the smoothing kernel
BMB_FN void sof_sobel(const uint8_t* I, int h, int w, int y, int x, float& dx, float& dy) {
    const float k0 = (float)(2.0 * (1.0 / 3060.0)), k1 = (float)(1.0 / 3060.0);
    const int xl = sof_reflect(x - 1, w), xr = sof_reflect(x + 1, w);
    const int yu = sof_reflect(y - 1, h), yd = sof_reflect(y + 1, h);
    const uint8_t *ru = I + (size_t)yu * w, *rc = I + (size_t)y * w, *rd = I + (size_t)yd * w;
    // dx: row [-1 0 1], column [1 2 1] * scale (SymmColumnFilter: centre tap, then the sum of the symmetric pair)
    const float du = (float)((int)ru[xr] - (int)ru[xl]), dc = (float)((int)rc[xr] - (int)rc[xl]);
    const float dd = (float)((int)rd[xr] - (int)rd[xl]);
    dx = dc * k0 + (du + dd) * k1;
    // dy: row [1 2 1] * scale, column [-1 0 1]
    const float su = (k1 * (float)ru[xl] + k0 * (float)ru[x]) + k1 * (float)ru[xr];
    const float sd = (k1 * (float)rd[xl] + k0 * (float)rd[x]) + k1 * (float)rd[xr];
    dy = sd - su;
}

// minimum eigenvalue from the Sobel images DX, DY (h x w float32): unnormalised 3x3 box of the products (reflect-101),
// summed in float64 and rounded once, then cv::calcMinEigenVal
BMB_FN float sof_eig_pixel(const float* DX, const float* DY, int h, int w, int y, int x) {
    double sa = 0.0, sb = 0.0, sc = 0.0;
    for (int r = -1; r <= 1; ++r) {
        const int yy = sof_reflect(y + r, h);
        for (int c = -1; c <= 1; ++c) {
            const size_t p = (size_t)yy * w + sof_reflect(x + c, w);
            const float gx = DX[p], gy = DY[p];
            sa += (double)(gx * gx);
            sb += (double)(gx * gy);
            sc += (double)(gy * gy);
        }
    }
    const float a = (float)sa * 0.5f, b = (float)sb, c = (float)sc * 0.5f;
    return (a + c) - sqrtf((a - c) * (a - c) + b * b);
}

// ---- goodFeaturesToTrack -------------------------------------------------------------------------------------------
// order-preserving bits of a float: larger value -> larger key
BMB_FN uint32_t sof_fkey(float v) {
#if BMB_DEVICE
    const uint32_t u = __float_as_uint(v);
#else
    uint32_t u;
    memcpy(&u, &v, 4);
#endif
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// a candidate corner: inside the one-pixel border, above the quality threshold (THRESH_TOZERO), equal to the 3x3
// dilation of the thresholded map, inside the mask.  Returns the sort key (value, then address, both descending =
// OpenCV's greaterThanPtr) or 0.
BMB_FN uint64_t sof_candidate(const float* E, const uint8_t* mask, int h, int w, int y, int x, float thr) {
    if (y < 1 || y >= h - 1 || x < 1 || x >= w - 1) return 0;
    const size_t p = (size_t)y * w + x;
    const float v = E[p] > thr ? E[p] : 0.f;
    if (v == 0.f || !mask[p]) return 0;
    for (int r = -1; r <= 1; ++r)
        for (int c = -1; c <= 1; ++c) {
            const float e = E[p + (ptrdiff_t)r * w + c];
            if ((e > thr ? e : 0.f) > v) return 0;
        }
    return ((uint64_t)sof_fkey(v) << 32) | (uint64_t)p;
}

BMB_FN void sof_key_point(uint64_t key, int w, float* xy) {
    const int p = (int)(key & 0xffffffffu);
    xy[0] = (float)(p % w);
    xy[1] = (float)(p / w);
}

// ---- cornerSubPix(winSize (5, 5), zeroZone (-1, -1), (COUNT | EPS, 30, 0.01)) ---------------------------------------
BMB_FN float sof_subpix_weight(int k) {   // exp(-x*x) for x = (k - 5) / 5 in float32
    const int a = k < SOF_SUBPIX_HALF ? SOF_SUBPIX_HALF - k : k - SOF_SUBPIX_HALF;
    const float t[6] = {0x1p+0f, 0x1.ebec98p-1f, 0x1.b44c3p-1f, 0x1.6535d4p-1f, 0x1.0df944p-1f, 0x1.78b564p-2f};
    return t[a];
}

// bilinear sample of the uint8 image at integer offset (iy, ix) + fractions (a, b), replicated border
BMB_FN float sof_rect_px(const uint8_t* I, int h, int w, int iy, int ix, float a, float b) {
    const int x0 = ix < 0 ? 0 : (ix >= w ? w - 1 : ix), x1 = ix + 1 < 0 ? 0 : (ix + 1 >= w ? w - 1 : ix + 1);
    const int y0 = iy < 0 ? 0 : (iy >= h ? h - 1 : iy), y1 = iy + 1 < 0 ? 0 : (iy + 1 >= h ? h - 1 : iy + 1);
    const float p00 = I[(size_t)y0 * w + x0], p01 = I[(size_t)y0 * w + x1];
    const float p10 = I[(size_t)y1 * w + x0], p11 = I[(size_t)y1 * w + x1];
    return (p00 * ((1.f - a) * (1.f - b)) + p01 * (a * (1.f - b))) + (p10 * ((1.f - a) * b) + p11 * (a * b));
}

BMB_FN void sof_subpix_point(const uint8_t* I, int h, int w, float* xy) {
    constexpr int WW = 2 * SOF_SUBPIX_HALF + 1, SW = WW + 2;
    const float cTx = xy[0], cTy = xy[1];
    float cx = cTx, cy = cTy;
    const double eps = 0.01 * 0.01;
    int iter = 0;
    double err = 0.0;
    do {
        // getRectSubPix(Size(13, 13), cI): window origin cI - 6, one bilinear fraction pair for every sample
        const float ox = cx - (float)(SW - 1) * 0.5f, oy = cy - (float)(SW - 1) * 0.5f;
        const int ix = (int)floorf(ox), iy = (int)floorf(oy);
        const float fa = ox - (float)ix, fb = oy - (float)iy;
        double a = 0, b = 0, c = 0, bb1 = 0, bb2 = 0;
        for (int i = 0; i < WW; ++i) {
            const double py = i - SOF_SUBPIX_HALF;
            const float wy = sof_subpix_weight(i);
            for (int j = 0; j < WW; ++j) {
                const double m = (double)(wy * sof_subpix_weight(j));
                const float sl = sof_rect_px(I, h, w, iy + i + 1, ix + j, fa, fb);
                const float sr = sof_rect_px(I, h, w, iy + i + 1, ix + j + 2, fa, fb);
                const float su = sof_rect_px(I, h, w, iy + i, ix + j + 1, fa, fb);
                const float sd = sof_rect_px(I, h, w, iy + i + 2, ix + j + 1, fa, fb);
                const double tgx = (double)(sr - sl), tgy = (double)(sd - su);
                const double gxx = tgx * tgx * m, gxy = tgx * tgy * m, gyy = tgy * tgy * m;
                const double px = j - SOF_SUBPIX_HALF;
                a += gxx; b += gxy; c += gyy;
                bb1 += gxx * px + gxy * py;
                bb2 += gxy * px + gyy * py;
            }
        }
        const double det = a * c - b * b;
        if (fabs(det) <= DBL_EPSILON * DBL_EPSILON) break;
        const double s = 1.0 / det;
        const float nx = (float)(cx + c * s * bb1 - b * s * bb2);
        const float ny = (float)(cy - b * s * bb1 + a * s * bb2);
        err = (double)((nx - cx) * (nx - cx) + (ny - cy) * (ny - cy));
        cx = nx; cy = ny;
        if (cx < 0 || cx >= w || cy < 0 || cy >= h) break;
    } while (++iter < SOF_SUBPIX_ITERS && err > eps);
    if (fabsf(cx - cTx) > SOF_SUBPIX_HALF || fabsf(cy - cTy) > SOF_SUBPIX_HALF) { cx = cTx; cy = cTy; }
    xy[0] = cx; xy[1] = cy;
}

// ---- pyramid: pyrDown (uint8, 5x5 [1 4 6 4 1]^2 / 256, reflect-101) and Scharr derivatives (int16, zero outside) ----
BMB_FN uint8_t sof_pyrdown_pixel(const uint8_t* S, int sh, int sw, int y, int x) {
    const int k[5] = {1, 4, 6, 4, 1};
    int acc = 0;
    for (int r = 0; r < 5; ++r) {
        const uint8_t* row = S + (size_t)sof_reflect(2 * y - 2 + r, sh) * sw;
        int rs = 0;
        for (int c = 0; c < 5; ++c) rs += k[c] * (int)row[sof_reflect(2 * x - 2 + c, sw)];
        acc += k[r] * rs;
    }
    return (uint8_t)((acc + 128) >> 8);
}

BMB_FN void sof_scharr_pixel(const uint8_t* I, int h, int w, int y, int x, int16_t* d) {
    const int yu = sof_reflect(y - 1, h), yd = sof_reflect(y + 1, h);
    const int xl = sof_reflect(x - 1, w), xr = sof_reflect(x + 1, w);
    const uint8_t *ru = I + (size_t)yu * w, *rc = I + (size_t)y * w, *rd = I + (size_t)yd * w;
    auto t0 = [&](int xx) { return ((int)ru[xx] + (int)rd[xx]) * 3 + (int)rc[xx] * 10; };
    auto t1 = [&](int xx) { return (int)rd[xx] - (int)ru[xx]; };
    d[0] = (int16_t)(t0(xr) - t0(xl));
    d[1] = (int16_t)((t1(xr) + t1(xl)) * 3 + t1(x) * 10);
}

// ---- calcOpticalFlowPyrLK(winSize 21, maxLevel 3, (COUNT | EPS, 30, 0.01), flags 0, minEigThreshold 1e-4) ---------
BMB_FN int sof_descale(int v, int n) { return (v + (1 << (n - 1))) >> n; }

BMB_FN long long sof_sum_ll(long long v) {   // sum over the warp (every lane gets it); exact, so any order
#if BMB_DEVICE
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
#endif
    return v;
}

#if BMB_DEVICE
constexpr int SOF_LK_SLOTS = (SOF_WIN_AREA + 31) / 32;   // window samples per lane
#define SOF_LK_LANE ((int)(threadIdx.x & 31))
#define SOF_LK_NL 32
#else
constexpr int SOF_LK_SLOTS = SOF_WIN_AREA;
#define SOF_LK_LANE 0
#define SOF_LK_NL 1
#endif

BMB_FN int sof_px(const uint8_t* I, int h, int w, int y, int x) {
    return I[(size_t)sof_reflect(y, h) * w + sof_reflect(x, w)];
}

BMB_FN void sof_dpx(const int16_t* D, int h, int w, int y, int x, int& dx, int& dy) {
    if (y < 0 || y >= h || x < 0 || x >= w) { dx = 0; dy = 0; return; }
    dx = D[2 * ((size_t)y * w + x)];
    dy = D[2 * ((size_t)y * w + x) + 1];
}

BMB_FN void sof_weights(float a, float b, int* iw) {
    iw[0] = BMB_F2I_RN((1.f - a) * (1.f - b) * 16384.f);
    iw[1] = BMB_F2I_RN(a * (1.f - b) * 16384.f);
    iw[2] = BMB_F2I_RN((1.f - a) * b * 16384.f);
    iw[3] = 16384 - iw[0] - iw[1] - iw[2];
}

// Track one point from the previous pyramid (images P, derivatives DP) to the current one (images C).  On the device
// a whole warp calls this for the same point (lanes stride over the window); on the host one thread does.
BMB_FN void sof_lk_point(const SofGeom& g, const uint8_t* P, const int16_t* DP, const uint8_t* C, float px, float py,
                         float* out, int* status) {
    const float half = (float)(SOF_WIN - 1) * 0.5f;
    const float FLT_SCALE = 1.f / (1 << 20);
    const int lane = SOF_LK_LANE;
    int Iv[SOF_LK_SLOTS], Ix[SOF_LK_SLOTS], Iy[SOF_LK_SLOTS];
    float sx = 0.f, sy = 0.f;   // nextPts[i] as OpenCV stores it between iterations and levels
    int st = 1;
    for (int level = g.nlev - 1; level >= 0; --level) {
        const int rows = g.lh[level], cols = g.lw[level];
        const uint8_t* I = P + g.off[level];
        const int16_t* dI = DP + 2 * (size_t)g.off[level];
        const uint8_t* J = C + g.off[level];
        const float ls = (float)(1.0 / (1 << level));
        float pX = px * ls, pY = py * ls;
        if (level == g.nlev - 1) { sx = pX; sy = pY; } else { sx = sx * 2.f; sy = sy * 2.f; }
        float nX = sx, nY = sy;
        pX -= half; pY -= half;
        const int ipx = (int)floorf(pX), ipy = (int)floorf(pY);
        if (ipx < -SOF_WIN || ipx >= cols || ipy < -SOF_WIN || ipy >= rows) {
            if (level == 0) st = 0;
            continue;
        }
        int iw[4];
        sof_weights(pX - (float)ipx, pY - (float)ipy, iw);
        long long a11 = 0, a12 = 0, a22 = 0;
        for (int s = 0; s < SOF_LK_SLOTS; ++s) {
            const int k = lane + s * SOF_LK_NL;
            if (k >= SOF_WIN_AREA) break;
            const int y = ipy + k / SOF_WIN, x = ipx + k % SOF_WIN;
            Iv[s] = sof_descale(sof_px(I, rows, cols, y, x) * iw[0] + sof_px(I, rows, cols, y, x + 1) * iw[1] +
                                sof_px(I, rows, cols, y + 1, x) * iw[2] + sof_px(I, rows, cols, y + 1, x + 1) * iw[3], 9);
            int d00x, d00y, d01x, d01y, d10x, d10y, d11x, d11y;
            sof_dpx(dI, rows, cols, y, x, d00x, d00y);
            sof_dpx(dI, rows, cols, y, x + 1, d01x, d01y);
            sof_dpx(dI, rows, cols, y + 1, x, d10x, d10y);
            sof_dpx(dI, rows, cols, y + 1, x + 1, d11x, d11y);
            Ix[s] = sof_descale(d00x * iw[0] + d01x * iw[1] + d10x * iw[2] + d11x * iw[3], 14);
            Iy[s] = sof_descale(d00y * iw[0] + d01y * iw[1] + d10y * iw[2] + d11y * iw[3], 14);
            a11 += (long long)Ix[s] * Ix[s];
            a12 += (long long)Ix[s] * Iy[s];
            a22 += (long long)Iy[s] * Iy[s];
        }
        const float A11 = (float)sof_sum_ll(a11) * FLT_SCALE, A12 = (float)sof_sum_ll(a12) * FLT_SCALE;
        const float A22 = (float)sof_sum_ll(a22) * FLT_SCALE;
        float D = A11 * A22 - A12 * A12;
        const float min_eig = (A22 + A11 - sqrtf((A11 - A22) * (A11 - A22) + 4.f * A12 * A12)) /
                              (float)(2 * SOF_WIN * SOF_WIN);
        if (min_eig < 1e-4f || D < FLT_EPSILON) {
            if (level == 0) st = 0;
            continue;
        }
        D = 1.f / D;
        nX -= half; nY -= half;
        float pdx = 0.f, pdy = 0.f;
        for (int j = 0; j < SOF_LK_ITERS; ++j) {
            const int inx = (int)floorf(nX), iny = (int)floorf(nY);
            if (inx < -SOF_WIN || inx >= cols || iny < -SOF_WIN || iny >= rows) {
                if (level == 0) st = 0;
                break;
            }
            sof_weights(nX - (float)inx, nY - (float)iny, iw);
            long long b1 = 0, b2 = 0;
            for (int s = 0; s < SOF_LK_SLOTS; ++s) {
                const int k = lane + s * SOF_LK_NL;
                if (k >= SOF_WIN_AREA) break;
                const int y = iny + k / SOF_WIN, x = inx + k % SOF_WIN;
                const int diff = sof_descale(sof_px(J, rows, cols, y, x) * iw[0] + sof_px(J, rows, cols, y, x + 1) * iw[1] +
                                             sof_px(J, rows, cols, y + 1, x) * iw[2] +
                                             sof_px(J, rows, cols, y + 1, x + 1) * iw[3], 9) - Iv[s];
                b1 += (long long)diff * Ix[s];
                b2 += (long long)diff * Iy[s];
            }
            const float B1 = (float)sof_sum_ll(b1) * FLT_SCALE, B2 = (float)sof_sum_ll(b2) * FLT_SCALE;
            const float dx = (A12 * B2 - A22 * B1) * D, dy = (A12 * B1 - A11 * B2) * D;
            nX += dx; nY += dy;
            sx = nX + half; sy = nY + half;
            if ((double)dx * dx + (double)dy * dy <= 0.01 * 0.01) break;
            if (j > 0 && fabsf(dx + pdx) < 0.01 && fabsf(dy + pdy) < 0.01) {
                sx -= dx * 0.5f; sy -= dy * 0.5f;
                break;
            }
            pdx = dx; pdy = dy;
        }
    }
    out[0] = sx; out[1] = sy;
    *status = st;
}

// ---- estimateAffinePartial2D(RANSAC, 3.0, 2000, 0.99, 10) -----------------------------------------------------------
// the index pairs RANSACPointSetRegistrator draws: cv::RNG((uint64)-1), rng.uniform(0, count), a second draw repeated
// while it equals the first (checkSubset never rejects two points).  The draws do not depend on the models.
BMB_FN void sof_draw_pairs(int count, int iters, int* pairs) {
    uint64_t s = ~0ull;
    auto next = [&]() -> unsigned { s = (uint64_t)(unsigned)s * 4164903690ull + (unsigned)(s >> 32); return (unsigned)s; };
    for (int it = 0; it < iters; ++it) {
        const int i0 = (int)(next() % (unsigned)count);
        int i1;
        do i1 = (int)(next() % (unsigned)count); while (i1 == i0);
        pairs[2 * it] = i0;
        pairs[2 * it + 1] = i1;
    }
}

// AffinePartial2DEstimatorCallback::runKernel: the similarity through two point pairs, M = [[a, -b, tx], [b, a, ty]]
BMB_FN void sof_model(const float* f0, const float* f1, const float* t0, const float* t1, double* M) {
    const double x1 = f0[0], y1 = f0[1], x2 = f1[0], y2 = f1[1];
    const double X1 = t0[0], Y1 = t0[1], X2 = t1[0], Y2 = t1[1];
    const double d = 1. / ((x1 - x2) * (x1 - x2) + (y1 - y2) * (y1 - y2));
    const double S0 = d * ((X1 - X2) * (x1 - x2) + (Y1 - Y2) * (y1 - y2));
    const double S1 = d * ((Y1 - Y2) * (x1 - x2) - (X1 - X2) * (y1 - y2));
    const double S2 = d * ((Y1 - Y2) * (x1 * y2 - x2 * y1) - (X1 * y2 - X2 * y1) * (y1 - y2) - (X1 * x2 - X2 * x1) * (x1 - x2));
    const double S3 = d * (-(X1 - X2) * (x1 * y2 - x2 * y1) - (Y1 * x2 - Y2 * x1) * (x1 - x2) - (Y1 * y2 - Y2 * y1) * (y1 - y2));
    M[0] = M[4] = S0;
    M[1] = -S1;
    M[2] = S2;
    M[3] = S1;
    M[5] = S3;
}

// Affine2DEstimatorCallback::computeError (float32) against the squared threshold
BMB_FN int sof_inlier(const double* M, const float* f, const float* t, float thr2) {
    const float F0 = (float)M[0], F1 = (float)M[1], F2 = (float)M[2], F3 = (float)M[3], F4 = (float)M[4], F5 = (float)M[5];
    const float a = F0 * f[0] + F1 * f[1] + F2 - t[0];
    const float b = F3 * f[0] + F4 * f[1] + F5 - t[1];
    return a * a + b * b <= thr2;
}

// RANSACUpdateNumIters(confidence, outlier ratio, 2 model points, current bound)
BMB_FN int sof_update_iters(double p, double ep, int max_iters) {
    ep = ep < 0. ? 0. : (ep > 1. ? 1. : ep);
    double num = 1. - p > DBL_MIN ? 1. - p : DBL_MIN;
    double denom = 1. - (1. - ep) * (1. - ep);
    if (denom < DBL_MIN) return 0;
    num = log(num);
    denom = log(denom);
    // log() is glibc's on the host and CUDA's (within 1 ulp) on the device: the two builds could disagree only if
    // num / denom fell within an ulp of a .5 boundary of cvRound, which none of the tested sequences does
    return denom >= 0 || -num >= max_iters * (-denom) ? max_iters : BMB_D2I_RN(num / denom);
}

// The serial part of RANSACPointSetRegistrator::run: walk the hypotheses in draw order with the adaptive bound and
// keep the first strictly better one (a model needs >= 2 inliers).  Returns the index of the best hypothesis or -1.
BMB_FN int sof_ransac_pick(const int* good, int count, int* best_good) {
    int niters = SOF_RANSAC_ITERS, best = -1, max_good = 0;
    for (int it = 0; it < niters; ++it) {
        const int gc = good[it];
        if (gc > (max_good > 1 ? max_good : 1)) {
            best = it;
            max_good = gc;
            niters = sof_update_iters(0.99, (double)(count - gc) / count, niters);
        }
    }
    *best_good = max_good;
    return best;
}

// ---- Levenberg-Marquardt refine of (a, b, tx, ty) over the inliers (AffinePartial2DRefineCallback) ------------------
// mode 0: sums of J^T J (|src|^2, sum x, sum y); mode 1: S = |r|^2, v = J^T r, max |r| at parameters x.  Slot t takes the
// points t, t + SOF_RED, ... in order.
BMB_FN void sof_lm_partial(const float* src, const float* dst, int n, const double* x, int mode, int t, double* o) {
    for (int k = 0; k < 6; ++k) o[k] = 0.0;
    for (int i = t; i < n; i += SOF_RED) {
        const double Mx = src[2 * i], My = src[2 * i + 1];
        if (mode == 0) {
            o[0] += Mx * Mx + My * My;
            o[1] += Mx;
            o[2] += My;
        } else {
            const double r0 = x[0] * Mx - x[1] * My + x[2] - (double)dst[2 * i];
            const double r1 = x[1] * Mx + x[0] * My + x[3] - (double)dst[2 * i + 1];
            o[0] += r0 * r0 + r1 * r1;
            o[1] += Mx * r0 + My * r1;
            o[2] += -My * r0 + Mx * r1;
            o[3] += r0;
            o[4] += r1;
            const double m = fabs(r0) > fabs(r1) ? fabs(r0) : fabs(r1);
            o[5] = o[5] > m ? o[5] : m;
        }
    }
}

// the slot partials reduced by a fixed tree; `red` is SOF_RED * 6 doubles (shared memory on the device).  Every caller
// thread leaves with the totals in `out`.
BMB_FN void sof_lm_eval(const float* src, const float* dst, int n, const double* x, int mode, double* red, double* out) {
#if BMB_DEVICE
    const int t = threadIdx.x;
    sof_lm_partial(src, dst, n, x, mode, t, red + 6 * t);
    __syncthreads();
    for (int o = SOF_RED / 2; o > 0; o >>= 1) {
        if (t < o)
            for (int k = 0; k < 6; ++k)
                red[6 * t + k] = k == 5 ? (red[6 * t + k] > red[6 * (t + o) + k] ? red[6 * t + k] : red[6 * (t + o) + k])
                                        : red[6 * t + k] + red[6 * (t + o) + k];
        __syncthreads();
    }
    for (int k = 0; k < 6; ++k) out[k] = red[k];
    __syncthreads();
#else
    for (int t = 0; t < SOF_RED; ++t) sof_lm_partial(src, dst, n, x, mode, t, red + 6 * t);
    for (int o = SOF_RED / 2; o > 0; o >>= 1)
        for (int t = 0; t < o; ++t)
            for (int k = 0; k < 6; ++k)
                red[6 * t + k] = k == 5 ? (red[6 * t + k] > red[6 * (t + o) + k] ? red[6 * t + k] : red[6 * (t + o) + k])
                                        : red[6 * t + k] + red[6 * (t + o) + k];
    for (int k = 0; k < 6; ++k) out[k] = red[k];
#endif
}

// 4x4 linear solve, Gaussian elimination with partial pivoting (a singular system gives a zero step)
BMB_FN void sof_solve4(const double* A_, const double* b_, double* x) {
    double A[4][5];
    for (int i = 0; i < 4; ++i) {
        for (int j = 0; j < 4; ++j) A[i][j] = A_[4 * i + j];
        A[i][4] = b_[i];
    }
    for (int c = 0; c < 4; ++c) {
        int p = c;
        for (int r = c + 1; r < 4; ++r)
            if (fabs(A[r][c]) > fabs(A[p][c])) p = r;
        if (A[p][c] == 0.0) { for (int k = 0; k < 4; ++k) x[k] = 0.0; return; }
        if (p != c)
            for (int k = 0; k < 5; ++k) { const double tmp = A[c][k]; A[c][k] = A[p][k]; A[p][k] = tmp; }
        for (int r = c + 1; r < 4; ++r) {
            const double f = A[r][c] / A[c][c];
            for (int k = c; k < 5; ++k) A[r][k] -= f * A[c][k];
        }
    }
    for (int r = 3; r >= 0; --r) {
        double s = A[r][4];
        for (int k = r + 1; k < 4; ++k) s -= A[r][k] * x[k];
        x[r] = s / A[r][r];
    }
}

// cv::LMSolver (maxIters 10, epsx = epsf = FLT_EPSILON) on the inlier pairs; M is refined in place.
BMB_FN void sof_refine(const float* src, const float* dst, int n, double* M, double* red) {
    double x[4] = {M[0], M[3], M[2], M[5]}, xd[4], d[4], s[6], sd[6], v[4];
    sof_lm_eval(src, dst, n, x, 0, red, s);
    const double nn = (double)n;
    const double A[16] = {s[0], 0.0, s[1], s[2],  0.0, s[0], -s[2], s[1],  s[1], -s[2], nn, 0.0,  s[2], s[1], 0.0, nn};
    const double Dg[4] = {A[0], A[5], A[10], A[15]};
    sof_lm_eval(src, dst, n, x, 1, red, s);
    double S = s[0], rmax = s[5];
    for (int k = 0; k < 4; ++k) v[k] = s[1 + k];
    double lambda = 1.0, lc = 0.75;
    for (int iter = 0;;) {
        double Ap[16];
        for (int k = 0; k < 16; ++k) Ap[k] = A[k];
        for (int i = 0; i < 4; ++i) Ap[5 * i] += lambda * Dg[i];
        sof_solve4(Ap, v, d);
        for (int k = 0; k < 4; ++k) xd[k] = x[k] - d[k];
        sof_lm_eval(src, dst, n, xd, 1, red, sd);
        const double Sd = sd[0];
        double dS = 0.0;
        for (int i = 0; i < 4; ++i) {
            double ad = 0.0;
            for (int j = 0; j < 4; ++j) ad += A[4 * i + j] * d[j];
            dS += d[i] * (-ad + 2.0 * v[i]);
        }
        const double R = (S - Sd) / (fabs(dS) > DBL_EPSILON ? dS : 1.0);
        if (R > 0.75) {
            lambda *= 0.5;
            if (lambda < lc) lambda = 0.0;
        } else if (R < 0.25) {
            double t = 0.0;
            for (int k = 0; k < 4; ++k) t += d[k] * v[k];
            double nu = (Sd - S) / (fabs(t) > DBL_EPSILON ? t : 1.0) + 2.0;
            nu = nu < 2.0 ? 2.0 : (nu > 10.0 ? 10.0 : nu);
            if (lambda == 0.0) {
                double maxval = DBL_EPSILON;
                for (int i = 0; i < 4; ++i) {   // diagonal of A^-1
                    double e[4] = {0.0, 0.0, 0.0, 0.0}, col[4];
                    e[i] = 1.0;
                    sof_solve4(A, e, col);
                    maxval = maxval > fabs(col[i]) ? maxval : fabs(col[i]);
                }
                lambda = lc = 1.0 / maxval;
                nu *= 0.5;
            }
            lambda *= nu;
        }
        if (Sd < S) {
            S = Sd;
            rmax = sd[5];
            for (int k = 0; k < 4; ++k) { x[k] = xd[k]; v[k] = sd[1 + k]; }
        }
        ++iter;
        double dmax = 0.0;
        for (int k = 0; k < 4; ++k) dmax = dmax > fabs(d[k]) ? dmax : fabs(d[k]);
        if (!(iter < SOF_LM_ITERS && dmax >= FLT_EPSILON && rmax >= FLT_EPSILON)) break;
    }
    M[0] = M[4] = x[0];
    M[1] = -x[1];
    M[2] = x[2];
    M[3] = x[1];
    M[5] = x[3];
}

// the returned warp of SOF.apply for an accepted model: float32 linear part, translation / scale in float32
BMB_FN void sof_warp_out(const double* M, float scale, float* w6) {
    for (int k = 0; k < 6; ++k) w6[k] = (float)M[k];
    if (scale < 1.0f) { w6[2] = w6[2] / scale; w6[5] = w6[5] / scale; }
}

BMB_FN bool sof_accept(int inliers, int matches, int min_inliers, double min_ratio) {
    return matches > 0 && inliers >= min_inliers && (double)inliers / matches >= min_ratio;
}

}  // namespace bmb
