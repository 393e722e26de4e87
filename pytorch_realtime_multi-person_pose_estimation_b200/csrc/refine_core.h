// Peak refinement at any integer up-sampling factor, host/device shared core (postprocess.cu's refine_kernel, and the
// host test driver tests/cuda/refine_core_host.cpp).  It restates the refine branch of NMS, paf_to_pose.py:107-136:
//   * cubic       : the clipped 5x5 window around a peak, cv2.resize(patch, fx=f, fy=f, INTER_CUBIC), first arg-max;
//   * cubic+gauss : as cubic, the resized patch first smoothed by scipy.ndimage.gaussian_filter(patch, sigma=3);
//   * none        : no refinement, position (p + 0.5) f - 0.5 (compute_resized_coords), score = the map value.
// OpenCV's float cubic resize with IPP off (4.13): f = 1 is a copy; otherwise resize_core.h's coefficients with source
// step 1 / f, the horizontal pass ((s0 a0 + s1 a1) + s2 a2) + s3 a3, and the vertical pass s0 b0 + (s1 b1 + (s2 b2 + s3 b3))
// for the columns its 4-wide vector loop covers (X < W - W mod 4) but ((s0 b0 + s1 b1) + s2 b2) + s3 b3 for the scalar
// tail of each row.
// scipy.ndimage.gaussian_filter on float32 (1.18, truncate 4: radius 12, mode 'reflect'): axis 0 then axis 1; each
// pass computes, in double over the line extended by reflection (d c b a | a b c d | d c b a, repeated for lines shorter
// than the radius), t = L[i] w[12], then t += (L[i-k] + L[i+k]) w[12-k] for k = 12 .. 1, and rounds t to float32; the
// second pass reads the float32 values of the first.
#pragma once
#include "resize_core.h"

namespace b2p {

enum RefineMode { kRefineNone = 0, kRefineCubic = 1, kRefineCubicGauss = 2 };
constexpr int kRefineWin = 2;          // paf_to_pose.py:100 - a 5 x 5 window
constexpr int kMaxUpsample = 16;
constexpr int kMaxUpCoord = 16384;     // round_half_up (post_core.h) is exact up to here: h*f and w*f stay below it
constexpr int kGaussRadius = 12;

// scipy.ndimage._filters._gaussian_kernel1d(3, 0, 12), exact doubles (tests/test_refine_host.py pins the table).  A
// table, not exp(): numpy's exp is not guaranteed to round like libm's or the device's.
#define B2P_GAUSS3_TABLE                                                                                                 \
    {0x1.763a210dfb306p-15, 0x1.4fbe39149e277p-13, 0x1.0d8a5ad43c165p-11, 0x1.8345966f69518p-10, 0x1.f1e9915139406p-9,  \
     0x1.1e6bccad344bap-7,  0x1.26defcaeb0202p-6,  0x1.0fa58939b528fp-5,  0x1.bfde9c12bec92p-5,  0x1.4a614d1afd337p-4,  \
     0x1.b42a57d56c0bep-4,  0x1.01a25f86eb137p-3,  0x1.105a329f98197p-3,  0x1.01a25f86eb137p-3,  0x1.b42a57d56c0bep-4,  \
     0x1.4a614d1afd337p-4,  0x1.bfde9c12bec92p-5,  0x1.0fa58939b528fp-5,  0x1.26defcaeb0202p-6,  0x1.1e6bccad344bap-7,  \
     0x1.f1e9915139406p-9,  0x1.8345966f69518p-10, 0x1.0d8a5ad43c165p-11, 0x1.4fbe39149e277p-13, 0x1.763a210dfb306p-15}

#if defined(__CUDACC__)
static __constant__ double c_gauss3[2 * kGaussRadius + 1] = B2P_GAUSS3_TABLE;
#endif
static const double k_gauss3_host[2 * kGaussRadius + 1] = B2P_GAUSS3_TABLE;
#if defined(__CUDA_ARCH__)
#define B2P_GAUSS_W c_gauss3
#else
#define B2P_GAUSS_W k_gauss3_host
#endif

B2P_RS_HD double rf_dmul(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    volatile double r = a * b;
    return r;
#endif
}
B2P_RS_HD double rf_dadd(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dadd_rn(a, b);
#else
    volatile double r = a + b;
    return r;
#endif
}
B2P_RS_HD float rf_to_float(double v) {
#if defined(__CUDA_ARCH__)
    return __double2float_rn(v);
#else
    return (float)v;
#endif
}

// index i (-radius .. n - 1 + radius) of a line of n elements extended by reflection with period 2n
B2P_RS_HD int rf_reflect(int i, int n) {
    int m = i % (2 * n);
    if (m < 0) m += 2 * n;
    return m >= n ? 2 * n - 1 - m : m;
}

// One output of a Gaussian pass before its rounding to float32: element i of the line line[0], line[step], ..
// line[(n-1) step].
B2P_RS_HD double rf_gauss_sum(const float* line, int step, int n, int i) {
    const double* w = B2P_GAUSS_W;
    double t = rf_dmul((double)line[i * step], w[kGaussRadius]);
    for (int k = kGaussRadius; k >= 1; --k) {
        const double s = rf_dadd((double)line[rf_reflect(i - k, n) * step], (double)line[rf_reflect(i + k, n) * step]);
        t = rf_dadd(t, rf_dmul(s, w[kGaussRadius - k]));
    }
    return t;
}
B2P_RS_HD float rf_gauss_at(const float* line, int step, int n, int i) { return rf_to_float(rf_gauss_sum(line, step, n, i)); }

// Element (Y, X) of cv2.resize(patch, fx=f, fy=f, INTER_CUBIC) of a ph x pw patch (row stride `sy` floats).
B2P_RS_HD float rf_up_at(const float* patch, long sy, int ph, int pw, int f, int Y, int X) {
    if (f == 1) return patch[Y * sy + X];
    const double step = 1.0 / (double)f;
    const CubCoef cx = rs_cubic_coef(X, pw, step), cy = rs_cubic_coef(Y, ph, step);
    const int W = pw * f;
    if (X < W - W % 4) return rs_cubic_at(patch, sy, 1, cx, cy);
    float hrow[4];
    for (int j = 0; j < 4; ++j) {
        const float* r = patch + (long)cy.s[j] * sy;
        float v = rs_mul(r[cx.s[0]], cx.w[0]);
        v = rs_add(v, rs_mul(r[cx.s[1]], cx.w[1]));
        v = rs_add(v, rs_mul(r[cx.s[2]], cx.w[2]));
        v = rs_add(v, rs_mul(r[cx.s[3]], cx.w[3]));
        hrow[j] = v;
    }
    float o = rs_mul(hrow[0], cy.w[0]);
    o = rs_add(o, rs_mul(hrow[1], cy.w[1]));
    o = rs_add(o, rs_mul(hrow[2], cy.w[2]));
    o = rs_add(o, rs_mul(hrow[3], cy.w[3]));
    return o;
}

// The clipped window of a low-resolution peak (x, y) on an h x w map.
struct RefineWin {
    int x0, y0, pw, ph;
};
B2P_RS_HD RefineWin rf_window(int x, int y, int h, int w) {
    const int x0 = x - kRefineWin < 0 ? 0 : x - kRefineWin, y0 = y - kRefineWin < 0 ? 0 : y - kRefineWin;
    const int x1 = x + kRefineWin > w - 1 ? w - 1 : x + kRefineWin, y1 = y + kRefineWin > h - 1 ? h - 1 : y + kRefineWin;
    return RefineWin{x0, y0, x1 - x0 + 1, y1 - y0 + 1};
}

// Up-sampled position of an unrefined peak p: (p + 0.5) f - 0.5 as the int the reference's pafprocess stores (its
// float-to-int truncation: f p + (f - 1) / 2 rounded down).  NMS itself reports the exact (p + 0.5) f - 0.5.
B2P_RS_HD int rf_unrefined_coord(int p, int f) { return f * p + (f - 1) / 2; }

// The arg-max rule of every mode: the larger value, the smaller row-major index among equals (np.argmax's first).
B2P_RS_HD bool rf_better(float v, int i, float bv, int bi) { return v > bv || (v == bv && i < bi); }

#if !defined(__CUDA_ARCH__)
// Host reference of one refinement: win = the ph x pw window (row stride pw), scratch >= 2 (5 f)^2 floats.  Returns the
// row-major arg-max index into the (ph f) x (pw f) patch and its value.
inline int rf_refine_host(const float* win, int ph, int pw, int f, bool gauss, float* scratch, float* score) {
    const int H = ph * f, W = pw * f;
    float* up = scratch;
    float* tmp = scratch + H * W;
    for (int Y = 0; Y < H; ++Y)
        for (int X = 0; X < W; ++X) up[Y * W + X] = rf_up_at(win, pw, ph, pw, f, Y, X);
    int bi = 0;
    float bv = up[0];
    if (gauss) {
        for (int Y = 0; Y < H; ++Y)
            for (int X = 0; X < W; ++X) tmp[Y * W + X] = rf_gauss_at(up + X, W, H, Y);       // axis 0
        for (int Y = 0; Y < H; ++Y)
            for (int X = 0; X < W; ++X) up[Y * W + X] = rf_gauss_at(tmp + Y * W, 1, W, X);   // axis 1
        bv = up[0];
    }
    for (int i = 1; i < H * W; ++i)
        if (rf_better(up[i], i, bv, bi)) { bv = up[i]; bi = i; }
    *score = bv;
    return bi;
}
#endif

}  // namespace b2p
