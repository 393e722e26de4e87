// COCO training targets, host/device shared core: what CocoKeypoints.get_ground_truth (lib/datasets/datasets.py:259-308,
// with add_neck :227-257 and remove_illegal_joint :216-225) builds with putGaussianMaps (lib/datasets/heatmap.py:20-36)
// and putVecMaps (lib/datasets/paf.py:18-68), restated (DESIGN.md 2.19):
//  * gt_person_joints: per person the 17 COCO keypoints (float32, as transforms.Normalize leaves them, or float64 after
//    transforms.HFlip) gain the neck (r_shoulder + l_shoulder) / 2 in that dtype, visibility 2 if both are 2 else their product, np.round (half to even) on
//    x, y and v; reordered to the 18-part order; a joint at x >= input_x, x < 0, y >= input_y or y < 0 becomes (-1, -1, 0);
//  * heat maps (gt_heat_term): per part, persons in annotation order, += exp(-d2 / 2 / sigma / sigma) where the exponent
//    is <= 4.6052, clamped to 1 after each person; background max(1 - max over the 18 parts, 0);
//  * PAFs (gt_limb_setup, gt_paf_step): per limb and person with both joints visible, the unit vector of B - A in grid
//    units (|.| as OpenBLAS's ddot forms it: sqrt(fma(dy, dy, dx * dx))), the limb's box rounded half to even, the
//    width test |ba_x u_y - ba_y u_x| < 1, and at every cell of the map acc = (acc * count + vec) / max(count', 1).
// Every float64 operation rounds as numpy's does: no contraction (the GT_* operations), an explicit fma only where
// OpenBLAS fuses, and gt_exp, this file's own exp, so that the host build (tests/cuda/gt_core_host.cpp) and the kernels
// of gt.cu give the same bits.  The results are cast to float32 at the end.
#pragma once

#if defined(__CUDACC__)
#define B2P_GT_HD __host__ __device__ __forceinline__
#else
#define B2P_GT_HD inline
#endif
#include <cmath>
#include <cstdint>
#include <cstring>

#if defined(__CUDA_ARCH__)
#define GT_ADD(a, b) __dadd_rn(a, b)
#define GT_SUB(a, b) __dsub_rn(a, b)
#define GT_MUL(a, b) __dmul_rn(a, b)
#define GT_DIV(a, b) __ddiv_rn(a, b)
#define GT_FMA(a, b, c) __fma_rn(a, b, c)
#define GT_SQRT(a) __dsqrt_rn(a)
#define GT_RINT(a) rint(a)
#else
#define GT_ADD(a, b) ((a) + (b))     // the host build compiles with -ffp-contract=off
#define GT_SUB(a, b) ((a) - (b))
#define GT_MUL(a, b) ((a) * (b))
#define GT_DIV(a, b) ((a) / (b))
#define GT_FMA(a, b, c) std::fma(a, b, c)
#define GT_SQRT(a) std::sqrt(a)
#define GT_RINT(a) std::nearbyint(a)      // the default rounding mode: half to even
#endif

namespace b2p {

constexpr int kGtCocoParts = 17;
constexpr int kGtParts = 18;                  // HEATMAP_COUNT
constexpr int kGtHeat = kGtParts + 1;         // the parts, then the background
constexpr int kGtLimbs = 19;                  // len(kp_connections(get_keypoints()))
constexpr int kGtPaf = 2 * kGtLimbs;          // x, y per limb
constexpr int kGtStride = 8;                  // get_ground_truth's stride
constexpr double kGtSigma = 7.0;              // putGaussianMaps' sigma as get_ground_truth passes it
constexpr double kGtExpMax = 4.6052;          // the heat-map exponent cut (log(100))
constexpr int kGtMaxImages = 1024;            // images of one call
constexpr int kGtMaxPersons = 256;            // persons of one image
constexpr int kGtMaxSize = 8192;              // input_y, input_x of one image (at least kGtStride)

// our_order of add_neck: 18-part index -> index into the 17 COCO keypoints with the neck appended as 17
B2P_GT_HD int gt_source_part(int p) {
    const int order[kGtParts] = {0, 17, 6, 8, 10, 5, 7, 9, 12, 14, 16, 11, 13, 15, 2, 1, 4, 3};
    return order[p];
}

// kp_connections(get_keypoints()): limb l joins parts gt_limb_a(l) -> gt_limb_b(l).  The tables are string literals
// (octal escapes), which the device reads from global memory instead of building a local array per thread.
B2P_GT_HD int gt_limb_a(int l) { return "\001\010\011\001\013\014\001\002\003\002\001\005\006\005\001\000\000\016\017"[l]; }
B2P_GT_HD int gt_limb_b(int l) { return "\010\011\012\013\014\015\002\003\004\016\005\006\007\017\000\016\017\020\021"[l]; }

// int(size / stride)
B2P_GT_HD int gt_grid(int size) { return size / kGtStride; }

// exp(x) for x <= 0 down to -708, within an ulp of the correctly rounded value: x = k ln2 + r with |r| <= ln2 / 2
// (Cody-Waite, ln2 split in two), e^r - 1 as r + r^2 (1/2! + r (1/3! + ... + r / 13!)) by Horner with explicit fma
// (the truncation error r^14 / 14! stays below 5e-18), 1 + that, times 2^k built from its bits.  The same operations
// on host and device, so the same bits on both.
B2P_GT_HD double gt_exp(double x) {
    const double inv_ln2 = 1.4426950408889634;
    const double ln2_hi = 6.93147180369123816490e-01, ln2_lo = 1.90821492927058770002e-10;
    const double k = GT_RINT(GT_MUL(x, inv_ln2));
    double r = GT_FMA(-k, ln2_hi, x);
    r = GT_FMA(-k, ln2_lo, r);
    const double c[12] = {1.0 / 2, 1.0 / 6, 1.0 / 24, 1.0 / 120, 1.0 / 720, 1.0 / 5040, 1.0 / 40320, 1.0 / 362880,
                          1.0 / 3628800, 1.0 / 39916800, 1.0 / 479001600, 1.0 / 6227020800.0};
    double q = c[11];
    for (int i = 10; i >= 0; --i) q = GT_FMA(q, r, c[i]);
    const double em1 = GT_FMA(GT_MUL(r, r), q, r);
    const double e = GT_ADD(1.0, em1);
    const int64_t bits = (int64_t)((long long)k + 1023) << 52;
    double two_k;
    memcpy(&two_k, &bits, 8);
    return GT_MUL(e, two_k);
}

// np.round (half to even) in the keypoints' own precision
B2P_GT_HD float gt_round(float v) { return rintf(v); }
B2P_GT_HD double gt_round(double v) { return GT_RINT(v); }

// add_neck + our_order + remove_illegal_joint of one person: kp [17][3] -> j [18][3], in the keypoints' dtype T: float32
// as transforms.Normalize leaves them, float64 after HFlip (horizontal_swap_coco returns float64, and every later step
// keeps it).  input_x / input_y: the image's width and height.
template <class T> B2P_GT_HD void gt_person_joints(const T* kp, int input_x, int input_y, T* j) {
    const T* rs = kp + 3 * 6;
    const T* ls = kp + 3 * 5;
    T neck[3];
    for (int t = 0; t < 2; ++t) neck[t] = (rs[t] + ls[t]) / (T)2;
    neck[2] = (rs[2] == (T)2 && ls[2] == (T)2) ? (T)2 : rs[2] * ls[2];
    for (int t = 0; t < 3; ++t) neck[t] = gt_round(neck[t]);
    const T fx = (T)input_x, fy = (T)input_y;
    for (int p = 0; p < kGtParts; ++p) {
        const int s = gt_source_part(p);
        const T* src = s == kGtCocoParts ? neck : kp + 3 * s;
        const T x = src[0], y = src[1];
        if (x >= fx || x < 0.0f || y >= fy || y < 0.0f) {
            j[3 * p] = (T)-1;
            j[3 * p + 1] = (T)-1;
            j[3 * p + 2] = (T)0;
        } else {
            j[3 * p] = x;
            j[3 * p + 1] = y;
            j[3 * p + 2] = src[2];
        }
    }
}

// putGaussianMaps' term of a joint at (cx, cy) for grid cell (gx, gy): exp(-exponent) where exponent <= 4.6052, else 0.
template <class T> B2P_GT_HD double gt_heat_term(T cx, T cy, int gx, int gy) {
    const double start = kGtStride / 2.0 - 0.5;
    const double dx = GT_SUB(GT_ADD((double)(gx * kGtStride), start), (double)cx);
    const double dy = GT_SUB(GT_ADD((double)(gy * kGtStride), start), (double)cy);
    const double d2 = GT_ADD(GT_MUL(dx, dx), GT_MUL(dy, dy));
    const double ex = GT_DIV(GT_DIV(GT_DIV(d2, 2.0), kGtSigma), kGtSigma);
    return ex <= kGtExpMax ? gt_exp(-ex) : 0.0;
}

// Heat-map channel p (0 .. 17) at cell (gx, gy) over np persons' joints [np][18][3]: accumulated in order, clamped to
// 1 after each person.
template <class T> B2P_GT_HD double gt_heat_part(const T* joints, int np, int p, int gx, int gy) {
    double acc = 0.0;
    for (int i = 0; i < np; ++i) {
        const T* jo = joints + (i * kGtParts + p) * 3;
        if (jo[2] > 0.5f) {
            acc = GT_ADD(acc, gt_heat_term(jo[0], jo[1], gx, gy));
            if (acc > 1.0) acc = 1.0;
        }
    }
    return acc;
}

// the background channel from the maximum of the 18 parts
B2P_GT_HD double gt_background(double part_max) {
    const double b = GT_SUB(1.0, part_max);
    return b > 0.0 ? b : 0.0;
}

// One person's limb in grid units: A, the unit vector A -> B and the box [x0, x1) x [y0, y1) of cells it may cover.
struct GtLimb {
    double ax, ay, ux, uy;
    int x0, x1, y0, y1;
};

// putVecMaps' set-up for joints ja, jb ([3] each): false when either is not visible (v <= 0.5) or the limb has zero
// length, which putVecMaps skips without touching the maps.
template <class T> B2P_GT_HD bool gt_limb_setup(const T* ja, const T* jb, int grid_x, int grid_y, GtLimb* L) {
    if (!(ja[2] > 0.5f && jb[2] > 0.5f)) return false;
    const double ax = GT_DIV((double)ja[0], (double)kGtStride), ay = GT_DIV((double)ja[1], (double)kGtStride);
    const double bx = GT_DIV((double)jb[0], (double)kGtStride), by = GT_DIV((double)jb[1], (double)kGtStride);
    const double dx = GT_SUB(bx, ax), dy = GT_SUB(by, ay);
    const double norm = GT_SQRT(GT_FMA(dy, dy, GT_MUL(dx, dx)));
    if (norm == 0.0) return false;
    L->ax = ax;
    L->ay = ay;
    L->ux = GT_DIV(dx, norm);
    L->uy = GT_DIV(dy, norm);
    const int x0 = (int)GT_RINT(GT_SUB(ax < bx ? ax : bx, 1.0)), x1 = (int)GT_RINT(GT_ADD(bx > ax ? bx : ax, 1.0));
    const int y0 = (int)GT_RINT(GT_SUB(ay < by ? ay : by, 1.0)), y1 = (int)GT_RINT(GT_ADD(by > ay ? by : ay, 1.0));
    L->x0 = x0 > 0 ? x0 : 0;
    L->x1 = x1 < grid_x ? x1 : grid_x;
    L->y0 = y0 > 0 ? y0 : 0;
    L->y1 = y1 < grid_y ? y1 : grid_y;
    return true;
}

// One putVecMaps call at cell (gx, gy): vec is mask * u inside the box and acc * 0.0 (+-0) outside it; then
// acc = acc * count + vec, count += (|vec_x| > 0 or |vec_y| > 0), acc /= max(count, 1) - at every cell, covered or not.
B2P_GT_HD void gt_paf_step(const GtLimb& L, int gx, int gy, double& vx, double& vy, int& count) {
    double nx, ny;
    if (gx >= L.x0 && gx < L.x1 && gy >= L.y0 && gy < L.y1) {
        const double bax = GT_SUB((double)gx, L.ax), bay = GT_SUB((double)gy, L.ay);
        const double w = fabs(GT_SUB(GT_MUL(bax, L.uy), GT_MUL(bay, L.ux)));
        const double m = w < 1.0 ? 1.0 : 0.0;
        nx = GT_MUL(m, L.ux);
        ny = GT_MUL(m, L.uy);
    } else {
        nx = GT_MUL(vx, 0.0);
        ny = GT_MUL(vy, 0.0);
    }
    const double c = (double)count;
    vx = GT_ADD(GT_MUL(vx, c), nx);
    vy = GT_ADD(GT_MUL(vy, c), ny);
    if (fabs(nx) > 0.0 || fabs(ny) > 0.0) ++count;
    const double d = count == 0 ? 1.0 : (double)count;
    vx = GT_DIV(vx, d);
    vy = GT_DIV(vy, d);
}

// PAF channels 2l, 2l + 1 of limb l at cell (gx, gy) over np persons' joints [np][18][3], persons in order.
template <class T>
B2P_GT_HD void gt_paf_limb(const T* joints, int np, int l, int grid_x, int grid_y, int gx, int gy, double* vx, double* vy) {
    double x = 0.0, y = 0.0;
    int count = 0;
    const int a = gt_limb_a(l), b = gt_limb_b(l);
    for (int i = 0; i < np; ++i) {
        GtLimb L;
        if (gt_limb_setup(joints + (i * kGtParts + a) * 3, joints + (i * kGtParts + b) * 3, grid_x, grid_y, &L))
            gt_paf_step(L, gx, gy, x, y, count);
    }
    *vx = x;
    *vy = y;
}

}  // namespace b2p
