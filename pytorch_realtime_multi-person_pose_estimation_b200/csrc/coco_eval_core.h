// COCO keypoint evaluation, host/device shared core: what pycocotools 2.0's COCOeval(cocoGt, cocoDt, 'keypoints')
// computes with default Params (maxDets 20, the three keypoint area ranges, the 17 kpt_oks_sigmas), restated
// (DESIGN.md 2.16):
//  * computeOks: detections of a (category, image) unit ranked by argsort(-score, kind='mergesort') and cut to 20;
//    e = (dx^2 + dy^2) / (2 sigma)^2 / (area + eps) / 2 over the gt's visible parts (dx, dy: detection minus gt), or,
//    for a gt with no visible part, over all 17 with dx, dy the distance outside the gt box enlarged to
//    [x - w, x + 2w] x [y - h, y + 2h]; oks = sum(exp(-e)) / n;
//  * evaluateImg: per area range and threshold, each detection in score order takes the gt of highest OKS >= the
//    threshold among the non-ignored gts that are unmatched or crowd, ties to the last; only when there is none, the
//    same among the ignored gts (coco_better is that scan's order);
//  * accumulate: the precision / recall walk over a category's detections in global score order (coco_pr,
//    coco_rec_segment).
// Every float64 operation rounds as numpy's does: no contraction (the COCO_* operations), numpy's summation order
// (coco_sum); only exp may differ from numpy's, by an ulp or so.  The work is split the way the kernels of
// coco_eval.cu run it; tests/cuda/coco_eval_core_host.cpp runs the same steps serially.
#pragma once

#if defined(__CUDACC__)
#define B2P_CE_HD __host__ __device__ __forceinline__
#else
#define B2P_CE_HD inline
#include <cmath>
#endif

#if defined(__CUDA_ARCH__)
#define COCO_ADD(a, b) __dadd_rn(a, b)
#define COCO_SUB(a, b) __dsub_rn(a, b)
#define COCO_MUL(a, b) __dmul_rn(a, b)
#define COCO_DIV(a, b) __ddiv_rn(a, b)
#define COCO_EXP(a) exp(a)
#else
#define COCO_ADD(a, b) ((a) + (b))     // the host build compiles with -ffp-contract=off
#define COCO_SUB(a, b) ((a) - (b))
#define COCO_MUL(a, b) ((a) * (b))
#define COCO_DIV(a, b) ((a) / (b))
#define COCO_EXP(a) std::exp(a)
#endif

namespace b2p {

constexpr int kCocoParts = 17;
constexpr int kCocoKpt = 3 * kCocoParts;      // x, y, v per part
constexpr int kCocoMaxDets = 20;              // Params.maxDets = [20]
constexpr int kCocoIouThrs = 10;              // np.linspace(.5, .95, 10)
constexpr int kCocoRecThrs = 101;             // np.linspace(0, 1, 101)
constexpr int kCocoAreas = 3;                 // all, medium, large
constexpr int kCocoMaxUnitDets = 1024;        // detections of one (category, image) unit, before the cut to 20
constexpr int kCocoMaxUnitGts = 1024;         // gts of one unit (32 per lane of the matching warp)
constexpr int kCocoMaxKept = 1 << 18;         // detections after the cut, all units (the ranking is quadratic per category)
constexpr int kCocoMaxTotal = 1 << 24;        // gts, and detections before the cut, of one call
constexpr int kCocoMaxCats = 1024;
// detection state per (area range, threshold) after matching
enum { kCocoIgnored = 0, kCocoTp = 1, kCocoFp = 2 };

// Params.areaRng for keypoints: [0, 1e5^2], [32^2, 96^2], [96^2, 1e5^2]; both bounds inclusive
B2P_CE_HD double coco_area_lo(int a) { return a == 0 ? 0.0 : (a == 1 ? 1024.0 : 9216.0); }
B2P_CE_HD double coco_area_hi(int a) { return a == 1 ? 9216.0 : 1e10; }
B2P_CE_HD bool coco_area_out(double area, int a) { return area < coco_area_lo(a) || area > coco_area_hi(a); }

// vars = (sigmas * 2) ** 2 with sigmas = np.array([.26, ...]) / 10.0
B2P_CE_HD double coco_kpt_var(int k) {
    const double s100[kCocoParts] = {.26, .25, .25, .35, .35, .79, .79, .72, .72, .62, .62, 1.07, 1.07, .87, .87, .89, .89};
    const double s2 = COCO_MUL(COCO_DIV(s100[k], 10.0), 2.0);
    return COCO_MUL(s2, s2);
}

// np.sum of n <= 17 float64 values as numpy (2.x) adds them: below 8 values one running sum from 0; from 8, eight
// running sums over the blocks of 8, combined as ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)), then the values
// past the last whole block one by one (pairwise_sum below its 128-value block size).  Found by experiment: this
// order agrees with np.sum bit for bit on 20 000 arrays of 1 .. 17 values chosen to expose the order, plain
// left-to-right summation does not from 8 values on (DESIGN.md 2.16).
B2P_CE_HD double coco_sum(const double* v, int n) {
    if (n < 8) {
        double r = 0.0;
        for (int i = 0; i < n; ++i) r = COCO_ADD(r, v[i]);
        return r;
    }
    double r[8];
    for (int j = 0; j < 8; ++j) r[j] = v[j];
    int i = 8;
    for (; i < n - n % 8; i += 8)
        for (int j = 0; j < 8; ++j) r[j] = COCO_ADD(r[j], v[i + j]);
    double s = COCO_ADD(COCO_ADD(COCO_ADD(r[0], r[1]), COCO_ADD(r[2], r[3])), COCO_ADD(COCO_ADD(r[4], r[5]), COCO_ADD(r[6], r[7])));
    for (; i < n; ++i) s = COCO_ADD(s, v[i]);
    return s;
}

// computeOks for one (detection, gt) pair.  g: the gt's 51 keypoint values, box: its bbox (x, y, w, h) and area.
B2P_CE_HD double coco_oks(const double* g, const double* box, const double* d) {
    const double eps = 2.220446049250313e-16;     // np.spacing(1)
    const double area = COCO_ADD(box[4], eps);
    int k1 = 0;
    for (int k = 0; k < kCocoParts; ++k) k1 += g[3 * k + 2] > 0;
    const double x0 = COCO_SUB(box[0], box[2]), x1 = COCO_ADD(box[0], COCO_MUL(box[2], 2.0));
    const double y0 = COCO_SUB(box[1], box[3]), y1 = COCO_ADD(box[1], COCO_MUL(box[3], 2.0));
    double v[kCocoParts];
    int n = 0;
    for (int k = 0; k < kCocoParts; ++k) {
        const double xd = d[3 * k], yd = d[3 * k + 1];
        double dx, dy;
        if (k1 > 0) {
            if (!(g[3 * k + 2] > 0)) continue;
            dx = COCO_SUB(xd, g[3 * k]);
            dy = COCO_SUB(yd, g[3 * k + 1]);
        } else {
            const double ax = COCO_SUB(x0, xd), bx = COCO_SUB(xd, x1), ay = COCO_SUB(y0, yd), by = COCO_SUB(yd, y1);
            dx = COCO_ADD(ax > 0.0 ? ax : 0.0, bx > 0.0 ? bx : 0.0);
            dy = COCO_ADD(ay > 0.0 ? ay : 0.0, by > 0.0 ? by : 0.0);
        }
        const double e = COCO_DIV(COCO_DIV(COCO_DIV(COCO_ADD(COCO_MUL(dx, dx), COCO_MUL(dy, dy)), coco_kpt_var(k)), area), 2.0);
        v[n++] = COCO_EXP(-e);
    }
    return COCO_DIV(coco_sum(v, n), (double)n);
}

// loadRes: the detection's box spans all 17 x and y values, undetected (0, 0) parts included; area = w * h
B2P_CE_HD double coco_dt_area(const double* d) {
    double x0 = d[0], x1 = d[0], y0 = d[1], y1 = d[1];
    for (int k = 1; k < kCocoParts; ++k) {
        const double x = d[3 * k], y = d[3 * k + 1];
        x0 = x < x0 ? x : x0;
        x1 = x > x1 ? x : x1;
        y0 = y < y0 ? y : y0;
        y1 = y > y1 ? y : y1;
    }
    return COCO_MUL(COCO_SUB(x1, x0), COCO_SUB(y1, y0));
}

// Position of entry i in argsort(-s, kind='mergesort'): the entries of higher score, and those of equal score before
// it (-0.0 and +0.0 compare equal, as numpy orders them).
B2P_CE_HD int coco_rank(const double* s, int n, int i) {
    int r = 0;
    for (int j = 0; j < n; ++j) r += s[j] > s[i] || (s[j] == s[i] && j < i);
    return r;
}

// evaluateImg's scan over the gts for one detection, as an order on candidates (oks, gt index): a gt is a candidate
// when it is unmatched or crowd and oks >= min(t, 1 - 1e-10); the scan keeps the highest oks, ties to the later gt.
// Within the non-ignored gts and within the ignored ones (each group keeps its order in the file) the best candidate
// is the maximum in this order; an ignored gt is taken only when no non-ignored gt is a candidate.  -1: no candidate.
B2P_CE_HD bool coco_better(double oks_a, int a, double oks_b, int b) {
    return b < 0 || (a >= 0 && (oks_a > oks_b || (oks_a == oks_b && a > b)));
}
B2P_CE_HD double coco_iou_floor(double t) { return t < 1.0 - 1e-10 ? t : 1.0 - 1e-10; }

// The detection's state after matching: a matched one inherits the gt's ignore flag; an unmatched one outside the
// area range is ignored.
B2P_CE_HD int coco_dt_state(bool matched, bool gt_ignored, double dt_area, int a) {
    if (matched) return gt_ignored ? kCocoIgnored : kCocoTp;
    return coco_area_out(dt_area, a) ? kCocoIgnored : kCocoFp;
}

// accumulate at one position of the global order: rc = tp / npig, pr = tp / (tp + fp + eps), the counts exact in float64
B2P_CE_HD void coco_pr(long long tp, long long fp, int npig, double* rc, double* pr) {
    const double t = (double)tp, f = (double)fp;
    *rc = COCO_DIV(t, (double)npig);
    *pr = COCO_DIV(t, COCO_ADD(COCO_ADD(f, t), 2.220446049250313e-16));
}

// searchsorted(rc, recThrs, side='left') places recall threshold r at the first position whose rc >= recThrs[r]; rc
// never decreases, so a position i serves the thresholds r with recThrs[r] <= rc_i, and the precision envelope at
// threshold r (the largest pr at or after its position) is the largest pr over the positions that serve r.  Returns
// the count of thresholds <= rc (thr ascending): position i's pr counts for the thresholds 0 .. count - 1.
B2P_CE_HD int coco_rec_count(const double* thr, double rc) {
    int lo = 0, hi = kCocoRecThrs;
    while (lo < hi) {
        const int mid = (lo + hi) / 2;
        if (thr[mid] <= rc) lo = mid + 1;
        else hi = mid;
    }
    return lo;
}

}  // namespace b2p
