// COCO keypoint evaluation kernels (DESIGN.md 2.16), four launches per call whatever the image count:
//  1. OKS: one CTA per (category, image) unit ranks its detections by score in shared memory (coco_rank), keeps the
//     first 20, writes their score, area and category, and computes the unit's 20 x G OKS block in float64.
//  2. matching: one warp per (unit, area range) runs the ten thresholds; each lane holds the ignore, crowd and matched
//     flags of 32 gts as bit masks, and each detection takes the best candidate of two warp arg-max reductions
//     (coco_better: the non-ignored gts first, then the ignored ones).  The warp also counts the unit's non-ignored gts.
//  3. global order: one thread per kept detection counts the detections of its category ahead of it in
//     argsort(-score, kind='mergesort') over the category's concatenation (ascending image id, then rank in the
//     image): a stable order without a sort, and the same count however the threads are scheduled.
//  4. accumulation: one CTA per (category, area range, threshold) walks the category's detections in that order: a
//     block scan of the packed tp / fp counts, rc and pr per position, and the precision envelope at the 101 recall
//     thresholds as a shared-memory max per threshold segment (coco_rec_count), folded right to left at the end.
#include <cub/block/block_scan.cuh>

#include "coco_eval.cuh"

namespace b2p {
namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kAccPer = 4;      // positions per thread per step of the accumulation walk

__global__ void __launch_bounds__(kThreads) coco_oks_kernel(CocoBatch b) {
    __shared__ double score[kCocoMaxUnitDets];
    __shared__ int kept[kCocoMaxDets];
    if (blockIdx.x >= b.n_units) return;     // a call without units still launches one CTA
    const CocoUnit u = b.units[blockIdx.x];
    for (int i = threadIdx.x; i < u.nd; i += kThreads) score[i] = b.dt_score[u.d0 + i];
    __syncthreads();
    for (int i = threadIdx.x; i < u.nd; i += kThreads) {
        const int r = coco_rank(score, u.nd, i);
        if (r < kCocoMaxDets) kept[r] = i;
    }
    __syncthreads();
    if (threadIdx.x < u.nk) {
        const int k = u.k0 + threadIdx.x, i = kept[threadIdx.x];
        b.k_score[k] = score[i];
        b.k_area[k] = coco_dt_area(b.dt_kpt + (size_t)kCocoKpt * (u.d0 + i));
        b.k_cat[k] = u.cat;
    }
    const int pairs = u.nk * u.ng;
    for (int p = threadIdx.x; p < pairs; p += kThreads) {
        const int r = p / u.ng, g = u.g0 + p % u.ng;
        b.oks[u.o0 + p] = coco_oks(b.gt_kpt + (size_t)kCocoKpt * g, b.gt_box + 5 * (size_t)g,
                                   b.dt_kpt + (size_t)kCocoKpt * (u.d0 + kept[r]));
    }
}

__device__ __forceinline__ void warp_best(double& oks, int& g) {
    for (int off = 16; off > 0; off >>= 1) {
        const double o = __shfl_xor_sync(0xffffffffu, oks, off);
        const int h = __shfl_xor_sync(0xffffffffu, g, off);
        if (coco_better(o, h, oks, g)) oks = o, g = h;
    }
}

__global__ void __launch_bounds__(kThreads) coco_match_kernel(CocoBatch b) {
    const int w = blockIdx.x * kWarps + threadIdx.x / 32, lane = threadIdx.x % 32;
    if (w >= b.n_units * kCocoAreas) return;
    const CocoUnit u = b.units[w / kCocoAreas];
    const int a = w % kCocoAreas;
    unsigned ig = 0, crowd = 0, valid = 0;     // bit j: gt lane + 32 j of the unit
    for (int j = 0; lane + 32 * j < u.ng; ++j) {
        const int g = u.g0 + lane + 32 * j;
        const unsigned f = b.gt_flag[g];
        valid |= 1u << j;
        if ((f & 2) || coco_area_out(b.gt_box[5 * (size_t)g + 4], a)) ig |= 1u << j;
        if (f & 1) crowd |= 1u << j;
    }
    int n = __popc(valid & ~ig);
    for (int off = 16; off > 0; off >>= 1) n += __shfl_xor_sync(0xffffffffu, n, off);
    if (lane == 0 && n) atomicAdd(b.npig + u.cat * kCocoAreas + a, n);
    for (int t = 0; t < kCocoIouThrs; ++t) {
        const double floor = coco_iou_floor(b.thr[t]);
        unsigned matched = 0;
        unsigned char* st = b.state + ((size_t)a * kCocoIouThrs + t) * b.kept + u.k0;
        for (int r = 0; r < u.nk; ++r) {
            double on = -1.0, oi = -1.0;
            int gn = -1, gi = -1;
            for (int j = 0; lane + 32 * j < u.ng; ++j) {
                if ((matched >> j & 1) && !(crowd >> j & 1)) continue;
                const int g = lane + 32 * j;
                const double o = b.oks[u.o0 + (long long)r * u.ng + g];
                if (o < floor) continue;
                if (ig >> j & 1) {
                    if (coco_better(o, g, oi, gi)) oi = o, gi = g;
                } else if (coco_better(o, g, on, gn)) {
                    on = o, gn = g;
                }
            }
            warp_best(on, gn);
            warp_best(oi, gi);
            const int m = gn >= 0 ? gn : gi;
            if (m >= 0 && lane == m % 32) matched |= 1u << (m / 32);
            if (lane == 0) st[r] = (unsigned char)coco_dt_state(m >= 0, gn < 0, b.k_area[u.k0 + r], a);
        }
    }
}

__global__ void __launch_bounds__(kThreads) coco_order_kernel(CocoBatch b) {
    __shared__ double tile[kThreads];
    if (b.kept == 0) return;                 // a call without detections still launches one CTA
    const int i = blockIdx.x * kThreads + threadIdx.x;
    const int last = min(b.kept, (int)(blockIdx.x + 1) * kThreads) - 1;
    const int lo = b.cat_k0[b.k_cat[blockIdx.x * kThreads]], hi = b.cat_k0[b.k_cat[last] + 1];
    const bool mine = i < b.kept;
    const int c = mine ? b.k_cat[i] : 0;
    const int jb = b.cat_k0[c], je = b.cat_k0[c + 1];
    const double s = mine ? b.k_score[i] : 0.0;
    int rank = 0;
    for (int base = lo; base < hi; base += kThreads) {
        if (base + threadIdx.x < hi) tile[threadIdx.x] = b.k_score[base + threadIdx.x];
        __syncthreads();
        if (mine) {
            const int from = max(jb, base), to = min(je, min(hi, base + kThreads));
            for (int j = from; j < to; ++j) {
                const double o = tile[j - base];
                rank += o > s || (o == s && j < i);
            }
        }
        __syncthreads();
    }
    if (mine) b.order[jb + rank] = i;
}

__global__ void __launch_bounds__(kThreads) coco_accumulate_kernel(CocoBatch b) {
    using Scan = cub::BlockScan<unsigned long long, kThreads>;
    __shared__ typename Scan::TempStorage scan;
    __shared__ double thr[kCocoRecThrs];
    __shared__ unsigned long long seg[kCocoRecThrs];     // per threshold segment: the largest pr's bits (pr >= 0)
    const int t = blockIdx.x % kCocoIouThrs, a = blockIdx.x / kCocoIouThrs % kCocoAreas;
    const int c = blockIdx.x / (kCocoIouThrs * kCocoAreas);
    const int npig = b.npig[c * kCocoAreas + a];
    double* prec = b.precision + ((size_t)t * kCocoRecThrs * b.n_cats + c) * kCocoAreas + a;
    const size_t pstride = (size_t)b.n_cats * kCocoAreas;
    double* rec = b.recall + ((size_t)t * b.n_cats + c) * kCocoAreas + a;
    if (npig == 0) {      // no non-ignored gt: precision and recall stay -1
        for (int r = threadIdx.x; r < kCocoRecThrs; r += kThreads) prec[r * pstride] = -1.0;
        if (threadIdx.x == 0) *rec = -1.0;
        return;
    }
    for (int r = threadIdx.x; r < kCocoRecThrs; r += kThreads) {
        thr[r] = b.thr[kCocoIouThrs + r];
        seg[r] = 0;
    }
    const int k0 = b.cat_k0[c], n = b.cat_k0[c + 1] - k0;
    const unsigned char* st = b.state + ((size_t)a * kCocoIouThrs + t) * b.kept;
    if (threadIdx.x == 0 && n == 0) *rec = 0.0;
    __syncthreads();
    unsigned long long carry = 0;      // tp in the low 32 bits, fp in the high 32
    for (int base = 0; base < n; base += kThreads * kAccPer) {
        unsigned long long v[kAccPer];
        for (int q = 0; q < kAccPer; ++q) {
            const int i = base + threadIdx.x * kAccPer + q;
            const int s = i < n ? st[b.order[k0 + i]] : kCocoIgnored;
            v[q] = s == kCocoTp ? 1ull : (s == kCocoFp ? 1ull << 32 : 0ull);
        }
        unsigned long long total;
        Scan(scan).InclusiveSum(v, v, total);
        for (int q = 0; q < kAccPer; ++q) {
            const int i = base + threadIdx.x * kAccPer + q;
            if (i >= n) break;
            const unsigned long long cum = carry + v[q];
            double rc, pr;
            coco_pr((long long)(cum & 0xffffffffull), (long long)(cum >> 32), npig, &rc, &pr);
            const int served = coco_rec_count(thr, rc);
            if (served > 0) atomicMax(&seg[served - 1], (unsigned long long)__double_as_longlong(pr));
            if (i == n - 1) *rec = rc;
        }
        carry += total;
        __syncthreads();      // the scan's storage is reused
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long run = 0;
        for (int r = kCocoRecThrs - 1; r >= 0; --r) {
            run = max(run, seg[r]);
            prec[r * pstride] = __longlong_as_double((long long)run);
        }
    }
}

}  // namespace

cudaError_t coco_eval_launch(const CocoBatch& b, cudaStream_t s) {
    coco_oks_kernel<<<max(b.n_units, 1), kThreads, 0, s>>>(b);
    if (cudaError_t e = cudaGetLastError()) return e;
    coco_match_kernel<<<max((b.n_units * kCocoAreas + kWarps - 1) / kWarps, 1), kThreads, 0, s>>>(b);
    if (cudaError_t e = cudaGetLastError()) return e;
    coco_order_kernel<<<max((b.kept + kThreads - 1) / kThreads, 1), kThreads, 0, s>>>(b);
    if (cudaError_t e = cudaGetLastError()) return e;
    coco_accumulate_kernel<<<b.n_cats * kCocoAreas * kCocoIouThrs, kThreads, 0, s>>>(b);
    return cudaGetLastError();
}

}  // namespace b2p
