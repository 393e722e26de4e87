// COCO training targets and stage losses on the device (gt.cuh, whose kernels this file instantiates for float32
// joints; arithmetic in gt_core.h, DESIGN.md 2.19).
#include "gt.cuh"

namespace b2p {
namespace {

// NaN-propagating max / min, as torch.max / torch.min
__device__ __forceinline__ float nan_max(float a, float b) { return (a > b || a != a) ? a : b; }
__device__ __forceinline__ float nan_min(float a, float b) { return (a < b || a != a) ? a : b; }

// One block per (stage map, image).  Thread t sums the squares of the image's own elements t, t + 256, ... (numbered
// over its C x h x w extent, not the canvas) in float64; the 256 partial sums are then added as a fixed tree.  So a sum
// depends on neither the canvas, nor the grid, nor the other images of the batch.
__global__ void __launch_bounds__(kGtLossThreads) gt_stage_loss_kernel(GtLossBatch b) {
    const int m = blockIdx.x, i = blockIdx.y, C = b.ch[m];
    const int h = b.ext ? b.ext[2 * i] >> 3 : b.mh, w = b.ext ? b.ext[2 * i + 1] >> 3 : b.mw;
    const long long plane = (long long)b.mh * b.mw, hw = (long long)h * w;
    const float* pred = b.maps[m] + (size_t)i * C * plane;
    const float* tgt = (C == kGtPaf ? b.paf : b.heat) + (size_t)i * C * plane;
    const bool ext_paf = m == b.last_paf, ext_heat = m == b.last_heat;
    const int ext_ch = ext_heat ? kGtParts : C;
    double s = 0.0;
    float hi = -INFINITY, lo = INFINITY;
    for (long long e = threadIdx.x; e < C * hw; e += kGtLossThreads) {
        const int c = (int)(e / hw);
        const long long r = e - c * hw;
        const int y = (int)(r / w), x = (int)(r - (long long)y * w);
        const size_t at = c * plane + (size_t)y * b.mw + x;
        const float p = pred[at];
        const float d = __fsub_rn(p, tgt[at]);
        s = __dadd_rn(s, (double)__fmul_rn(d, d));
        if (c < ext_ch) {
            hi = nan_max(hi, p);
            lo = nan_min(lo, p);
        }
    }
    __shared__ double red[kGtLossThreads];
    __shared__ float rhi[kGtLossThreads], rlo[kGtLossThreads];
    red[threadIdx.x] = s;
    rhi[threadIdx.x] = hi;
    rlo[threadIdx.x] = lo;
    __syncthreads();
    for (int k = kGtLossThreads / 2; k > 0; k >>= 1) {
        if (threadIdx.x < k) {
            red[threadIdx.x] = __dadd_rn(red[threadIdx.x], red[threadIdx.x + k]);
            rhi[threadIdx.x] = nan_max(rhi[threadIdx.x], rhi[threadIdx.x + k]);
            rlo[threadIdx.x] = nan_min(rlo[threadIdx.x], rlo[threadIdx.x + k]);
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        b.sums[(size_t)i * b.n_maps + m] = red[0];
        if (ext_heat) {
            b.extrema[4 * i] = rhi[0];
            b.extrema[4 * i + 1] = rlo[0];
        }
        if (ext_paf) {
            b.extrema[4 * i + 2] = rhi[0];
            b.extrema[4 * i + 3] = rlo[0];
        }
    }
}

}  // namespace

cudaError_t gt_launch(const GtBatch& b, cudaStream_t s) { return b.f64 ? gt_launch_f64(b, s) : gt_launch_t<float>(b, s); }

cudaError_t gt_stage_loss_launch(const GtLossBatch& b, cudaStream_t s) {
    gt_stage_loss_kernel<<<dim3(b.n_maps, b.n), kGtLossThreads, 0, s>>>(b);
    return cudaGetLastError();
}

}  // namespace b2p
