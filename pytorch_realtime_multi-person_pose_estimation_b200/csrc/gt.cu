// COCO training targets and stage losses on the device (gt.cuh; arithmetic in gt_core.h, DESIGN.md 2.19).
#include "gt.cuh"

namespace b2p {
namespace {

constexpr int kThreads = 128;

// One thread per (image, canvas cell): the 18 part channels, each over the image's persons in order, then the
// background from their maximum.  Cells outside the image's grid get +0 in every channel.
__global__ void __launch_bounds__(kThreads) gt_heat_kernel(GtBatch b) {
    const long long plane = (long long)b.ch * b.cw;
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (t >= plane * b.n) return;
    const int i = (int)(t / plane);
    const long long at = t - (long long)i * plane;
    const int y = (int)(at / b.cw), x = (int)(at - (long long)y * b.cw);
    const GtImage im = b.images[i];
    const bool in = y < im.gh && x < im.gw;
    const float* jo = b.joints + (size_t)im.j0 * kGtParts * 3;
    float* out = b.heat + (size_t)i * kGtHeat * plane + at;
    double mx = 0.0;
    for (int c = 0; c < kGtParts; ++c) {
        const double v = in ? gt_heat_part(jo, im.np, c, x, y) : 0.0;
        mx = v > mx ? v : mx;
        out[c * plane] = __double2float_rn(v);
    }
    out[kGtParts * plane] = in ? __double2float_rn(gt_background(mx)) : 0.0f;
}

// One thread per (image, limb, canvas cell): the limb's x and y channels over the image's persons in order.
__global__ void __launch_bounds__(kThreads) gt_paf_kernel(GtBatch b) {
    const long long plane = (long long)b.ch * b.cw;
    const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
    if (t >= plane * b.n * kGtLimbs) return;
    const long long il = t / plane;
    const int i = (int)(il / kGtLimbs), l = (int)(il - (long long)i * kGtLimbs);
    const long long at = t - il * plane;
    const int y = (int)(at / b.cw), x = (int)(at - (long long)y * b.cw);
    const GtImage im = b.images[i];
    double vx = 0.0, vy = 0.0;
    const bool in = y < im.gh && x < im.gw;
    if (in) gt_paf_limb(b.joints + (size_t)im.j0 * kGtParts * 3, im.np, l, im.gw, im.gh, x, y, &vx, &vy);
    float* out = b.paf + ((size_t)i * kGtPaf + 2 * l) * plane + at;
    out[0] = in ? __double2float_rn(vx) : 0.0f;
    out[plane] = in ? __double2float_rn(vy) : 0.0f;
}

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

cudaError_t gt_launch(const GtBatch& b, cudaStream_t s) {
    const long long cells = (long long)b.n * b.ch * b.cw;
    gt_heat_kernel<<<(unsigned)((cells + kThreads - 1) / kThreads), kThreads, 0, s>>>(b);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    gt_paf_kernel<<<(unsigned)((cells * kGtLimbs + kThreads - 1) / kThreads), kThreads, 0, s>>>(b);
    return cudaGetLastError();
}

cudaError_t gt_stage_loss_launch(const GtLossBatch& b, cudaStream_t s) {
    gt_stage_loss_kernel<<<dim3(b.n_maps, b.n), kGtLossThreads, 0, s>>>(b);
    return cudaGetLastError();
}

}  // namespace b2p
