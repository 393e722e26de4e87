// Flip test-time averaging kernels.  All three are pure streaming kernels (HBM/L2-bound, a few MB per batch): one
// thread per output element, consecutive threads on consecutive addresses of the OUTPUT; the mirrored reads stay
// inside one 128-byte line per warp (reversed order), so both sides are fully coalesced.
#include "tta.cuh"
#include "tta_core.h"

namespace b2p {
namespace {

constexpr int kThreads = 256;

__global__ void __launch_bounds__(kThreads) mirror_u8hwc_kernel(const unsigned char* __restrict__ in,
                                                                unsigned char* __restrict__ out, long rows, int W) {
    // one thread per output byte; row = (image, y)
    const long total = rows * W * 3;
    for (long i = blockIdx.x * (long)kThreads + threadIdx.x; i < total; i += (long)gridDim.x * kThreads) {
        const long row = i / (W * 3);
        const int r = (int)(i - row * (W * 3));
        const int x = r / 3, ch = r - 3 * x;
        out[i] = in[row * (W * 3) + (W - 1 - x) * 3 + ch];
    }
}

__global__ void __launch_bounds__(kThreads) mirror_f32_kernel(const float* __restrict__ in, float* __restrict__ out,
                                                              long rows, int W) {
    const long total = rows * W;
    for (long i = blockIdx.x * (long)kThreads + threadIdx.x; i < total; i += (long)gridDim.x * kThreads) {
        const long row = i / W;
        const int x = (int)(i - row * W);
        out[i] = in[row * W + (W - 1 - x)];
    }
}

__global__ void __launch_bounds__(kThreads) flip_merge_kernel(const float* __restrict__ normal,
                                                              const float* __restrict__ flipped,
                                                              float* __restrict__ out, int n, int channels, int h, int w,
                                                              long sc, long sy, long sx) {
    const long per = (long)channels * h * w;
    const long total = per * n;
    const bool paf = channels == kTtaPaf;
    // enumerate outputs in memory order of the layout: NCHW (sx == 1) -> (c, y, x), HWC (sc == 1) -> (y, x, c)
    for (long i = blockIdx.x * (long)kThreads + threadIdx.x; i < total; i += (long)gridDim.x * kThreads) {
        const long img = i / per;
        const long r = i - img * per;
        int c, y, x;
        if (sx == 1) {
            c = (int)(r / ((long)h * w));
            const int q = (int)(r - (long)c * h * w);
            y = q / w; x = q - y * w;
        } else {
            y = (int)(r / ((long)w * channels));
            const int q = (int)(r - (long)y * w * channels);
            x = q / channels; c = q - x * channels;
        }
        out[img * per + c * sc + y * sy + x * sx] =
            tta_flip_merge_at(normal + img * per, flipped + img * per, paf, c, y, x, w, sc, sy, sx);
    }
}

int grid_for(long total) {
    long b = (total + kThreads - 1) / kThreads;
    const long cap = 132L * 8;          // 8 resident blocks of 256 threads per SM
    return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace

cudaError_t tta_mirror_u8hwc(const unsigned char* in, unsigned char* out, int n, int H, int W, cudaStream_t s) {
    const long rows = (long)n * H;
    mirror_u8hwc_kernel<<<grid_for(rows * W * 3), kThreads, 0, s>>>(in, out, rows, W);
    return cudaGetLastError();
}

cudaError_t tta_mirror_f32(const float* in, float* out, long planes, int H, int W, cudaStream_t s) {
    const long rows = planes * H;
    mirror_f32_kernel<<<grid_for(rows * W), kThreads, 0, s>>>(in, out, rows, W);
    return cudaGetLastError();
}

cudaError_t tta_flip_merge(const float* normal, const float* flipped, float* out, int n, int channels, int h, int w,
                           long sc, long sy, long sx, cudaStream_t s) {
    if (channels != kTtaHeat && channels != kTtaPaf) return cudaErrorInvalidValue;
    if (!(sx == 1 && sy == w && sc == (long)h * w) && !(sc == 1 && sx == channels && sy == (long)w * channels))
        return cudaErrorInvalidValue;
    flip_merge_kernel<<<grid_for((long)n * channels * h * w), kThreads, 0, s>>>(normal, flipped, out, n, channels, h, w,
                                                                                sc, sy, sx);
    return cudaGetLastError();
}

}  // namespace b2p
