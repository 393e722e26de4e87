// Training-time augmentation on the device (aug.cuh; arithmetic in aug_core.h, DESIGN.md 2.20).  Every kernel runs on a
// grid of (pixels, image): the launch count of a call does not depend on its batch.
#include "aug.cuh"
#include "gt.cuh"
#include "preprocess_core.h"

namespace b2p {
namespace {

constexpr int kThreads = 256;

// Pillow's horizontal pass over the rows the vertical pass reads, for the cropped columns only: one thread per
// intermediate pixel.  The flip is the source index.
__global__ void __launch_bounds__(kThreads) aug_hpass_kernel(AugBatch b) {
    const AugImage im = b.images[blockIdx.y];
    const int t = blockIdx.x * kThreads + threadIdx.x;
    if (t >= im.rows * im.cw) return;
    const int r = t / im.cw, c = t - r * im.cw;
    int xmin;
    int32_t k[kAugMaxTaps];
    const int cnt = aug_taps(im.w, im.rw, im.x0 + c, &xmin, k);
    const unsigned char* row = b.src + im.src + (size_t)(im.r0 + r) * im.w * 3;
    int32_t s0 = 1 << (kAugPrecisionBits - 1), s1 = s0, s2 = s0;
    for (int x = 0; x < cnt; ++x) {
        const int sx = im.flip ? im.w - 1 - (xmin + x) : xmin + x;
        const unsigned char* p = row + 3 * sx;
        s0 += p[2] * k[x];
        s1 += p[1] * k[x];
        s2 += p[0] * k[x];
    }
    unsigned char* o = b.tmp + im.tmp + 3 * (size_t)t;
    o[0] = aug_clip8(s0);
    o[1] = aug_clip8(s1);
    o[2] = aug_clip8(s2);
}

// The vertical pass inside the pasted window, CenterPad's fill outside it, then ColorJitter's operations up to
// contrast; the image's sum of L for contrast's mean.
__global__ void __launch_bounds__(kThreads) aug_vpass_kernel(AugBatch b) {
    const int i = blockIdx.y, E = b.edge;
    const AugImage im = b.images[i];
    const int t = blockIdx.x * kThreads + threadIdx.x;
    unsigned lum = 0;
    if (t < E * E) {
        const int py = t / E, px = t - py * E;
        unsigned char v[3] = {kAugPad[0], kAugPad[1], kAugPad[2]};
        if (py >= im.top && py < im.top + im.ch && px >= im.left && px < im.left + im.cw) {
            int ymin;
            int32_t k[kAugMaxTaps];
            const int cnt = aug_taps(im.h, im.rh, im.y0 + py - im.top, &ymin, k);
            const unsigned char* col = b.tmp + im.tmp + 3 * (size_t)(px - im.left);
            int32_t s[3] = {1 << (kAugPrecisionBits - 1), 1 << (kAugPrecisionBits - 1), 1 << (kAugPrecisionBits - 1)};
            for (int y = 0; y < cnt; ++y) {
                const unsigned char* p = col + (size_t)(ymin + y - im.r0) * im.cw * 3;
                for (int c = 0; c < 3; ++c) s[c] += p[c] * k[y];
            }
            for (int c = 0; c < 3; ++c) v[c] = aug_clip8(s[c]);
        }
        for (int o = 0; o < 4 && im.order[o] != kAugContrast; ++o) aug_pointwise(im.order[o], v, im.f[im.order[o]], im.dh);
        unsigned char* d = b.px + ((size_t)i * E * E + t) * 3;
        for (int c = 0; c < 3; ++c) d[c] = v[c];
        lum = aug_luma(v[0], v[1], v[2]);
    }
    for (int o = 16; o > 0; o >>= 1) lum += __shfl_down_sync(0xffffffffu, lum, o);
    __shared__ unsigned warp_sum[kThreads / 32];
    if ((threadIdx.x & 31) == 0) warp_sum[threadIdx.x >> 5] = lum;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long s = 0;
        for (int w = 0; w < kThreads / 32; ++w) s += warp_sum[w];
        atomicAdd(b.lsum + i, s);      // integer sums: the order does not matter
    }
}

// Contrast against the image's mean grey, then the operations after it; stored as BGR.
__global__ void __launch_bounds__(kThreads) aug_contrast_kernel(AugBatch b) {
    const int i = blockIdx.y, E = b.edge;
    const int t = blockIdx.x * kThreads + threadIdx.x;
    if (t >= E * E) return;
    const AugImage im = b.images[i];
    const int mean = aug_contrast_mean(b.lsum[i], (long long)E * E);
    unsigned char* d = b.px + ((size_t)i * E * E + t) * 3;
    unsigned char v[3] = {d[0], d[1], d[2]};
    int o = 0;
    while (im.order[o] != kAugContrast) ++o;
    for (int c = 0; c < 3; ++c) v[c] = aug_blend(mean, v[c], im.f[kAugContrast]);
    for (++o; o < 4; ++o) aug_pointwise(im.order[o], v, im.f[im.order[o]], im.dh);
    d[0] = v[2];
    d[1] = v[1];
    d[2] = v[0];
}

// RandomGrayscale, ToTensor + Normalize (vgg: pre_value), mask_valid_area.
__global__ void __launch_bounds__(kThreads) aug_finish_kernel(AugBatch b) {
    const int i = blockIdx.y, E = b.edge;
    const int t = blockIdx.x * kThreads + threadIdx.x;
    if (t >= E * E) return;
    const AugImage im = b.images[i];
    const int py = t / E, px = t - py * E;
    const size_t at = (size_t)i * E * E + t;
    const unsigned char* d = b.px + at * 3;
    unsigned char v[3] = {d[0], d[1], d[2]};       // BGR
    if (im.gray) {
        const unsigned char l = (unsigned char)aug_luma(v[2], v[1], v[0]);
        v[0] = v[1] = v[2] = l;
    }
    if (b.out_u8)
        for (int c = 0; c < 3; ++c) b.out_u8[at * 3 + c] = v[c];
    const bool masked = px < im.mx0 || px >= im.mx1 || py < im.my0 || py >= im.my1;
    float* o = b.out + (size_t)i * 3 * E * E + t;
    for (int c = 0; c < 3; ++c) o[(size_t)c * E * E] = masked ? 0.0f : pre_value(kPreVgg, v[pre_src_channel(kPreVgg, c)], c);
}

}  // namespace

cudaError_t aug_jitter_launch(const AugBatch& b, cudaStream_t s) {
    const unsigned px_blocks = (unsigned)(((long long)b.edge * b.edge + kThreads - 1) / kThreads);
    aug_hpass_kernel<<<dim3((unsigned)((b.max_tmp_px + kThreads - 1) / kThreads), b.n), kThreads, 0, s>>>(b);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    aug_vpass_kernel<<<dim3(px_blocks, b.n), kThreads, 0, s>>>(b);
    if ((e = cudaGetLastError()) != cudaSuccess) return e;
    aug_contrast_kernel<<<dim3(px_blocks, b.n), kThreads, 0, s>>>(b);
    return cudaGetLastError();
}

// The targets of flipped samples, whose keypoints are float64 (gt.cuh's kernels for double joints)
cudaError_t gt_launch_f64(const GtBatch& b, cudaStream_t s) { return gt_launch_t<double>(b, s); }

cudaError_t aug_finish_launch(const AugBatch& b, cudaStream_t s) {
    const unsigned px_blocks = (unsigned)(((long long)b.edge * b.edge + kThreads - 1) / kThreads);
    aug_finish_kernel<<<dim3(px_blocks, b.n), kThreads, 0, s>>>(b);
    return cudaGetLastError();
}

}  // namespace b2p
