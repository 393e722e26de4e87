// crop_with_factor kernel: one thread per destination pixel (3 channels), consecutive threads on consecutive pixels
// of a destination row.  Streaming / gather kernel, HBM- and L2-bound: a frame is read at most once (each source row
// pair is shared by the threads of a destination row and stays in L1/L2) and written once; the per-pixel work is two
// double multiplications for the source coordinates and 12 integer MACs.
#include "resize.cuh"

namespace b2p {
namespace {

constexpr int kThreads = 256;

// The three bytes of destination pixel (y, x); zero outside the resized area (bottom / right padding).
__device__ __forceinline__ void crop_pixel(const unsigned char* src, int src_h, int src_w, const CropGeom& g, int y, int x,
                                           unsigned char* dst) {
    unsigned char v0 = 0, v1 = 0, v2 = 0;
    if (y < g.res_h && x < g.res_w) {
        const long stride = (long)src_w * 3;
        if (g.area2) {
            v0 = rs_area2_px(src, src_h, src_w, stride, 3, 0, x, y);
            v1 = rs_area2_px(src, src_h, src_w, stride, 3, 1, x, y);
            v2 = rs_area2_px(src, src_h, src_w, stride, 3, 2, x, y);
        } else {
            const LinCoef cx = rs_coef_x(x, src_w, g.step), cy = rs_coef_y(y, src_h, g.step);
            v0 = rs_linear_px(src, stride, 3, 0, cx, cy);
            v1 = rs_linear_px(src, stride, 3, 1, cx, cy);
            v2 = rs_linear_px(src, stride, 3, 2, cx, cy);
        }
    }
    dst[0] = v0;
    dst[1] = v1;
    dst[2] = v2;
}

// Frame `img` (source f.src_h x f.src_w at in + f.off) is cropped to its own f.g.pad_h x f.g.pad_w in the top-left
// corner of its Hc x Wc canvas slot; the rest of the slot is zero.  f.g.pad_h == 0: the frame is already cropped
// (f.src_h x f.src_w) and is copied as it is.
__global__ void __launch_bounds__(kThreads) crop_frames_kernel(const unsigned char* __restrict__ in,
                                                               const RaggedFrame* __restrict__ frames,
                                                               unsigned char* __restrict__ out, int Hc, int Wc) {
    const int img = blockIdx.y;
    const RaggedFrame f = frames[img];
    const long dst_px = (long)Hc * Wc;
    const unsigned char* src = in + f.off;
    unsigned char* dst = out + img * dst_px * 3;
    for (long p = blockIdx.x * (long)kThreads + threadIdx.x; p < dst_px; p += (long)gridDim.x * kThreads) {
        const int y = (int)(p / Wc), x = (int)(p - (long)y * Wc);
        if (f.g.pad_h == 0) {
            const bool in_frame = y < f.src_h && x < f.src_w;
            const unsigned char* s = src + ((long)y * f.src_w + x) * 3;
            dst[3 * p + 0] = in_frame ? s[0] : 0;
            dst[3 * p + 1] = in_frame ? s[1] : 0;
            dst[3 * p + 2] = in_frame ? s[2] : 0;
        } else if (y < f.g.pad_h && x < f.g.pad_w) {
            crop_pixel(src, f.src_h, f.src_w, f.g, y, x, dst + 3 * p);
        } else {
            dst[3 * p + 0] = dst[3 * p + 1] = dst[3 * p + 2] = 0;
        }
    }
}

// One thread per destination element of the base canvas, with frame (plane / channels)'s own extents and steps; 16
// gathers from the (L1/L2-resident, <= 34 KB) source plane.
__global__ void __launch_bounds__(kThreads) resize_cubic_accum_kernel(const float* __restrict__ src,
                                                                      float* __restrict__ dst,
                                                                      const RaggedResize* __restrict__ frames,
                                                                      long planes, int channels, int shc, int swc,
                                                                      int dhc, int dwc, int first, float divide_by) {
    const long per = (long)dhc * dwc, total = planes * per;
    for (long i = blockIdx.x * (long)kThreads + threadIdx.x; i < total; i += (long)gridDim.x * kThreads) {
        const long plane = i / per;
        const int q = (int)(i - plane * per);
        const int y = q / dwc, x = q - y * dwc;
        const RaggedResize f = frames[plane / channels];
        float v = 0.f;
        if (y < f.dh && x < f.dw) {
            v = rs_cubic_ragged_at(src + plane * (long)shc * swc, swc, f, y, x);
            if (!first) v = __fadd_rn(dst[i], v);
            if (divide_by > 0.f) v = __fdiv_rn(v, divide_by);
        }
        dst[i] = v;
    }
}

}  // namespace

cudaError_t resize_cubic_accum_launch(const float* src, float* dst, const RaggedResize* frames, int n, int channels,
                                      int src_hc, int src_wc, int dst_hc, int dst_wc, int first, float divide_by,
                                      cudaStream_t s) {
    if (n < 1 || channels < 1 || src_hc < 1 || src_wc < 1 || dst_hc < 1 || dst_wc < 1) return cudaErrorInvalidValue;
    const long planes = (long)n * channels, total = planes * dst_hc * dst_wc;
    long b = (total + kThreads - 1) / kThreads;
    if (b > 132L * 8) b = 132L * 8;
    resize_cubic_accum_kernel<<<(unsigned)b, kThreads, 0, s>>>(src, dst, frames, planes, channels, src_hc, src_wc, dst_hc,
                                                             dst_wc, first, divide_by);
    return cudaGetLastError();
}

cudaError_t crop_frames_launch(const unsigned char* in, const RaggedFrame* frames, int n, unsigned char* out, int Hc,
                               int Wc, cudaStream_t s) {
    if (n < 1 || n > 65535 || Hc < 1 || Wc < 1) return cudaErrorInvalidValue;
    const long px = (long)Hc * Wc;
    long bx = (px + kThreads - 1) / kThreads;
    const long cap = (132L * 8 + n - 1) / n;      // about one wave of 8 blocks per SM over the whole batch
    if (bx > cap) bx = cap;
    if (bx < 1) bx = 1;
    crop_frames_kernel<<<dim3((unsigned)bx, (unsigned)n), kThreads, 0, s>>>(in, frames, out, Hc, Wc);
    return cudaGetLastError();
}

}  // namespace b2p
