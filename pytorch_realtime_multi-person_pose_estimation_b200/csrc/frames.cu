// Video-frame conversion kernel: one thread per output pixel (3 bytes), consecutive threads on consecutive pixels of
// an output row.  Streaming kernel, HBM-bound: an NV12 / I420 1920x1080 frame is 3.1 MB read and 6.2 MB written.  A
// rotated frame reads a stored column per output row; the stored frame stays in L2 (50 MB) while it is walked.
#include "frames.cuh"

namespace b2p {
namespace {

constexpr int kThreads = 256;

__global__ void __launch_bounds__(kThreads) convert_frames_kernel(const FrameSrc* __restrict__ frames, int fmt, int rot,
                                                                  unsigned char* __restrict__ out) {
    const FrameSrc f = frames[blockIdx.y];
    int oh, ow;
    fr_rotated_size(f.h, f.w, rot, &oh, &ow);
    const long px = (long)oh * ow;
    unsigned char* dst = out + f.off;
    for (long p = blockIdx.x * (long)kThreads + threadIdx.x; p < px; p += (long)gridDim.x * kThreads) {
        const int y = (int)(p / ow), x = (int)(p - (long)y * ow);
        unsigned char bgr[3];
        frame_px(f, fmt, rot, y, x, bgr);
        dst[3 * p + 0] = bgr[0];
        dst[3 * p + 1] = bgr[1];
        dst[3 * p + 2] = bgr[2];
    }
}

}  // namespace

cudaError_t convert_frames_launch(const FrameSrc* frames, int n, int fmt, int rot, long max_px, unsigned char* out,
                                  cudaStream_t s) {
    if (n < 1 || n > 65535 || max_px < 1) return cudaErrorInvalidValue;
    long bx = (max_px + kThreads - 1) / kThreads;
    const long cap = (132L * 8 + n - 1) / n;      // about one wave of 8 blocks per SM over the whole batch
    if (bx > cap) bx = cap;
    if (bx < 1) bx = 1;
    convert_frames_kernel<<<dim3((unsigned)bx, (unsigned)n), kThreads, 0, s>>>(frames, fmt, rot, out);
    return cudaGetLastError();
}

}  // namespace b2p
