// Person drawing kernels.  plan: one thread per primitive (35 per person row) solves its pixel set once (draw_plan).
// raster: one CTA per (frame, 32 x 32 pixel tile); it walks its frame's primitives in draw order, skips those whose box
// misses the tile, and each thread keeps, in registers, the index of the last primitive that covers each of its four
// pixels.  No two threads share a pixel, so no barrier is needed per primitive and CTAs need no order between them:
// the colour written is that of the last covering primitive, as if cv2 had drawn them one after the other.
#include "draw.cuh"

namespace b2p {
namespace {

constexpr int kPlanThreads = 128;
constexpr int kTile = 32, kRasterThreads = 256, kRowsPerThread = kTile * kTile / kRasterThreads;

__global__ void __launch_bounds__(kPlanThreads) draw_plan_kernel(const DrawImage* __restrict__ images,
                                                                 const float* __restrict__ rows,
                                                                 const int* __restrict__ person_img, int prims,
                                                                 DrawPrim* __restrict__ out) {
    const int t = blockIdx.x * kPlanThreads + threadIdx.x;
    if (t >= prims) return;
    const int person = t / kDrawPrimsPerPerson;
    const DrawImage im = images[person_img[person]];
    DrawPrim p;
    draw_plan(rows + (long)person * kDrawRowFloats, im.h, im.w, im.net_h, im.net_w, t % kDrawPrimsPerPerson, p);
    out[t] = p;
}

__global__ void __launch_bounds__(kRasterThreads) draw_raster_kernel(const DrawImage* __restrict__ images,
                                                                     const DrawPrim* __restrict__ prims,
                                                                     unsigned char* __restrict__ frames) {
    const DrawImage im = images[blockIdx.y];
    const int tiles_x = (im.w + kTile - 1) / kTile;
    if ((int)blockIdx.x >= tiles_x * ((im.h + kTile - 1) / kTile)) return;
    const int tx0 = (blockIdx.x % tiles_x) * kTile, ty0 = (blockIdx.x / tiles_x) * kTile;
    const int x = tx0 + (threadIdx.x % kTile), y0 = ty0 + (threadIdx.x / kTile);
    const int tx1 = min(tx0 + kTile, im.w) - 1, ty1 = min(ty0 + kTile, im.h) - 1;
    int last[kRowsPerThread];
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j) last[j] = -1;
    const int k0 = im.person0 * kDrawPrimsPerPerson, k1 = k0 + im.persons * kDrawPrimsPerPerson;
    for (int k = k0; k < k1; ++k) {
        const DrawPrim& p = prims[k];
        if (p.kind == 0 || p.x1 < tx0 || p.x0 > tx1 || p.y1 < ty0 || p.y0 > ty1) continue;
#pragma unroll
        for (int j = 0; j < kRowsPerThread; ++j)
            if (draw_covers(p, x, y0 + j * (kRasterThreads / kTile))) last[j] = k;
    }
    if (x >= im.w) return;
#pragma unroll
    for (int j = 0; j < kRowsPerThread; ++j) {
        const int y = y0 + j * (kRasterThreads / kTile);
        if (last[j] < 0 || y >= im.h) continue;
        unsigned char* q = frames + im.off + 3 * ((long long)y * im.w + x);
        const unsigned char* c = prims[last[j]].bgr;
        q[0] = c[0];
        q[1] = c[1];
        q[2] = c[2];
    }
}

}  // namespace

cudaError_t draw_launch(const DrawImage* images, int n, const float* rows, const int* person_img, int persons,
                        DrawPrim* prims, int max_h, int max_w, unsigned char* frames, cudaStream_t s) {
    if (n < 1 || n > 65535 || max_h < 1 || max_w < 1 || persons < 0) return cudaErrorInvalidValue;
    if (persons == 0) return cudaSuccess;
    const int np = persons * kDrawPrimsPerPerson;
    draw_plan_kernel<<<(np + kPlanThreads - 1) / kPlanThreads, kPlanThreads, 0, s>>>(images, rows, person_img, np, prims);
    const long tiles = (long)((max_h + kTile - 1) / kTile) * ((max_w + kTile - 1) / kTile);
    if (tiles > 0x7fffffffL) return cudaErrorInvalidValue;
    draw_raster_kernel<<<dim3((unsigned)tiles, (unsigned)n), kRasterThreads, 0, s>>>(images, prims, frames);
    return cudaGetLastError();
}

}  // namespace b2p
