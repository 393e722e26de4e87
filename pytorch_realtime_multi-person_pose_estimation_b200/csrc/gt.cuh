// COCO training targets and the stage losses on the device: CocoKeypoints.get_ground_truth batched (core in
// gt_core.h) and get_loss's per-stage squared errors over the net's stage maps (DESIGN.md 2.19).
#pragma once
#include <cuda_runtime.h>

#include "gt_core.h"

namespace b2p {

// One image of a target call: its persons' joints (gt_person_joints, [np][18][3]) from joint j0 on, and its grid.
struct GtImage {
    int j0, np;       // first person in the call's joint table, persons
    int gh, gw;       // int(input_y / 8), int(input_x / 8)
};

// One call, every array in device memory.  Maps [n][19 | 38][ch][cw] with the canvas grid ch x cw >= every image's.
struct GtBatch {
    const GtImage* images;
    const void* joints;       // [persons][18][3], float, or double when f64
    bool f64;
    int n, ch, cw;
    float* heat;
    float* paf;
};

// Two launches: the 19 heat channels per (image, cell), the two PAF channels per (image, limb, cell).  gt.cu
// instantiates the kernels for float32 joints, aug.cu for float64 joints (gt_launch_f64), which gt_launch runs when f64.
constexpr int kGtLaunches = 2;
constexpr int kGtThreads = 128;
cudaError_t gt_launch(const GtBatch& b, cudaStream_t s);
cudaError_t gt_launch_f64(const GtBatch& b, cudaStream_t s);

// One thread per (image, canvas cell): the 18 part channels, each over the image's persons in order, then the
// background from their maximum.  Cells outside the image's grid get +0 in every channel.
template <class T> __global__ void __launch_bounds__(kGtThreads) gt_heat_kernel(GtBatch b) {
    const long long plane = (long long)b.ch * b.cw;
    const long long t = (long long)blockIdx.x * kGtThreads + threadIdx.x;
    if (t >= plane * b.n) return;
    const int i = (int)(t / plane);
    const long long at = t - (long long)i * plane;
    const int y = (int)(at / b.cw), x = (int)(at - (long long)y * b.cw);
    const GtImage im = b.images[i];
    const bool in = y < im.gh && x < im.gw;
    const T* jo = static_cast<const T*>(b.joints) + (size_t)im.j0 * kGtParts * 3;
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
template <class T> __global__ void __launch_bounds__(kGtThreads) gt_paf_kernel(GtBatch b) {
    const long long plane = (long long)b.ch * b.cw;
    const long long t = (long long)blockIdx.x * kGtThreads + threadIdx.x;
    if (t >= plane * b.n * kGtLimbs) return;
    const long long il = t / plane;
    const int i = (int)(il / kGtLimbs), l = (int)(il - (long long)i * kGtLimbs);
    const long long at = t - il * plane;
    const int y = (int)(at / b.cw), x = (int)(at - (long long)y * b.cw);
    const GtImage im = b.images[i];
    double vx = 0.0, vy = 0.0;
    const bool in = y < im.gh && x < im.gw;
    if (in) gt_paf_limb(static_cast<const T*>(b.joints) + (size_t)im.j0 * kGtParts * 3, im.np, l, im.gw, im.gh, x, y, &vx, &vy);
    float* out = b.paf + ((size_t)i * kGtPaf + 2 * l) * plane + at;
    out[0] = in ? __double2float_rn(vx) : 0.0f;
    out[plane] = in ? __double2float_rn(vy) : 0.0f;
}

template <class T> cudaError_t gt_launch_t(const GtBatch& b, cudaStream_t s) {
    const long long cells = (long long)b.n * b.ch * b.cw;
    gt_heat_kernel<T><<<(unsigned)((cells + kGtThreads - 1) / kGtThreads), kGtThreads, 0, s>>>(b);
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    gt_paf_kernel<T><<<(unsigned)((cells * kGtLimbs + kGtThreads - 1) / kGtThreads), kGtThreads, 0, s>>>(b);
    return cudaGetLastError();
}

// The stage losses of one forward: per (image, stage map) the float64 sum of float32 (pred - target)^2 over the image's
// own (H_i / 8) x (W_i / 8) cells, and per image the extrema of the final maps.
constexpr int kGtMaxMaps = 12;
struct GtLossBatch {
    const float* maps[kGtMaxMaps];    // the forward's stage maps, canvas layout [n][C][mh][mw]
    int ch[kGtMaxMaps];               // their channels: 38 (PAF) or 19 (heat)
    int n_maps, n, mh, mw;
    const int* ext;                   // device extents {H_0, W_0, ...} of a ragged forward (input pixels), or null
    int last_paf, last_heat;          // the maps whose extrema are reported
    const float* heat;                // targets [n][19][mh][mw] and [n][38][mh][mw]
    const float* paf;
    double* sums;                     // [n][n_maps]
    float* extrema;                   // [n][4]: max_ht, min_ht (heat channels 0 .. 17), max_paf, min_paf
};
constexpr int kGtLossThreads = 256;
cudaError_t gt_stage_loss_launch(const GtLossBatch& b, cudaStream_t s);

}  // namespace b2p
