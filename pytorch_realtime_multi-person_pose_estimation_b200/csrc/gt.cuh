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
    const float* joints;      // [persons][18][3]
    int n, ch, cw;
    float* heat;
    float* paf;
};

// Two launches: the 19 heat channels per (image, cell), the two PAF channels per (image, limb, cell).
constexpr int kGtLaunches = 2;
cudaError_t gt_launch(const GtBatch& b, cudaStream_t s);

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
