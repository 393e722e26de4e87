// COCO keypoint evaluation on the device: pycocotools' COCOeval(..., 'keypoints').evaluate() and .accumulate() with
// default Params (core in coco_eval_core.h).
#pragma once
#include <cuda_runtime.h>

#include "coco_eval_core.h"

namespace b2p {

// One (category, image) unit with a gt or a detection.  Units are ordered by category, and within a category by
// ascending image id; the unit's gts and detections keep their order in the gt file and in the result list.
struct CocoUnit {
    int cat;            // index into the call's sorted category ids
    int g0, ng;         // its gts
    int d0, nd;         // its detections before the cut
    int k0, nk;         // its kept detections (nk = min(nd, 20)) in the call-wide kept order
    long long o0;       // its OKS block [nk][ng]
};

// One evaluation call, every array in device memory.
struct CocoBatch {
    const CocoUnit* units;
    int n_units, n_cats;
    const int* cat_k0;            // [n_cats + 1]: each category's first kept detection
    const double* gt_kpt;         // [G][51]
    const double* gt_box;         // [G][5]: bbox x, y, w, h, then the annotation's area
    const unsigned char* gt_flag; // [G]: 1 crowd, 2 ignore (iscrowd, or num_keypoints == 0)
    const double* dt_kpt;         // [D][51]
    const double* dt_score;       // [D]
    const double* thr;            // iouThrs [10], then recThrs [101]
    int kept;                     // kept detections, all units
    double* k_score;              // [kept]: score, area and category of each kept detection
    double* k_area;
    int* k_cat;
    double* oks;                  // the units' OKS blocks
    unsigned char* state;         // [3][10][kept]: kCocoTp / kCocoFp / kCocoIgnored
    int* order;                   // [kept]: per category, its kept detections in global score order
    int* npig;                    // [n_cats][3]: non-ignored gts (zeroed before the launch)
    double* precision;            // [10][101][n_cats][3]
    double* recall;               // [10][n_cats][3]
};

// Four launches: OKS per unit, matching per (unit, area range), global order per category, accumulation per
// (category, area range, threshold).
constexpr int kCocoLaunches = 4;
cudaError_t coco_eval_launch(const CocoBatch& b, cudaStream_t s);

}  // namespace b2p
