// Host build of the training-target core (csrc/gt_core.h), laid out the way the kernels of gt.cu write it: per image
// the joints of its persons, then per cell of the canvas the 19 heat channels and per (limb, cell) the two PAF channels,
// +0 outside the image's own grid.  The arguments are those of b200pose_ground_truth without the device.  GT_CORE
// overrides the header's path, so that a test can compile a copy with a planted mistake.
#ifndef GT_CORE
#define GT_CORE "../../pytorch_realtime_multi-person_pose_estimation_b200/csrc/gt_core.h"
#endif
#include GT_CORE

#include <vector>

using namespace b2p;

extern "C" double core_exp(double x) { return gt_exp(x); }

extern "C" double core_limb_norm(double dx, double dy) { return GT_SQRT(GT_FMA(dy, dy, GT_MUL(dx, dx))); }

// keypoints [sum persons][17][3], persons [n], hw [2n] (input_y, input_x per image); heat [n][19][gh][gw] and
// paf [n][38][gh][gw] with gh, gw >= every image's grid; paf64 (may be null): the PAFs before the float32 cast.
extern "C" void core_ground_truth(const float* keypoints, const int* persons, const int* hw, int n, int gh, int gw,
                                  float* heat, float* paf, double* paf64) {
    const float* kp = keypoints;
    for (int i = 0; i < n; ++i) {
        const int np = persons[i], iy = hw[2 * i], ix = hw[2 * i + 1], gy_n = gt_grid(iy), gx_n = gt_grid(ix);
        std::vector<float> joints((size_t)np * kGtParts * 3);
        for (int p = 0; p < np; ++p) gt_person_joints(kp + (size_t)p * kGtCocoParts * 3, ix, iy, joints.data() + p * kGtParts * 3);
        kp += (size_t)np * kGtCocoParts * 3;
        float* h = heat + (size_t)i * kGtHeat * gh * gw;
        float* f = paf + (size_t)i * kGtPaf * gh * gw;
        for (int y = 0; y < gh; ++y)
            for (int x = 0; x < gw; ++x) {
                const size_t at = (size_t)y * gw + x, plane = (size_t)gh * gw;
                const bool in = y < gy_n && x < gx_n;
                double mx = 0.0;
                for (int c = 0; c < kGtParts; ++c) {
                    const double v = in ? gt_heat_part(joints.data(), np, c, x, y) : 0.0;
                    mx = v > mx ? v : mx;
                    h[c * plane + at] = (float)v;
                }
                h[kGtParts * plane + at] = in ? (float)gt_background(mx) : 0.0f;
                for (int l = 0; l < kGtLimbs; ++l) {
                    double vx = 0.0, vy = 0.0;
                    if (in) gt_paf_limb(joints.data(), np, l, gx_n, gy_n, x, y, &vx, &vy);
                    f[2 * l * plane + at] = in ? (float)vx : 0.0f;
                    f[(2 * l + 1) * plane + at] = in ? (float)vy : 0.0f;
                    if (paf64) {
                        paf64[((size_t)i * kGtPaf + 2 * l) * plane + at] = vx;
                        paf64[((size_t)i * kGtPaf + 2 * l + 1) * plane + at] = vy;
                    }
                }
            }
    }
}
