// Host build of the augmentation core (csrc/aug_core.h): Pillow's two-pass BICUBIC resize of a whole image, each
// colour operation over a list of RGB triples, and a whole ColorJitter as aug.cu orders it.  AUG_CORE overrides the
// header's path, so that a test can compile a copy with a planted mistake.
#ifndef AUG_CORE
#define AUG_CORE "../../pytorch_realtime_multi-person_pose_estimation_b200/csrc/aug_core.h"
#endif
#include AUG_CORE

#include <vector>

using namespace b2p;

// Image.resize((ow, oh), BICUBIC) of an RGB image [h][w][3]: the horizontal pass over the rows the vertical pass reads
// to a uint8 intermediate, then the vertical pass.
extern "C" void core_resize(const unsigned char* src, int h, int w, int oh, int ow, unsigned char* dst) {
    int32_t k[kAugMaxTaps];
    int first, last;
    aug_taps(h, oh, 0, &first, k);
    const int cnt_last = aug_taps(h, oh, oh - 1, &last, k);
    const int rows = last + cnt_last - first;
    std::vector<unsigned char> tmp((size_t)rows * ow * 3);
    for (int r = 0; r < rows; ++r)
        for (int x = 0; x < ow; ++x) {
            int xmin;
            const int cnt = aug_taps(w, ow, x, &xmin, k);
            for (int c = 0; c < 3; ++c) {
                int32_t s = 1 << (kAugPrecisionBits - 1);
                for (int t = 0; t < cnt; ++t) s += src[((size_t)(first + r) * w + xmin + t) * 3 + c] * k[t];
                tmp[((size_t)r * ow + x) * 3 + c] = aug_clip8(s);
            }
        }
    for (int y = 0; y < oh; ++y) {
        int ymin;
        const int cnt = aug_taps(h, oh, y, &ymin, k);
        for (int x = 0; x < ow; ++x)
            for (int c = 0; c < 3; ++c) {
                int32_t s = 1 << (kAugPrecisionBits - 1);
                for (int t = 0; t < cnt; ++t) s += tmp[((size_t)(ymin + t - first) * ow + x) * 3 + c] * k[t];
                dst[((size_t)y * ow + x) * 3 + c] = aug_clip8(s);
            }
    }
}

// One operation on n RGB triples in place: op 0 brightness, 2 saturation, 3 hue (f: the hue factor) as aug_pointwise;
// 1: a contrast blend against the grey `mean`; 4: L into the first byte of each triple.
extern "C" void core_pixels(int op, unsigned char* px, long long n, double f, int mean) {
    const int dh = (int)(f * 255.0) & 255;
    for (long long i = 0; i < n; ++i) {
        unsigned char* p = px + 3 * i;
        if (op == kAugContrast) {
            for (int c = 0; c < 3; ++c) p[c] = aug_blend(mean, p[c], f);
        } else if (op == 4) {
            p[0] = (unsigned char)aug_luma(p[0], p[1], p[2]);
        } else {
            aug_pointwise(op, p, f, dh);
        }
    }
}

// ColorJitter on an RGB image of n pixels in place: the operations in `order`, factors f[4] by fn id (f[3]: hue).
extern "C" void core_jitter(unsigned char* px, long long n, const int* order, const double* f) {
    const int dh = (int)(f[3] * 255.0) & 255;
    for (int o = 0; o < 4; ++o) {
        if (order[o] == kAugContrast) {
            unsigned long long s = 0;
            for (long long i = 0; i < n; ++i) s += aug_luma(px[3 * i], px[3 * i + 1], px[3 * i + 2]);
            core_pixels(kAugContrast, px, n, f[kAugContrast], aug_contrast_mean(s, n));
        } else {
            for (long long i = 0; i < n; ++i) aug_pointwise(order[o], px + 3 * i, f[order[o]], dh);
        }
    }
}

// CocoKeypoints.get_ground_truth of one image from float64 keypoints [np][17][3] (a flipped sample's), as gt.cu's
// float64 instantiation computes it: heat [19][gh][gw], paf [38][gh][gw] with gh = input_y / 8, gw = input_x / 8.
#include "../../pytorch_realtime_multi-person_pose_estimation_b200/csrc/gt_core.h"

extern "C" void core_ground_truth_f64(const double* kp, int np, int input_y, int input_x, float* heat, float* paf) {
    const int gh = gt_grid(input_y), gw = gt_grid(input_x);
    std::vector<double> joints((size_t)np * kGtParts * 3);
    for (int p = 0; p < np; ++p) gt_person_joints(kp + (size_t)p * kGtCocoParts * 3, input_x, input_y, joints.data() + p * kGtParts * 3);
    const size_t plane = (size_t)gh * gw;
    for (int y = 0; y < gh; ++y)
        for (int x = 0; x < gw; ++x) {
            const size_t at = (size_t)y * gw + x;
            double mx = 0.0;
            for (int c = 0; c < kGtParts; ++c) {
                const double v = gt_heat_part(joints.data(), np, c, x, y);
                mx = v > mx ? v : mx;
                heat[c * plane + at] = (float)v;
            }
            heat[kGtParts * plane + at] = (float)gt_background(mx);
            for (int l = 0; l < kGtLimbs; ++l) {
                double vx, vy;
                gt_paf_limb(joints.data(), np, l, gw, gh, x, y, &vx, &vy);
                paf[2 * l * plane + at] = (float)vx;
                paf[(2 * l + 1) * plane + at] = (float)vy;
            }
        }
}
