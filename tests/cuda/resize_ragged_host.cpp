// Host build of the ragged bicubic resize (csrc/resize_core.h: ragged_resize, rs_cubic_ragged_at), walked over a whole
// destination canvas exactly as resize_cubic_accum_kernel walks it (one plane, no running sum).
#include "../../pytorch_realtime_multi-person_pose_estimation_b200/csrc/resize_core.h"

using namespace b2p;

// src [n, shc, swc] float32 (one plane per frame, canvas pitch); hw[4i .. 4i+3] = frame i's sh, sw, dh, dw;
// out [n, dhc, dwc]: frame i resized from its own sh x sw to its own dh x dw, +0 elsewhere.
extern "C" int core_resize_cubic_ragged(const float* src, int n, int shc, int swc, const int* hw, float* out, int dhc,
                                        int dwc) {
    for (int i = 0; i < n; ++i) {
        const RaggedResize f = ragged_resize(hw[4 * i], hw[4 * i + 1], hw[4 * i + 2], hw[4 * i + 3]);
        const float* plane = src + (long)i * shc * swc;
        for (int y = 0; y < dhc; ++y)
            for (int x = 0; x < dwc; ++x)
                out[((long)i * dhc + y) * dwc + x] = (y < f.dh && x < f.dw) ? rs_cubic_ragged_at(plane, swc, f, y, x) : 0.f;
    }
    return 0;
}
