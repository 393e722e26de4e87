// Host build of the peak refinement core (csrc/refine_core.h) for tests/test_refine_host.py.  REFINE_CORE overrides the
// header's path, so that a test can compile a copy with a planted mistake (csrc is on the include path).
#ifndef REFINE_CORE
#define REFINE_CORE "refine_core.h"
#endif
#include REFINE_CORE

using namespace b2p;

// cv2.resize(win, fx=f, fy=f, INTER_CUBIC): out [(ph f) x (pw f)]
extern "C" void core_up(const float* win, int ph, int pw, int f, float* out) {
    for (int Y = 0; Y < ph * f; ++Y)
        for (int X = 0; X < pw * f; ++X) out[Y * pw * f + X] = rf_up_at(win, pw, ph, pw, f, Y, X);
}

// the whole refinement of one window: returns the row-major arg-max index, its value in *score, and the patch the
// arg-max was taken on (resized, and smoothed if gauss) in patch [(ph f) x (pw f)]
extern "C" int core_refine(const float* win, int ph, int pw, int f, int gauss, float* score, float* patch) {
    static float scratch[2 * 80 * 80];
    const int i = rf_refine_host(win, ph, pw, f, gauss != 0, scratch, score);
    for (int k = 0; k < ph * f * pw * f; ++k) patch[k] = scratch[k];
    return i;
}

// one Gaussian pass along the rows of an h x w array, before the rounding to float32: out [h x w] doubles
extern "C" void core_gauss_rows(const float* in, int h, int w, double* out) {
    for (int y = 0; y < h; ++y)
        for (int x = 0; x < w; ++x) out[y * w + x] = rf_gauss_sum(in + y * w, 1, w, x);
}

// the Gaussian weight table
extern "C" void core_gauss_weights(double* out) {
    for (int i = 0; i < 2 * kGaussRadius + 1; ++i) out[i] = k_gauss3_host[i];
}
