// crop_with_factor on the device, host/device shared core.
//   crop_with_factor / _factor_closest        /root/reference/lib/network/im_transform.py:113-134
// The reference scales the frame with cv2.resize(im, None, fx=s, fy=s) (OpenCV's default INTER_LINEAR on uint8) and
// zero-pads bottom/right to a multiple of `factor`.  OpenCV is a third-party dependency of the reference (not pinned
// in requirements.txt; 4.13.0 in the build container); its published 8-bit bilinear algorithm is restated here:
//   * destination size  = cvRound(src * s) per axis (round half to even), source step scale = 1 / s (double);
//   * per destination index d: f = (float)((d + 0.5) * scale - 0.5), s0 = floor(f), f -= s0; horizontally f is zeroed
//     and s0 clamped when s0 < 0 or s0 >= width - 1, vertically the two rows are clipped to [0, height - 1];
//   * 11-bit fixed-point weights a0 = cvRound((1 - f) * 2048), a1 = cvRound(f * 2048) (float arithmetic);
//   * horizontal pass in int32: S0 * a0 + S1 * a1; vertical pass
//       dst = (((b0 * (H0 >> 4)) >> 16) + ((b1 * (H1 >> 4)) >> 16) + 2) >> 2;
//   * an exact 2x reduction is silently switched to INTER_AREA by cv::resize: dst = (p00 + p01 + p10 + p11 + 2) >> 2.
// tests/test_host.py checks this core (compiled for the host) bit for bit against cv2.resize on random frames and
// against the golden vector produced by the reference's crop_with_factor.
#pragma once
#include <cmath>
#include <cstdint>

#if defined(__CUDACC__)
#define B2P_RS_HD __host__ __device__ __forceinline__
#else
#define B2P_RS_HD inline
#endif

namespace b2p {

struct LinCoef {
    int s0, s1;     // source indices of the two taps
    int w0, w1;     // 11-bit fixed-point weights
};

B2P_RS_HD int rs_round_half_even_f(float v) {
#if defined(__CUDA_ARCH__)
    return __float2int_rn(v);
#else
    return (int)lrintf(v);
#endif
}

B2P_RS_HD int rs_sat_short(int v) { return v < -32768 ? -32768 : (v > 32767 ? 32767 : v); }

// f = (float)((d + 0.5) * scale - 0.5), split into floor and fraction.  No fused multiply-add: OpenCV's scalar code
// rounds the product before the subtraction.
B2P_RS_HD void rs_src_coord(int d, double scale, int* s, float* frac) {
#if defined(__CUDA_ARCH__)
    const float f = __double2float_rn(__dadd_rn(__dmul_rn((double)d + 0.5, scale), -0.5));
    const float fl = floorf(f);
    *s = (int)fl;
    *frac = __fsub_rn(f, fl);
#else
    volatile double prod = ((double)d + 0.5) * scale;      // volatile: keep the product rounded on its own
    const float f = (float)(prod - 0.5);
    const float fl = floorf(f);
    *s = (int)fl;
    *frac = f - fl;
#endif
}

B2P_RS_HD void rs_weights(float frac, int* w0, int* w1) {
#if defined(__CUDA_ARCH__)
    *w0 = rs_sat_short(rs_round_half_even_f(__fmul_rn(__fsub_rn(1.f, frac), 2048.f)));
    *w1 = rs_sat_short(rs_round_half_even_f(__fmul_rn(frac, 2048.f)));
#else
    *w0 = rs_sat_short(rs_round_half_even_f((1.f - frac) * 2048.f));
    *w1 = rs_sat_short(rs_round_half_even_f(frac * 2048.f));
#endif
}

B2P_RS_HD LinCoef rs_coef_x(int dx, int src_w, double scale) {
    LinCoef c;
    float f;
    rs_src_coord(dx, scale, &c.s0, &f);
    if (c.s0 < 0) { f = 0.f; c.s0 = 0; }
    if (c.s0 >= src_w - 1) { f = 0.f; c.s0 = src_w - 1; }
    c.s1 = c.s0 + 1 < src_w ? c.s0 + 1 : src_w - 1;      // weight 0 whenever it is clamped
    rs_weights(f, &c.w0, &c.w1);
    return c;
}

B2P_RS_HD LinCoef rs_coef_y(int dy, int src_h, double scale) {
    LinCoef c;
    float f;
    int s;
    rs_src_coord(dy, scale, &s, &f);
    c.s0 = s < 0 ? 0 : (s > src_h - 1 ? src_h - 1 : s);
    c.s1 = s + 1 < 0 ? 0 : (s + 1 > src_h - 1 ? src_h - 1 : s + 1);
    rs_weights(f, &c.w0, &c.w1);
    return c;
}

// One channel of one destination pixel.  src: uint8 HWC, `row_stride` bytes per row, `cn` channels.
B2P_RS_HD unsigned char rs_linear_px(const unsigned char* src, long row_stride, int cn, int ch, const LinCoef& cx,
                                     const LinCoef& cy) {
    const unsigned char* r0 = src + (long)cy.s0 * row_stride;
    const unsigned char* r1 = src + (long)cy.s1 * row_stride;
    const int h0 = (int)r0[cx.s0 * cn + ch] * cx.w0 + (int)r0[cx.s1 * cn + ch] * cx.w1;
    const int h1 = (int)r1[cx.s0 * cn + ch] * cx.w0 + (int)r1[cx.s1 * cn + ch] * cx.w1;
    const int v = (((cy.w0 * (h0 >> 4)) >> 16) + ((cy.w1 * (h1 >> 4)) >> 16) + 2) >> 2;
    return (unsigned char)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// 2x2 box average (cv::resize switches an exact 2x INTER_LINEAR reduction to INTER_AREA).  Full boxes use the integer
// form (sum + 2) >> 2; a box cut by the right / bottom edge (odd source size whose half rounds up) averages the
// available pixels in float and rounds half to even, as OpenCV's border loop does.
B2P_RS_HD unsigned char rs_area2_px(const unsigned char* src, int src_h, int src_w, long row_stride, int cn, int ch, int dx,
                                    int dy) {
    const int x0 = 2 * dx, y0 = 2 * dy;
    if (x0 >= src_w || y0 >= src_h) return 0;
    const int nx = x0 + 1 < src_w ? 2 : 1, ny = y0 + 1 < src_h ? 2 : 1;
    int sum = 0;
    for (int j = 0; j < ny; ++j)
        for (int i = 0; i < nx; ++i) sum += (int)src[(long)(y0 + j) * row_stride + (x0 + i) * cn + ch];
    if (nx * ny == 4) return (unsigned char)((sum + 2) >> 2);
#if defined(__CUDA_ARCH__)
    const int v = rs_round_half_even_f(__fdiv_rn((float)sum, (float)(nx * ny)));
#else
    const int v = rs_round_half_even_f((float)sum / (float)(nx * ny));
#endif
    return (unsigned char)(v > 255 ? 255 : v);
}

// ---------------------------------------------------------------------------------------------------------------
// Bicubic resize of float32 maps (multi-scale test-time averaging): OpenCV's INTER_CUBIC formula restated -
// interpolateCubic with A = -0.75 in float, source coordinate f = (float)((d + 0.5) * (src / dst) - 0.5), taps
// floor(f) - 1 .. floor(f) + 2 with replicated borders, horizontal pass ((s0*a0 + s1*a1) + s2*a2) + s3*a3, vertical
// pass s0*b0 + (s1*b1 + (s2*b2 + s3*b3)), no fused multiply-add.  This is the arithmetic of the x8 refinement in
// peaks_kernel generalised to any size ratio.  cv2.resize itself is only matched to ~2.4e-7 in general: its SIMD
// build evaluates the last (row_length mod 4) elements of a row in a different order (and the IPP-enabled default
// of the build container differs by up to 2e-5), so the ORACLE of the multi-scale composition is this restatement.
struct CubCoef {
    int s[4];
    float w[4];
};

B2P_RS_HD float rs_mul(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fmul_rn(a, b);
#else
    return a * b;
#endif
}
B2P_RS_HD float rs_add(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fadd_rn(a, b);
#else
    return a + b;
#endif
}

B2P_RS_HD CubCoef rs_cubic_coef(int d, int src_n, double step) {
    CubCoef c;
    int s;
    float x;
    rs_src_coord(d, step, &s, &x);
    const float A = -0.75f;
    const float x1 = rs_add(x, 1.f), y = rs_add(1.f, -x);
    // ((A*(x+1) - 5A)*(x+1) + 8A)*(x+1) - 4A
    c.w[0] = rs_add(rs_mul(rs_add(rs_mul(rs_add(rs_mul(A, x1), -rs_mul(5.f, A)), x1), rs_mul(8.f, A)), x1), -rs_mul(4.f, A));
    // ((A+2)*x - (A+3))*x*x + 1
    c.w[1] = rs_add(rs_mul(rs_mul(rs_add(rs_mul(rs_add(A, 2.f), x), -rs_add(A, 3.f)), x), x), 1.f);
    c.w[2] = rs_add(rs_mul(rs_mul(rs_add(rs_mul(rs_add(A, 2.f), y), -rs_add(A, 3.f)), y), y), 1.f);
    c.w[3] = rs_add(rs_add(rs_add(1.f, -c.w[0]), -c.w[1]), -c.w[2]);
    for (int j = 0; j < 4; ++j) {
        const int t = s - 1 + j;
        c.s[j] = t < 0 ? 0 : (t > src_n - 1 ? src_n - 1 : t);
    }
    return c;
}

// source step per destination element, as cv::resize derives it from an explicit destination size (host only)
inline double rs_step(int dst_n, int src_n) { return 1.0 / ((double)dst_n / (double)src_n); }

// One destination element of one plane (row stride `sy`, element stride `sx` in floats).
B2P_RS_HD float rs_cubic_at(const float* plane, long sy, long sx, const CubCoef& cx, const CubCoef& cy) {
    float hrow[4];
    for (int j = 0; j < 4; ++j) {
        const float* r = plane + (long)cy.s[j] * sy;
        float v = rs_mul(r[cx.s[0] * sx], cx.w[0]);
        v = rs_add(v, rs_mul(r[cx.s[1] * sx], cx.w[1]));
        v = rs_add(v, rs_mul(r[cx.s[2] * sx], cx.w[2]));
        v = rs_add(v, rs_mul(r[cx.s[3] * sx], cx.w[3]));
        hrow[j] = v;
    }
    float o = rs_mul(hrow[3], cy.w[3]);
    o = rs_add(rs_mul(hrow[2], cy.w[2]), o);
    o = rs_add(rs_mul(hrow[1], cy.w[1]), o);
    o = rs_add(rs_mul(hrow[0], cy.w[0]), o);
    return o;
}

// One frame of a ragged multi-scale average (DESIGN.md 2.7): its sh x sw maps, read at the pitch of a larger source
// canvas, resized to its own dh x dw base grid.  The taps clamp at the frame's extent, not the canvas's, so every value
// is the one the frame resized alone gives.
struct RaggedResize {
    int sh, sw, dh, dw;
    double step_y, step_x;     // rs_step(dh, sh), rs_step(dw, sw)
};

// host only
inline RaggedResize ragged_resize(int sh, int sw, int dh, int dw) {
    return RaggedResize{sh, sw, dh, dw, rs_step(dh, sh), rs_step(dw, sw)};
}

// Destination element (y, x) of frame f, y < f.dh and x < f.dw; `plane` is the frame's source plane, `pitch` floats per row.
B2P_RS_HD float rs_cubic_ragged_at(const float* plane, long pitch, const RaggedResize& f, int y, int x) {
    return rs_cubic_at(plane, pitch, 1, rs_cubic_coef(x, f.sw, f.step_x), rs_cubic_coef(y, f.sh, f.step_y));
}

struct CropGeom {
    double im_scale;       // dest_size / min(h, w)                       (im_transform.py:125)
    double step;           // 1 / im_scale: source pixels per destination pixel
    int res_h, res_w;      // size after cv2.resize
    int pad_h, pad_w;      // rounded up to a multiple of `factor`        (im_transform.py:129-130)
    int area2;             // exact 2x reduction -> INTER_AREA arithmetic
};

// host only
inline CropGeom crop_geometry(int src_h, int src_w, int dest_size, int factor) {
    CropGeom g;
    const int mn = src_h < src_w ? src_h : src_w;
    g.im_scale = (double)dest_size / (double)mn;
    g.res_w = (int)lrint((double)src_w * g.im_scale);        // saturate_cast<int>(double) = round half to even
    g.res_h = (int)lrint((double)src_h * g.im_scale);
    g.step = 1.0 / g.im_scale;
    g.pad_h = (int)std::ceil((double)g.res_h / factor) * factor;
    g.pad_w = (int)std::ceil((double)g.res_w / factor) * factor;
    const int is = (int)lrint(g.step);
    g.area2 = (is == 2 && std::fabs(g.step - 2.0) < 2.220446049250313e-16) ? 1 : 0;
    return g;
}

// One byte of the padded output frame [pad_h, pad_w, 3] (zero outside the resized area).
B2P_RS_HD unsigned char crop_px(const unsigned char* src, int src_h, int src_w, int cn, const CropGeom& g, int y, int x,
                                int ch) {
    if (y >= g.res_h || x >= g.res_w) return 0;
    const long stride = (long)src_w * cn;
    if (g.area2) return rs_area2_px(src, src_h, src_w, stride, cn, ch, x, y);
    return rs_linear_px(src, stride, cn, ch, rs_coef_x(x, src_w, g.step), rs_coef_y(y, src_h, g.step));
}

}  // namespace b2p
