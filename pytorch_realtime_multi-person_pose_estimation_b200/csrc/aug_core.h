// Training-time image augmentation, host/device shared core: the Pillow 12 / torchvision 0.26 arithmetic of the
// reference's loader (train/train_VGG19.py:124-130 preprocess, lib/datasets/transforms.py:53-65 image_transform_train),
// restated (DESIGN.md 2.20):
//  * aug_taps: Image.resize(..., BICUBIC)'s window of one output index (Resample.c precompute_coeffs with a = -0.5 and
//    support 2 * max(in / out, 1), weights normalised in double, then 22-bit fixed point rounded away from zero);
//    aug_clip8: one pass's 8-bit clip.  Pillow runs the horizontal pass to a uint8 image, then the
//    vertical one;
//  * aug_blend: Image.blend(degenerate, image, f) of one byte, which ImageEnhance.Brightness (degenerate 0), Contrast
//    (the mean grey) and Color (the pixel's own L) use;
//  * aug_luma: convert('L'); aug_hue: convert('HSV'), the hue byte shifted by np.int32(f * 255).astype(uint8) with
//    wraparound, convert('RGB') (Convert.c rgb2hsv_row / hsv2rgb).
// Every double and float operation rounds as the x86-64 build of Pillow rounds it: no contraction (the AUG_*
// operations on the device, -ffp-contract=off on the host), so that tests/cuda/aug_core_host.cpp and aug.cu give the
// same bits.
#pragma once

#if defined(__CUDACC__)
#define B2P_AUG_HD __host__ __device__ __forceinline__
#else
#define B2P_AUG_HD inline
#endif
#include <cmath>
#include <cstdint>

#if defined(__CUDA_ARCH__)
#define AUG_DADD(a, b) __dadd_rn(a, b)
#define AUG_DSUB(a, b) __dsub_rn(a, b)
#define AUG_DMUL(a, b) __dmul_rn(a, b)
#define AUG_DDIV(a, b) __ddiv_rn(a, b)
#define AUG_FADD(a, b) __fadd_rn(a, b)
#define AUG_FMUL(a, b) __fmul_rn(a, b)
#define AUG_FSUB(a, b) __fsub_rn(a, b)
#define AUG_FDIV(a, b) __fdiv_rn(a, b)
#else
#define AUG_DADD(a, b) ((a) + (b))     // the host build compiles with -ffp-contract=off
#define AUG_DSUB(a, b) ((a) - (b))
#define AUG_DMUL(a, b) ((a) * (b))
#define AUG_DDIV(a, b) ((a) / (b))
#define AUG_FADD(a, b) ((a) + (b))
#define AUG_FMUL(a, b) ((a) * (b))
#define AUG_FSUB(a, b) ((a) - (b))
#define AUG_FDIV(a, b) ((a) / (b))
#endif

namespace b2p {

constexpr int kAugMaxTaps = 16;         // a window spans at most 2 * ceil(2 * 3) + 1 = 13 inputs (in / out <= 3)
constexpr int kAugPrecisionBits = 22;   // Resample.c PRECISION_BITS (32 - 8 - 2)
constexpr int kAugMaxImages = 1024;
constexpr int kAugMinSide = 2, kAugMaxSide = 8192;     // int(side * 0.5) >= 1
constexpr int kAugMinEdge = 8, kAugMaxEdge = 1024;
constexpr unsigned char kAugPad[3] = {124, 116, 104};  // CenterPad's fill, RGB
enum : int { kAugBrightness = 0, kAugContrast = 1, kAugSaturation = 2, kAugHue = 3 };   // ColorJitter's fn_idx

// bicubic_filter with a = -0.5, evaluated as Resample.c's expressions are
B2P_AUG_HD double aug_bicubic(double x) {
    if (x < 0.0) x = -x;
    if (x < 1.0) return AUG_DADD(AUG_DMUL(AUG_DMUL(AUG_DSUB(AUG_DMUL(1.5, x), 2.5), x), x), 1.0);
    if (x < 2.0) return AUG_DMUL(AUG_DSUB(AUG_DMUL(AUG_DADD(AUG_DMUL(AUG_DSUB(x, 5.0), x), 8.0), x), 4.0), -0.5);
    return 0.0;
}

// The window of output index xx of an in_size -> out_size resize: first input *xmin, count returned, weights k[].
B2P_AUG_HD int aug_taps(int in_size, int out_size, int xx, int* xmin_out, int32_t* k) {
    const double scale = AUG_DDIV((double)(float)in_size, (double)out_size);
    const double filterscale = scale < 1.0 ? 1.0 : scale;
    const double support = AUG_DMUL(2.0, filterscale);
    const double center = AUG_DMUL(AUG_DADD((double)xx, 0.5), scale);      // in0 + ..., in0 = 0
    const double ss = AUG_DDIV(1.0, filterscale);
    int xmin = (int)AUG_DADD(AUG_DSUB(center, support), 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)AUG_DADD(AUG_DADD(center, support), 0.5);
    if (xmax > in_size) xmax = in_size;
    const int cnt = xmax - xmin;
    double w[kAugMaxTaps];
    double ww = 0.0;
    for (int x = 0; x < cnt; ++x) {
        w[x] = aug_bicubic(AUG_DMUL(AUG_DADD(AUG_DSUB((double)(x + xmin), center), 0.5), ss));
        ww = AUG_DADD(ww, w[x]);
    }
    for (int x = 0; x < cnt; ++x) {
        const double v = ww != 0.0 ? AUG_DDIV(w[x], ww) : w[x];
        const double f = AUG_DMUL(v, (double)(1 << kAugPrecisionBits));
        k[x] = v < 0 ? (int32_t)AUG_DADD(-0.5, f) : (int32_t)AUG_DADD(0.5, f);
    }
    *xmin_out = xmin;
    return cnt;
}

// clip8 of a finished fixed-point sum (which started at 1 << 21)
B2P_AUG_HD unsigned char aug_clip8(int32_t ss) {
    const int32_t v = ss >> kAugPrecisionBits;
    return (unsigned char)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// Image.blend(degenerate, image, f) of one byte (Blend.c, whose alpha is a C float): in1 + f (in2 - in1) in float,
// truncated; clipped to 0 .. 255 outside f in [0, 1]
B2P_AUG_HD unsigned char aug_blend(int in1, int in2, double f) {
    const float a = (float)f;
    const float t = AUG_FADD((float)in1, AUG_FMUL(a, (float)(in2 - in1)));
    if (a >= 0.0f && a <= 1.0f) return (unsigned char)(int)t;
    if (t <= 0.0f) return 0;
    if (t >= 255.0f) return 255;
    return (unsigned char)(int)t;
}

// convert('L')
B2P_AUG_HD int aug_luma(int r, int g, int b) { return (r * 19595 + g * 38470 + b * 7471 + 0x8000) >> 16; }

B2P_AUG_HD unsigned char aug_clip_int(int v) { return (unsigned char)(v < 0 ? 0 : (v > 255 ? 255 : v)); }

// adjust_hue of one RGB triple (in place) by the byte shift dh = np.int32(hue_factor * 255).astype(uint8)
B2P_AUG_HD void aug_hue(unsigned char* px, int dh) {
    const int r = px[0], g = px[1], b = px[2];
    const int maxc = r > g ? (r > b ? r : b) : (g > b ? g : b);
    const int minc = r < g ? (r < b ? r : b) : (g < b ? g : b);
    int uh = 0, us = 0;
    if (minc != maxc) {
        const float cr = (float)(maxc - minc);
        const float s = AUG_FDIV(cr, (float)maxc);
        const float rc = AUG_FDIV((float)(maxc - r), cr);
        const float gc = AUG_FDIV((float)(maxc - g), cr);
        const float bc = AUG_FDIV((float)(maxc - b), cr);
        float h;
        if (r == maxc) h = AUG_FSUB(bc, gc);
        else if (g == maxc) h = (float)AUG_DSUB(AUG_DADD(2.0, (double)rc), (double)bc);
        else h = (float)AUG_DSUB(AUG_DADD(4.0, (double)gc), (double)rc);
        h = (float)fmod(AUG_DADD(AUG_DDIV((double)h, 6.0), 1.0), 1.0);
        uh = aug_clip_int((int)AUG_DMUL((double)h, 255.0));
        us = aug_clip_int((int)AUG_DMUL((double)s, 255.0));
    }
    const int h8 = (uh + dh) & 255, s8 = us, v = maxc;
    if (s8 == 0) {
        px[0] = px[1] = px[2] = (unsigned char)v;
        return;
    }
    const double h6 = AUG_DDIV(AUG_DMUL((double)(float)h8, 6.0), 255.0);
    const int i = (int)floor(h6);
    const float f = (float)AUG_DSUB(h6, (double)(float)i);
    const float fs = (float)AUG_DDIV((double)(float)s8, 255.0);
    const double fv = (double)(float)v;
    const unsigned char up = aug_clip_int((int)round(AUG_DMUL(fv, AUG_DSUB(1.0, (double)fs))));
    const unsigned char uq = aug_clip_int((int)round(AUG_DMUL(fv, AUG_DSUB(1.0, (double)AUG_FMUL(fs, f)))));
    const unsigned char ut =
        aug_clip_int((int)round(AUG_DMUL(fv, AUG_DSUB(1.0, AUG_DMUL((double)fs, AUG_DSUB(1.0, (double)f))))));
    const unsigned char uv = (unsigned char)v;
    unsigned char o0, o1, o2;
    switch (i % 6) {
        case 0: o0 = uv; o1 = ut; o2 = up; break;
        case 1: o0 = uq; o1 = uv; o2 = up; break;
        case 2: o0 = up; o1 = uv; o2 = ut; break;
        case 3: o0 = up; o1 = uq; o2 = uv; break;
        case 4: o0 = ut; o1 = up; o2 = uv; break;
        default: o0 = uv; o1 = up; o2 = uq; break;
    }
    px[0] = o0;
    px[1] = o1;
    px[2] = o2;
}

// One ColorJitter operation other than contrast on an RGB triple (in place).  f: its factor; dh: the hue byte shift.
B2P_AUG_HD void aug_pointwise(int op, unsigned char* px, double f, int dh) {
    if (op == kAugBrightness) {
        for (int c = 0; c < 3; ++c) px[c] = aug_blend(0, px[c], f);
    } else if (op == kAugSaturation) {
        const int l = aug_luma(px[0], px[1], px[2]);
        for (int c = 0; c < 3; ++c) px[c] = aug_blend(l, px[c], f);
    } else if (op == kAugHue) {
        aug_hue(px, dh);
    }
}

// Contrast's degenerate grey: int(ImageStat mean of L + 0.5) from the integer sum of L over `count` pixels
B2P_AUG_HD int aug_contrast_mean(unsigned long long sum, long long count) {
    return (int)AUG_DADD(AUG_DDIV((double)sum, (double)count), 0.5);
}

}  // namespace b2p
