// FP8 (OCP E4M3FN) scaling rules of the fp8 mode (DESIGN.md §2.3), shared by the kernels, the host weight packer and the
// host test build (tests/test_fp8_host.py).  Plain C++ plus __host__ __device__: no CUDA header is needed on the host.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

#ifdef __CUDACC__
#define B2P_HD __host__ __device__ __forceinline__
#else
#define B2P_HD inline
#endif

namespace b2p {

constexpr int kFp8ExpClamp = 63;      // scale exponents are clamped to [-63, 63]: 2^-(ea + ew), |ea + ew| <= 126, is a normal float
constexpr float kE4m3Max = 448.f;

// e = floor(log2(448 / amax)) from the bits of amax >= 0 (an fp32 bit pattern), clamped to [-63, 63]; 0 for amax = 0.
// 448 = 1.75 * 2^8, so for amax = 1.m * 2^E the quotient is (1.75 / 1.m) * 2^(8 - E): e = 8 - E, less one when 1.m > 1.75.
// A denormal amax (< 2^-126) gives e >= 134, i.e. the clamp.
B2P_HD int fp8_exp_from_amax(uint32_t bits) {
    bits &= 0x7fffffffu;
    if (bits == 0) return 0;
    const int E = (int)(bits >> 23) - 127;
    if (E == -127) return kFp8ExpClamp;
    int e = 8 - E - ((bits & 0x7fffffu) > 0x600000u ? 1 : 0);
    return e < -kFp8ExpClamp ? -kFp8ExpClamp : (e > kFp8ExpClamp ? kFp8ExpClamp : e);
}

// 2^e as a float, |e| <= 126
B2P_HD float exp2_int(int e) {
    const uint32_t u = (uint32_t)(e + 127) << 23;
    float f;
    memcpy(&f, &u, 4);
    return f;
}

// Host reference of the device conversion (cvt.rn.satfinite.e4m3x2.f32): round to nearest even on the E4M3FN grid
// (subnormal step 2^-9, 3 mantissa bits, largest finite 448), saturating to +-448.  Returns the byte encoding.
inline uint8_t e4m3_rn_bits(float x) {
    const uint8_t sign = std::signbit(x) ? 0x80 : 0;
    const double a = std::fabs((double)x);
    if (std::isnan(x)) return sign | 0x7f;
    if (a >= 464.0) return sign | 0x7e;                  // satfinite (464: the midpoint above 448)
    int e = a > 0 ? (int)std::floor(std::log2(a)) : -9;  // binade; refined below (log2 is not trusted at exact powers)
    if (a > 0) {
        if (std::ldexp(1.0, e) > a) --e;
        if (std::ldexp(1.0, e + 1) <= a) ++e;
    }
    if (e < -6) e = -6;                                  // subnormals share the exponent of the smallest normal
    const double step = std::ldexp(1.0, e - 3);
    double q = std::nearbyint(a / step);                 // default rounding mode: ties to even
    double v = q * step;                                 // may carry into the next binade (q == 16)
    if (v == 0) return sign;
    int ev = e;
    if (q >= 16) { ev = e + 1; q /= 2; }
    if (ev == -6 && q < 8) return sign | (uint8_t)q;     // subnormal: exponent field 0
    return sign | (uint8_t)(((ev + 7) << 3) | ((int)q - 8));
}

inline float e4m3_to_float(uint8_t b) {
    const int s = b >> 7, ef = (b >> 3) & 15, m = b & 7;
    const double v = ef == 0 ? std::ldexp((double)m, -9) : std::ldexp(1.0 + m / 8.0, ef - 7);
    return (float)(s ? -v : v);
}

// K order of an e4m3 k32 wgmma step fed from two bf16 k16 ldmatrix fragments (conv_tc.cu): logical k of the step ->
// input channel within its 32-channel slice.  Byte j of A register 0 / 2 holds row r, k = 4q + j / 16 + 4q + j, which the
// bf16 fragments hold at channels 2q, 2q + 1, 2q + 8, 2q + 9 of k16 step 0 / 1.
B2P_HD int fp8_k_to_channel(int k) {
    const int half = k >> 4, kk = k & 15, q = kk >> 2, j = kk & 3;
    return 16 * half + 2 * q + (j & 1) + 8 * (j >> 1);
}

}  // namespace b2p
