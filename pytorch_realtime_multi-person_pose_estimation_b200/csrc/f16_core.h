// IEEE binary16 rounding of the fp16 mode's weight packer (DESIGN.md §2.3), shared by the library and the host test build
// (tests/test_fp16_host.py).  Plain C++: no CUDA header is needed.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

namespace b2p {

// fp32 -> binary16 bits, round to nearest even, subnormals kept (step 2^-24), |x| >= 65520 (the midpoint above 65504,
// which ties to the even inf) -> +-inf, NaN -> quiet NaN.  One rounding: the same result as a direct conversion of the
// float's exact value.
inline uint16_t f16_rn_bits(float x) {
    uint32_t u;
    memcpy(&u, &x, 4);
    const uint16_t sign = (uint16_t)((u >> 16) & 0x8000u);
    const uint32_t a = u & 0x7fffffffu;
    if (a > 0x7f800000u) return sign | 0x7e00u;
    if (a >= 0x477ff000u) return sign | 0x7c00u;
    if (a >= 0x38800000u) {            // normal in binary16 (>= 2^-14): drop 13 mantissa bits, ties to even, rebias 127 -> 15
        const uint32_t r = a + 0xfffu + ((a >> 13) & 1u);
        return sign | (uint16_t)((r - 0x38000000u) >> 13);
    }
    // subnormal in binary16: a multiple of 2^-24; |x| * 2^24 is exact in double, nearbyint ties to even (default mode)
    return sign | (uint16_t)std::nearbyint((double)std::fabs(x) * 16777216.0);
}

}  // namespace b2p
