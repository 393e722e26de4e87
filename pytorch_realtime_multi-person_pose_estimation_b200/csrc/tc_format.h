// The arithmetic format of the tensor-core path (DESIGN.md §2.3).  Every launch of a forward - conv1_1 and the 51
// conv_tc launches - runs in one format; what differs between the formats is written once here.
#pragma once
#include <cuda.h>

#ifdef __CUDACC__
#define B2P_HD __host__ __device__ __forceinline__
#else
#define B2P_HD inline
#endif

namespace b2p {

enum class TcFormat {
    kBf16,      // bf16 activations and weights, full-K fp32 accumulation
    kBf16x3,    // split precision: hi + residual bf16 planes, A_hi W_hi + A_hi W_lo + A_lo W_hi, K-chunked
    kFp8,       // e4m3 operands with per-image activation and per-row weight scales, K-chunked
    kFp16,      // IEEE binary16 activations and weights, full-K fp32 accumulation, overflow flags
};

// Packed weights a format reads (one copy per net and encoding)
enum class TcWeights {
    kBf16HiLo,  // [2 taps][rows][cin_pad] bf16: bf16(w) in the first `taps` slices, the residual bf16(w - hi) after them
    kE4m3,      // [taps][rows][cin_pad] e4m3(w * 2^ew[row]), each 32-channel slice in the K order of fp8_k_to_channel
    kBinary16,  // [taps][rows][cin_pad] binary16(w)
};
constexpr int kNumTcWeights = 3;

// Per-image table every launch of a format writes besides its outputs
enum class TcAux {
    kNone,
    kAmax,      // max |stored bf16| (fp32 bits) per launch and image: the next launches' activation scales
    kOverflow,  // 1 per image once a stored value is +-inf or NaN in binary16
};

// activation planes: the residual plane of bf16x3 holds v - bf16(v)
B2P_HD constexpr int tc_planes(TcFormat f) { return f == TcFormat::kBf16x3 ? 2 : 1; }
// K-chunked accumulation: the tensor core accumulates chunks of K that are added in fp32 into a second register set
B2P_HD constexpr bool tc_chunked(TcFormat f) { return f == TcFormat::kBf16x3 || f == TcFormat::kFp8; }
// activations (and weights) are IEEE binary16 rather than bf16
B2P_HD constexpr bool tc_binary16(TcFormat f) { return f == TcFormat::kFp16; }
B2P_HD constexpr TcWeights tc_weights(TcFormat f) {
    return f == TcFormat::kFp8 ? TcWeights::kE4m3 : (tc_binary16(f) ? TcWeights::kBinary16 : TcWeights::kBf16HiLo);
}
B2P_HD constexpr TcAux tc_aux(TcFormat f) {
    return f == TcFormat::kFp8 ? TcAux::kAmax : (tc_binary16(f) ? TcAux::kOverflow : TcAux::kNone);
}
// widest n-tile: the chunked formats' second register set leaves room for N <= 64
B2P_HD constexpr int tc_max_n_tile(TcFormat f) { return tc_chunked(f) ? 64 : 128; }

// TMA element type of the activation planes: fp8 reads bf16 and converts in registers
B2P_HD constexpr CUtensorMapDataType tc_act_type(TcFormat f) {
    return tc_binary16(f) ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
}
// bytes of one 64-channel weight row and the matching swizzle: 64 e4m3 bytes, or 64 16-bit values
B2P_HD constexpr int tc_w_row_bytes(TcFormat f) { return tc_weights(f) == TcWeights::kE4m3 ? 64 : 128; }
B2P_HD constexpr CUtensorMapSwizzle tc_w_swizzle(TcFormat f) {
    return tc_w_row_bytes(f) == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B;
}
B2P_HD constexpr CUtensorMapDataType tc_w_type(TcFormat f) {
    return tc_weights(f) == TcWeights::kE4m3 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : tc_act_type(f);
}
// tap slices of the packed weights: hi and residual slices for the bf16 encoding
B2P_HD constexpr int tc_w_slices(TcFormat f, int taps) { return tc_weights(f) == TcWeights::kBf16HiLo ? 2 * taps : taps; }

}  // namespace b2p
