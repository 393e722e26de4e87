// Host-side interface of the wgmma "halo-patch" implicit-GEMM convolution (conv_tc.cu).
// Replaces the nn.Conv2d(+ReLU)(+MaxPool2d)(+torch.cat) sequences of the reference's
// lib/network/rtpose_vgg.py for every conv with Cin >= 64.
#pragma once
#include <cstdint>
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

namespace b2p {

constexpr int kTileW = 8;         // CTA tile: 8 (w) x 16 (h) output pixels = two wgmma M=64 halves of 8 x 8 (one per consumer warpgroup)
constexpr int kTileH = 16;
constexpr int kPatchPitch = 16;   // patch row pitch in pixels (8 + 6 halo, rounded up so that a patch is a multiple of 1024 B)
constexpr int kMaxKs = 7;
constexpr int kPatchBytes = kPatchPitch * (kTileH + kMaxKs - 1) * 128;  // 45,056 B per 64-channel block
constexpr int kBStageBytes = 128 * 128;                                 // up to N=128 rows of 64 bf16
#ifndef B2P_CONV_B_STAGES
#define B2P_CONV_B_STAGES 6      // weight (B operand) ring: 96 KB, cut into stages of `tps` taps (conv_tc.cu); with the two patch
                                 // stages a CTA holds 185 KB of the 227 KB an H100 block may use
#endif
constexpr int kNumBStages = B2P_CONV_B_STAGES;
#ifndef B2P_CONV_MIN_B_STAGES
#define B2P_CONV_MIN_B_STAGES 3
#endif
constexpr int kMinBStages = B2P_CONV_MIN_B_STAGES;     // a stage holds as many taps as still leave this many stages in the ring
constexpr int kMaxBStages = 16;       // the ring is cut into stages of the size the layer's n-tile needs (conv_tc.cu)
constexpr int kNumPatchStages = 2;
constexpr int kConvTcThreads = 384;   // warpgroup 0: producers (warp 0 patch TMA, warp 1 weight TMA); warpgroups 1, 2: MMA + epilogue
constexpr int kConvTcSmemBytes = kNumPatchStages * kPatchBytes + kNumBStages * kBStageBytes + 1024 /*align*/ + 512;

struct ConvTcArgs {
    // ---- geometry (stride 1, "same" padding, square kernel)
    int n_img, H, W;
    int ksize;                // 1, 3 or 7
    int cin_blocks;           // 64-channel blocks per group
    int in_ch_base;           // first input channel (in the NHWC buffer) of group 0
    int in_ch_group_stride;   // channel offset between groups in the input buffer (0 = groups share input)
    int groups;               // 1 or 2
    int n_tile;               // wgmma N: 32, 48, 64 or 128
    int n_tiles;              // N tiles per group
    // ---- epilogue
    const float* bias;        // [groups * n_tiles * n_tile]
    int relu;
    int pool;                 // fuse MaxPool2d(2,2): output is (H/2, W/2)
    __nv_bfloat16* out;       // NHWC bf16 (may be null)
    int out_cstride;          // channels per pixel of the output buffer
    int out_ch_off[2];        // first output channel per group
    int store_ch[2];          // channels (multiple of 8) stored per group *per n-tile*
    float* out_f32[2];        // optional NCHW fp32 copy per group (heads), may be null
    int f32_ch[2];            // valid channels of the fp32 copy
    // ---- split-precision ("bf16x3") mode: operands are hi + lo bf16 planes, three MMA terms per K block
    int split;                // 0: plain bf16; 1: A_hi*W_hi + A_hi*W_lo + A_lo*W_hi
    __nv_bfloat16* out_lo;    // residual plane of the output (same geometry as `out`), split mode only
    // ---- K-chunked accumulation (n_tile <= 64): see conv_tc_chunk_kernel
    int chunk;
    // ---- taps per weight stage (set by conv_tc_make_maps together with the weight map's box)
    int tps;
    // ---- programmatic dependent launch of this layer behind the previous one (small-batch plans)
    int pdl;
    // ---- tensor maps
    CUtensorMap tm_in;        // 4D (C, W, H, N) bf16, box (64, 16, 16+ks-1, 1), SWIZZLE_128B
    CUtensorMap tm_w;         // 3D (cin_pad, groups*n_tiles*n_tile, 2*taps) bf16 [hi taps | lo taps], box (64, n_tile, tps)
    CUtensorMap tm_in_lo;     // residual plane of the input (split mode)
};

// Builds the tensor maps. `in` (and `in_lo` in split mode): NHWC buffers with `in_cstride` channels per pixel.
// `w`: packed weights [2*taps][groups*n_tiles*n_tile][cin_blocks*64]: bf16(w) for the first `taps` slices, the
// residual bf16(w - hi) for the second.
cudaError_t conv_tc_make_maps(ConvTcArgs& a, const __nv_bfloat16* in, int in_cstride, const __nv_bfloat16* w,
                              const __nv_bfloat16* in_lo = nullptr);
cudaError_t conv_tc_launch(const ConvTcArgs& a, int num_sms, cudaStream_t stream);

#ifdef B2P_CONV_TIMELINE
// Debug builds only (tools/conv_timeline.sh): clock64() stamps of the first 64 CTAs at the phase boundaries of conv_tc_body.
constexpr int kTlSlots = 16;
cudaError_t conv_tc_read_timeline(unsigned long long* out /*[64 * kTlSlots]*/);     // copies and clears
#endif

}  // namespace b2p
