// wgmma "halo-patch" implicit-GEMM convolution for sm_90a (H100).
//
// Computes, for every conv of the rtpose VGG19 net with Cin >= 64 (the reference's lib/network/rtpose_vgg.py),
// out = act(conv_kxk(in) + bias) with optional fused MaxPool2d(2,2) and "concat by construction" (the epilogue writes
// straight into a channel slice of the next layer's NHWC buffer, replacing the reference's torch.cat).
//
// Mapping to the hardware (see DESIGN.md "conv_tc"):
//   * A CTA owns an 8 (w) x 16 (h) block of output pixels; each of its two consumer warpgroups owns one 8 x 8 half, i.e.
//     the M = 64 rows of its wgmma (row m = pixel (h = m / 8, w = m % 8) of the half).
//   * For each 64-channel block of the input, ONE TMA 4-D tile load brings the (16+k-1) x 16 pixel halo patch (NHWC bf16,
//     128 B per pixel, SWIZZLE_128B, out-of-image pixels zero-filled by TMA = conv padding) into shared memory.  Every one
//     of the k*k filter taps then reads its shifted window of that SAME patch, so the activation tile is fetched from L2
//     once instead of k*k times.  bf16, bf16x3 and fp16 hand the window to wgmma as a shared-memory descriptor (start at
//     patch pixel (8 wg + dy, dx), one patch row between 8-row core groups, base offset 0); fp8 loads it with ldmatrix
//     (the swizzle undone in the address: 16-byte chunk c of patch pixel p sits at chunk c ^ (p & 7)) and converts the
//     fragments to e4m3 for a wgmma with A in registers.
//   * TMA 3-D loads bring the [n_tile x 64] weight slices (K-major, SWIZZLE_128B) of `tps` consecutive taps per stage into
//     a 96 KB ring; wgmma reads them through a shared-memory descriptor.
//   * A warpgroup issues each weight stage as one wgmma group and lets it run while it waits for the previous stage's
//     group, then releases that stage (and its patch after the patch's last stage); only a K-chunk end (bf16x3) and the
//     tile end wait for all.  fp8 issues one group per tap and waits for it, since the next tap's conversion reuses the
//     A registers.
//   * The fp32 accumulators stay in registers: bias, ReLU, the optional 2x2 max-pool (vertical pair in-thread, horizontal
//     pair through one shuffle), conversion to bf16 and NHWC stores; the stage heads additionally emit fp32 NCHW outputs.
//   * Persistent grid (one CTA per SM), static round-robin tile schedule; warp 0 (patches) and warp 1 (weights) run
//     ahead of the consumers through mbarrier rings and prefetch the next tile's operands during the epilogue.
#include <cstdio>
#include <type_traits>

#include "conv_tc.cuh"
#include "fp8_core.h"
#include "host_util.h"
#include "ptx.cuh"

namespace b2p {

#ifdef B2P_CONV_TIMELINE
__device__ unsigned long long g_conv_timeline[64 * kTlSlots];
#define B2P_TL(slot) do { if (blockIdx.x < 64) g_conv_timeline[blockIdx.x * kTlSlots + (slot)] = clock64(); } while (0)
// clocks a consumer thread spends in `stmt`, added to `acc` (slots kTlPatchWait.. of conv_tc.cuh)
#define B2P_TL_TIME(acc, stmt) do { const long long t0_ = clock64(); stmt; acc += clock64() - t0_; } while (0)
#else
#define B2P_TL(slot) do { } while (0)
#define B2P_TL_TIME(acc, stmt) stmt
#endif

namespace {

struct TileCoord {
    int n, y0, x0, g, nt;
};

// Work item t = one (pixel tile, group, n-tile).  (n-tile, group) vary fastest so that CTAs running at the same time read
// the same activation patches from L2.
__device__ __forceinline__ TileCoord decode_tile(int t, int n_tiles, int groups, int tiles_x, int tiles_y) {
    TileCoord c;
    c.nt = t % n_tiles;
    t /= n_tiles;
    c.g = t % groups;
    t /= groups;
    c.x0 = (t % tiles_x) * kTileW;
    t /= tiles_x;
    c.y0 = (t % tiles_y) * kTileH;
    c.n = t / tiles_y;
    return c;
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
    __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<uint32_t*>(&v);
}

// fp8: k32 wgmma on e4m3 operands with A in registers (converted from the bf16 patch per tap)
#define B2P_MMA(SHAPE) SHAPE("e4m3", "32", "")
template <TcFormat F, int N>
__device__ __forceinline__ void mma(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t desc_b, uint32_t scale_d) {
    static_assert(tc_weights(F) == TcWeights::kE4m3, "the 16-bit formats read A from shared memory (mma_ss)");
    if constexpr (N == 128) { B2P_MMA(B2P_WGMMA_M64N128_RS); }
    else if constexpr (N == 64) { B2P_MMA(B2P_WGMMA_M64N64_RS); }
    else if constexpr (N == 48) { B2P_MMA(B2P_WGMMA_M64N48_RS); }
    else { static_assert(N == 32, "n-tile"); B2P_MMA(B2P_WGMMA_M64N32_RS); }
}
#undef B2P_MMA

// bf16, bf16x3 and fp16: k16 wgmma with A read from the halo patch through a descriptor
#define B2P_MMA(SHAPE)                             \
    if constexpr (tc_binary16(F)) SHAPE("f16");    \
    else SHAPE("bf16")
template <TcFormat F, int N>
__device__ __forceinline__ void mma_ss(float (&d)[N / 2], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
    if constexpr (N == 128) { B2P_MMA(B2P_WGMMA_M64N128_SS); }
    else if constexpr (N == 64) { B2P_MMA(B2P_WGMMA_M64N64_SS); }
    else if constexpr (N == 48) { B2P_MMA(B2P_WGMMA_M64N48_SS); }
    else { static_assert(N == 32, "n-tile"); B2P_MMA(B2P_WGMMA_M64N32_SS); }
}
#undef B2P_MMA

constexpr int kConsumerWarps = 8;

// A consumer warp is done with weight stage b and, when p >= 0, with patch stage p: one arrive on each.
__device__ __forceinline__ void release_stage(int b, int p, int lane, uint64_t* b_empty, uint64_t* patch_empty) {
    __syncwarp();
    if (lane == 0) {
        mbar_arrive(&b_empty[b]);
        if (p >= 0) mbar_arrive(&patch_empty[p]);
    }
}

// F: the arithmetic format (tc_format.h).  kRagged: a.ext is set (ragged batch); a separate instantiation so that uniform
// batches run the unmasked epilogue.
// fp8 (DESIGN.md §2.3): each tap's A fragments are converted from the bf16 patch to e4m3 in registers, the weights are
// e4m3 slices of 64-byte rows, every tap's two k32 MMAs start a fresh accumulator that is then added to the fp32 sum,
// and the epilogue records the per-image max |stored bf16|.
// fp16: the bf16 plan with binary16 activations and weights (same fragments, same full-K fp32 accumulation); the
// epilogue stores binary16 and flags every image for which a stored value is +-inf or NaN.
// kPrelu: the epilogue applies the per-channel PReLU of a.slope instead of a.relu (a separate instantiation, so that the
// kernels without it keep their machine code).
template <TcFormat F, int N, bool kRagged, bool kPrelu>
__device__ __forceinline__ void conv_tc_body(const ConvTcArgs& a) {
    constexpr bool kChunk = tc_chunked(F);
    constexpr bool kE4m3 = tc_weights(F) == TcWeights::kE4m3;
    constexpr TcAux kAux = tc_aux(F);
    extern __shared__ uint8_t smem_raw[];
    // SWIZZLE_128B operands need 1024 B alignment.
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t* patch_smem = smem;
    uint8_t* b_smem = smem + kNumPatchStages * kPatchBytes;
    uint64_t* bars = reinterpret_cast<uint64_t*>(b_smem + kNumBStages * kBStageBytes);
    uint64_t* patch_full = bars;                          // [2]
    uint64_t* patch_empty = bars + kNumPatchStages;       // [2]
    uint64_t* b_full = bars + 2 * kNumPatchStages;        // [kMaxBStages]
    uint64_t* b_empty = b_full + kMaxBStages;             // [kMaxBStages]

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    if (threadIdx.x == 0) B2P_TL(0);

    const int tiles_x = (a.W + kTileW - 1) / kTileW;
    const int tiles_y = (a.H + kTileH - 1) / kTileH;
    const int total_tiles = a.n_img * tiles_y * tiles_x * a.groups * a.n_tiles;
    const int taps = a.ksize * a.ksize;
    const int pad = a.ksize >> 1;
    const uint32_t patch_tx = kPatchPitch * (kTileH + a.ksize - 1) * 128;
    constexpr uint32_t b_tx = N * tc_w_row_bytes(F);         // one tap's weight slice
    // The weight ring is cut into stages of `tps` consecutive taps (a.tps, chosen with the tensor map's box): fewer, larger
    // stages mean fewer barrier round trips per tile.
    const int tps = a.tps;
    const uint32_t b_stride = b_tx * tps;                    // multiples of 1024 B (n_tile % 8 == 0)
    const uint32_t nb_fit = (kNumBStages * kBStageBytes) / b_stride;
    const uint32_t nb = nb_fit < (uint32_t)kMaxBStages ? nb_fit : (uint32_t)kMaxBStages;
    const int nterms = a.split ? 3 : 1;   // split mode: A_hi*W_hi, A_hi*W_lo, A_lo*W_hi per K block

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&a.tm_in);
        tma_prefetch_desc(&a.tm_w);
        if (a.split) tma_prefetch_desc(&a.tm_in_lo);
        for (int i = 0; i < kNumPatchStages; ++i) {
            mbar_init(&patch_full[i], 1);
            mbar_init(&patch_empty[i], kConsumerWarps);     // one arrive per consumer warp
        }
        for (uint32_t i = 0; i < nb; ++i) {
            mbar_init(&b_full[i], 1);
            mbar_init(&b_empty[i], kConsumerWarps);
        }
        fence_mbar_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) B2P_TL(1);
    // PDL (no-ops unless the launch carries the attribute): let the next layer start its prologue now; everything that reads
    // or writes activations first waits for the previous layer's grid to complete (weights / bias are constants).
    pdl_launch_dependents();

    if (warp == 0) {
        // =========================== TMA producer: activation halo patches ===========================
        if (lane == 0) {
            pdl_wait();
            uint32_t pi = 0, pph = 0;
            for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
                const TileCoord tc = decode_tile(t, a.n_tiles, a.groups, tiles_x, tiles_y);
                const int ch0 = a.in_ch_base + tc.g * a.in_ch_group_stride;
                for (int cb = 0; cb < a.cin_blocks; ++cb) {
                    for (int plane = 0; plane <= a.split; ++plane) {     // hi plane, then (split mode) the residual plane
                        mbar_wait(&patch_empty[pi], pph ^ 1);
                        mbar_expect_tx(&patch_full[pi], patch_tx);
                        tma_load_4d(patch_smem + pi * kPatchBytes, plane ? &a.tm_in_lo : &a.tm_in, &patch_full[pi],
                                    ch0 + cb * 64, tc.x0 - pad, tc.y0 - pad, tc.n);
                        if (++pi == kNumPatchStages) { pi = 0; pph ^= 1; }
                    }
                }
            }
        }
    } else if (warp == 1) {
        // =========================== TMA producer: weight slices ===========================
        if (lane == 0) {
            uint32_t bi = 0, bph = 0;
            for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
                const TileCoord tc = decode_tile(t, a.n_tiles, a.groups, tiles_x, tiles_y);
                const int wrow = (tc.g * a.n_tiles + tc.nt) * N;
                for (int cb = 0; cb < a.cin_blocks; ++cb) {
                    for (int term = 0; term < nterms; ++term) {          // W_hi, (split) W_lo, W_hi
                        const int wsel = (term == 1) ? taps : 0;
                        for (int tap0 = 0; tap0 < taps; tap0 += tps) {       // (the last box of a block may run past `taps`:
                            mbar_wait(&b_empty[bi], bph ^ 1);             //  those slices are loaded and not read)
                            mbar_expect_tx(&b_full[bi], b_stride);
                            tma_load_3d(b_smem + bi * b_stride, &a.tm_w, &b_full[bi], cb * 64, wrow, wsel + tap0);
                            if (++bi == nb) { bi = 0; bph ^= 1; }
                        }
                    }
                }
            }
        }
    } else if (warp >= 4) {
        // =========================== consumers: MMAs + epilogue (warpgroups 1 and 2) ===========================
        pdl_wait();               // (stores of this layer may overwrite what the previous layer still reads)
        const int wg = (warp >> 2) - 1;      // pixel rows 8 * wg .. 8 * wg + 7 of the tile
        const int wi = warp & 3;             // accumulator rows 16 * wi .. 16 * wi + 15 of the warpgroup
        // fp8's ldmatrix: this lane addresses A row r (pixel (lh, lw) of the tile), 16-byte K chunk kc of each k16 step
        const int r = (lane & 7) + ((lane >> 3) & 1) * 8;
        const int kc = lane >> 4;
        const int lh = 8 * wg + 2 * wi + (r >> 3);
        const int lw = r & 7;
        // accumulators: this lane holds pixels (hA, wA) and (hA + 1, wA), columns 8 j + cq, 8 j + cq + 1
        const int hA = 8 * wg + 2 * wi;
        const int wA = lane >> 2;
        const int cq = 2 * (lane & 3);
        const uint32_t patch0 = smem_u32(patch_smem);
        const uint64_t bdesc_hi = kE4m3 ? make_sdesc_sw64(0, 512) : make_sdesc_sw128(0, 1024);
        const uint32_t b_lo0 = (smem_u32(b_smem) & 0x3FFFFu) >> 4;
        // The 16-bit formats' A operand, read by wgmma from the patch: row m of the warpgroup is pixel (m / 8, m % 8) of
        // its half, so the 8-row core groups are the half's pixel rows, one patch row (SBO) apart, and the window of tap
        // (dy, dx) starts at patch pixel (8 wg + dy, dx).  The broadcast keeps the descriptors on the uniform datapath.
        const uint64_t adesc_hi = make_sdesc_sw128(0, kPatchPitch * 128);
        uint32_t a_lo0 = 0;
        if constexpr (!kE4m3)
            a_lo0 = ((smem_u32(patch_smem) & 0x3FFFFu) >> 4) + __shfl_sync(0xffffffffu, wg, 0) * (8 * kPatchPitch * 128 >> 4);
        // bf16x3: one K chunk per filter row (7x7; tps == 1), else per (channel block, term); fp8: per tap
        const bool row_chunks = kChunk && !kE4m3 && a.ksize == 7;
        const int Ho = a.pool ? a.H >> 1 : a.H;
        const int Wo = a.pool ? a.W >> 1 : a.W;
        float acc[N / 2];
        float sum[kChunk ? N / 2 : 1];
#pragma unroll
        for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
        uint32_t pi = 0, pph = 0, bi = 0, bph = 0;
#ifdef B2P_CONV_TIMELINE
        long long tl_pw = 0, tl_bw = 0, tl_dr = 0, tl_main = 0, tl_epi = 0, tl_t = 0;
        int tl_tiles = 0;
#endif
        for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
#ifdef B2P_CONV_TIMELINE
            tl_t = clock64();
            ++tl_tiles;
#endif
            const TileCoord tc = decode_tile(t, a.n_tiles, a.groups, tiles_x, tiles_y);
            if (kChunk) {
#pragma unroll
                for (int i = 0; i < N / 2; ++i) sum[i] = 0.f;
            }
            int ea = 0;           // fp8: the activation scale exponent of this tile's image
            float sa = 1.f;
            if constexpr (kE4m3) {
                uint32_t m = __ldcg(a.amax_in[0] + tc.n);
                if (a.amax_in[1] != nullptr) m = max(m, __ldcg(a.amax_in[1] + tc.n));
                ea = fp8_exp_from_amax(m);
                sa = exp2_int(ea);
                if (a.ea_out != nullptr && warp == 4 && lane == 0) a.ea_out[tc.n] = ea;
            }
            uint32_t scale = 0;       // 0: the next MMA overwrites the accumulators
            if constexpr (!kE4m3) {
                // One wgmma group per weight stage.  After committing it, wait_group 1 shows the previous stage's group
                // complete, so that stage (and, after its patch's last stage, the patch) is released while this one
                // runs.  pend_b, pend_p: the stage and patch (-1: none) whose group may still be in flight.
                // bf16x3 drains at each K-chunk end and adds the chunk in fp32.  The chunk ends are loop exits, not
                // branches: ptxas serialises every wgmma when the accumulators are read on a conditional path while a
                // group may be in flight.
                int pend_b = -1, pend_p = -1;
                for (int cb = 0; cb < a.cin_blocks; ++cb) {
                    for (int term = 0; term < nterms; ++term) {
                        // term 0 and 1 read the hi patch (against W_hi, W_lo), term 2 the residual patch (against W_hi)
                        if (term != 1) B2P_TL_TIME(tl_pw, mbar_wait(&patch_full[pi], pph));
                        if (wi == 0 && lane == 0 && t == (int)blockIdx.x) B2P_TL(2 + (cb & 1));
                        const bool release_patch = (term == nterms - 1) || (term == 1);
                        const uint32_t a_lo = a_lo0 + pi * (kPatchBytes >> 4);
                        int dy = 0, dx = 0, tap0 = 0;
                        while (tap0 < taps) {        // bf16x3: one K chunk (a 7x7 filter row, or the block) per pass
                            do {                     // one weight stage = tps consecutive taps
                                const int cnt = taps - tap0 < tps ? taps - tap0 : tps;
                                B2P_TL_TIME(tl_bw, mbar_wait(&b_full[bi], bph));
                                const uint32_t b_lo = b_lo0 + bi * (b_stride >> 4);
                                fence_regs(acc);
                                wgmma_fence();
                                for (int j = 0; j < cnt; ++j) {
                                    const uint32_t a_tap = a_lo + (dy * kPatchPitch + dx) * (128 >> 4);
#pragma unroll
                                    for (int k = 0; k < 4; ++k) {
                                        mma_ss<F, N>(acc, adesc_hi | (a_tap + k * 2),
                                                     bdesc_hi | (b_lo + j * (b_tx >> 4) + k * 2), scale);
                                        scale = 1;
                                    }
                                    if (++dx == a.ksize) { dx = 0; ++dy; }
                                }
                                wgmma_commit();
                                tap0 += tps;
                                B2P_TL_TIME(tl_dr, wgmma_wait<1>());
                                if (pend_b >= 0) release_stage(pend_b, pend_p, lane, b_empty, patch_empty);
                                pend_b = bi;
                                pend_p = tap0 >= taps && release_patch ? (int)pi : -1;
                                if (++bi == nb) { bi = 0; bph ^= 1; }
                            } while (tap0 < taps && !(row_chunks && dx == 0));
                            if constexpr (kChunk) {
                                B2P_TL_TIME(tl_dr, wgmma_wait<0>());
                                fence_regs(acc);
                                release_stage(pend_b, pend_p, lane, b_empty, patch_empty);
                                pend_b = -1;
#pragma unroll
                                for (int i = 0; i < N / 2; ++i) sum[i] = __fadd_rn(sum[i], acc[i]);
                                scale = 0;           // the next chunk starts from fresh accumulators
                            }
                        }
                        if (release_patch) {
                            if (++pi == kNumPatchStages) { pi = 0; pph ^= 1; }
                        }
                    }
                }
                B2P_TL_TIME(tl_dr, wgmma_wait<0>());     // the tile's last group, before the epilogue reads acc
                fence_regs(acc);
                if (pend_b >= 0) release_stage(pend_b, pend_p, lane, b_empty, patch_empty);
            } else {
            for (int cb = 0; cb < a.cin_blocks; ++cb) {
                for (int term = 0; term < nterms; ++term) {
                    // term 0 and 1 read the hi patch (against W_hi, W_lo), term 2 the residual patch (against W_hi)
                    if (term != 1) B2P_TL_TIME(tl_pw, mbar_wait(&patch_full[pi], pph));
                    if (wi == 0 && lane == 0 && t == (int)blockIdx.x) B2P_TL(2 + (cb & 1));
                    const bool release_patch = (term == nterms - 1) || (term == 1);
                    const uint32_t pbase = patch0 + pi * kPatchBytes;
                    int dy = 0, dx = 0;
                    for (int tap0 = 0; tap0 < taps; tap0 += tps) {          // one weight stage = tps consecutive taps
                        const int cnt = taps - tap0 < tps ? taps - tap0 : tps;
                        B2P_TL_TIME(tl_bw, mbar_wait(&b_full[bi], bph));
                        const uint32_t b_lo = b_lo0 + bi * (b_stride >> 4);
                        for (int j = 0; j < cnt; ++j) {
                            const int p = (lh + dy) * kPatchPitch + lw + dx;     // patch pixel of this lane's A row
                            const uint32_t row_addr = pbase + p * 128;
                            const int sw = p & 7;
                            uint32_t af[4][4];
#pragma unroll
                            for (int k = 0; k < 4; ++k) ldmatrix_x4(row_addr + (((2 * k + kc) ^ sw) << 4), af[k]);
                            // k32 step s takes bf16 k16 steps 2s, 2s + 1 (K order: fp8_k_to_channel)
                            uint32_t a8[2][4];
#pragma unroll
                            for (int s = 0; s < 2; ++s) {
                                a8[s][0] = bf16x4_to_e4m3x4(af[2 * s][0], af[2 * s][2], sa);
                                a8[s][1] = bf16x4_to_e4m3x4(af[2 * s][1], af[2 * s][3], sa);
                                a8[s][2] = bf16x4_to_e4m3x4(af[2 * s + 1][0], af[2 * s + 1][2], sa);
                                a8[s][3] = bf16x4_to_e4m3x4(af[2 * s + 1][1], af[2 * s + 1][3], sa);
                            }
                            fence_regs(acc);
                            wgmma_fence();
#pragma unroll
                            for (int s = 0; s < 2; ++s)
                                mma<F, N>(acc, a8[s], bdesc_hi | (b_lo + j * (b_tx >> 4) + s * 2), s);
                            wgmma_commit();
                            B2P_TL_TIME(tl_dr, wgmma_wait_all());
                            fence_regs(acc);
#pragma unroll
                            for (int i = 0; i < N / 2; ++i) sum[i] = __fadd_rn(sum[i], acc[i]);
                            if (++dx == a.ksize) { dx = 0; ++dy; }
                        }
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&b_empty[bi]);
                        if (++bi == nb) { bi = 0; bph ^= 1; }
                    }
                    if (release_patch) {
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&patch_empty[pi]);
                        if (++pi == kNumPatchStages) { pi = 0; pph ^= 1; }
                    }
                }
            }
            }
            if (wi == 0 && lane == 0 && t == (int)blockIdx.x) B2P_TL(5);
#ifdef B2P_CONV_TIMELINE
            tl_main += clock64() - tl_t;
            tl_t = clock64();
#endif

            // ---- epilogue
            const int ch_tile = tc.nt * N;                     // first channel of this n-tile within the group
            const float* bias = a.bias + (tc.g * a.n_tiles + tc.nt) * N;
            const int* w_exp = a.w_exp + (tc.g * a.n_tiles + tc.nt) * N;
            uint32_t amax = 0;    // fp8: max |stored bf16| bits of this lane
            uint32_t ovf = 0;     // fp16: non-zero once a value this lane stored is not finite
            const int store_ch = a.store_ch[tc.g];
            float* of32 = a.out_f32[tc.g];
            const int f32_ch = a.f32_ch[tc.g];
            const int x = tc.x0 + wA;
            __nv_bfloat16* out_px[2] = {nullptr, nullptr};     // first channel of this n-tile at the lane's output pixel(s)
            int yo_px[2] = {0, 0}, xo = a.pool ? x >> 1 : x;
            bool wr[2], inside[2];
            int eh = Ho, ew = Wo;                              // the image's extent at the output resolution
            if (kRagged) {
                eh = __ldg(a.ext + 2 * tc.n) >> a.ext_shift;
                ew = __ldg(a.ext + 2 * tc.n + 1) >> a.ext_shift;
            }
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                const int y = tc.y0 + hA + hh;
                // pooled: the lane with even w holds the 2x2 window (both rows) after the shuffle
                wr[hh] = (y < a.H) && (x < a.W) && (a.pool ? (hh == 0 && !(lane & 4)) : true);
                yo_px[hh] = a.pool ? y >> 1 : y;
                inside[hh] = !kRagged || (yo_px[hh] < eh && xo < ew);
                if (a.out != nullptr)
                    out_px[hh] = a.out + (static_cast<size_t>(tc.n * Ho + yo_px[hh]) * Wo + xo) * a.out_cstride +
                                 a.out_ch_off[tc.g] + ch_tile + cq;
            }
            // The per-channel constants of kEpC column groups at a time are loaded before any of their stores: loaded next to
            // each group's stores, every one of the N / 8 groups waited a full load latency behind the previous group.
            constexpr int kEpC = N / 8 < 8 ? N / 8 : 8;
            // The column groups are unrolled, so their code is the largest part of the kernel, and every tile runs it once,
            // after the main loop has taken the instruction caches.  Only the stage heads write fp32 maps and only bf16x3
            // has a residual plane, so those paths are compiled into a separate copy (kF32) or only into the bf16x3
            // kernels: the copy a launch runs holds none of the stores it never makes (DESIGN.md §6, *Epilogue code*).
            auto columns = [&](auto f32_tag) {
            constexpr bool kF32 = decltype(f32_tag)::value;
#pragma unroll
            for (int j0 = 0; j0 < N / 8; j0 += kEpC) {
            float2 bias2[kEpC];
            [[maybe_unused]] float2 slope2[kPrelu ? kEpC : 1];
            [[maybe_unused]] int2 wexp2[kE4m3 ? kEpC : 1];
#pragma unroll
            for (int j = j0; j < j0 + kEpC; ++j) {
                bias2[j - j0] = __ldg(reinterpret_cast<const float2*>(bias + 8 * j + cq));
                if constexpr (kE4m3) wexp2[j - j0] = __ldg(reinterpret_cast<const int2*>(w_exp + 8 * j + cq));
                if constexpr (kPrelu)
                    slope2[j - j0] = __ldg(reinterpret_cast<const float2*>(a.slope + (tc.g * a.n_tiles + tc.nt) * N + 8 * j + cq));
            }
#pragma unroll
            for (int j = j0; j < j0 + kEpC; ++j) {
                const float2 b2 = bias2[j - j0];
                float v[4];
                if constexpr (kE4m3) {    // acc * 2^-(ea + ew) is exact: one rounding, at the bias add
                    const int2 w2 = wexp2[j - j0];
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        v[e] = __fadd_rn(__fmul_rn(sum[4 * j + e], exp2_int(-(ea + ((e & 1) ? w2.y : w2.x)))),
                                         (e & 1) ? b2.y : b2.x);
                        if (a.relu) v[e] = fmaxf(v[e], 0.f);
                    }
                } else if constexpr (kPrelu) {    // torch's prelu: one multiply, after the bias
                    const float2 s2 = slope2[j - j0];
#pragma unroll
                    for (int e = 0; e < 4; ++e) {
                        const float u = (kChunk ? sum[4 * j + e] : acc[4 * j + e]) + ((e & 1) ? b2.y : b2.x);
                        v[e] = u > 0.f ? u : __fmul_rn((e & 1) ? s2.y : s2.x, u);
                    }
                } else {
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    v[e] = (kChunk ? sum[4 * j + e] : acc[4 * j + e]) + ((e & 1) ? b2.y : b2.x);
                    if (a.relu) v[e] = fmaxf(v[e], 0.f);
                }
                }
                if (a.pool) {
                    v[0] = fmaxf(v[0], v[2]);
                    v[1] = fmaxf(v[1], v[3]);
                    v[0] = fmaxf(v[0], __shfl_xor_sync(0xffffffffu, v[0], 4));
                    v[1] = fmaxf(v[1], __shfl_xor_sync(0xffffffffu, v[1], 4));
                }
#pragma unroll
                for (int hh = 0; hh < 2; ++hh) {
                    if (!wr[hh]) continue;
                    const float lo = inside[hh] ? v[2 * hh] : 0.f, hi = inside[hh] ? v[2 * hh + 1] : 0.f;
                    if (out_px[hh] != nullptr && 8 * j < store_ch) {
                        if constexpr (kAux == TcAux::kAmax) {
                            const uint32_t pk = pack_bf16x2(lo, hi);
                            *reinterpret_cast<uint32_t*>(out_px[hh] + 8 * j) = pk;
                            amax = max(amax, max(pk & 0x7fffu, (pk >> 16) & 0x7fffu));
                        } else if constexpr (kAux == TcAux::kOverflow) {
                            const uint32_t pk = pack_f16x2(lo, hi);
                            *reinterpret_cast<uint32_t*>(out_px[hh] + 8 * j) = pk;
                            ovf |= f16x2_nonfinite(pk);
                        } else {
                            *reinterpret_cast<uint32_t*>(out_px[hh] + 8 * j) = pack_bf16x2(lo, hi);
                        }
                        if constexpr (tc_planes(F) == 2) {
                            if (a.out_lo != nullptr) {      // bf16x3: residual plane v - bf16(v)
                                __nv_bfloat16* dlo = a.out_lo + (out_px[hh] - a.out) + 8 * j;
                                *reinterpret_cast<uint32_t*>(dlo) = pack_bf16x2(lo - __bfloat162float(__float2bfloat16_rn(lo)),
                                                                                hi - __bfloat162float(__float2bfloat16_rn(hi)));
                            }
                        }
                    }
                    if constexpr (kF32) {
                        const int c = ch_tile + 8 * j + cq;
                        if (c < f32_ch) of32[(static_cast<size_t>(tc.n * f32_ch + c) * Ho + yo_px[hh]) * Wo + xo] = lo;
                        if (c + 1 < f32_ch) of32[(static_cast<size_t>(tc.n * f32_ch + c + 1) * Ho + yo_px[hh]) * Wo + xo] = hi;
                    }
                }
            }
            }
            };
            if (of32 != nullptr) columns(std::true_type{});
            else columns(std::false_type{});
            if constexpr (kAux == TcAux::kAmax) {     // max of non-negative float bits: order-independent, so runs stay deterministic
                amax = __reduce_max_sync(0xffffffffu, amax);
                if (lane == 0 && amax != 0) atomicMax(a.amax_out + tc.n, amax << 16);
            }
            // fp16: only lanes that stored a non-finite value take part; ptxas aggregates them into one reduction per warp.
            // No vote and no lane-0 branch here: either makes the whole tile loop divergent for the compiler, which then
            // builds the wgmma descriptors in vector registers instead of on the uniform datapath (5 % slower).
            if constexpr (kAux == TcAux::kOverflow) {
                if (ovf) atomicOr(a.ovf_out + tc.n, 1u);
            }
            if (wi == 0 && lane == 0 && t == (int)blockIdx.x) B2P_TL(7);
#ifdef B2P_CONV_TIMELINE
            tl_epi += clock64() - tl_t;
#endif
        }
#ifdef B2P_CONV_TIMELINE
        if (warp == 4 && lane == 0 && blockIdx.x < 64) {
            unsigned long long* s = g_conv_timeline + blockIdx.x * kTlSlots;
            s[kTlPatchWait] = tl_pw;
            s[kTlWeightWait] = tl_bw;
            s[kTlMain] = tl_main;
            s[kTlEpilogue] = tl_epi;
            s[kTlTiles] = tl_tiles;
            s[kTlDrain] = tl_dr;
        }
#endif
    }
    if (threadIdx.x == 0) B2P_TL(9);
}

template <TcFormat F, int N, bool kRagged, bool kPrelu>
__global__ void __launch_bounds__(kConvTcThreads, 1) conv_tc_kernel(const __grid_constant__ ConvTcArgs a) {
    conv_tc_body<F, N, kRagged, kPrelu>(a);
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode_fn() {
    static PFN_encodeTiled fn = nullptr;
    if (fn == nullptr) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess ||
            qres != cudaDriverEntryPointSuccess)
            return nullptr;
        fn = reinterpret_cast<PFN_encodeTiled>(p);
    }
    return fn;
}

}  // namespace

cudaError_t conv_tc_make_maps(ConvTcArgs& a, const __nv_bfloat16* in, int in_cstride, const void* w,
                              const __nv_bfloat16* in_lo) {
    PFN_encodeTiled enc = get_encode_fn();
    if (enc == nullptr) return cudaErrorNotSupported;
    if (a.ksize != 1 && a.ksize != 3 && a.ksize != 7) return cudaErrorInvalidValue;
    if (a.n_tile != 32 && a.n_tile != 48 && a.n_tile != 64 && a.n_tile != 128) return cudaErrorInvalidValue;
    if (a.groups < 1 || a.groups > 2 || in_cstride % 8 != 0) return cudaErrorInvalidValue;
    if (a.n_tile > tc_max_n_tile(a.fmt)) return cudaErrorInvalidValue;
    if (tc_planes(a.fmt) == 2 && in_lo == nullptr) return cudaErrorInvalidValue;
    a.split = tc_planes(a.fmt) - 1;
    for (int plane = 0; plane < tc_planes(a.fmt); ++plane) {
        cuuint64_t dims[4] = {(cuuint64_t)in_cstride, (cuuint64_t)a.W, (cuuint64_t)a.H, (cuuint64_t)a.n_img};
        cuuint64_t strides[3] = {(cuuint64_t)in_cstride * 2, (cuuint64_t)a.W * in_cstride * 2,
                                 (cuuint64_t)a.H * a.W * in_cstride * 2};
        cuuint32_t box[4] = {64, (cuuint32_t)kPatchPitch, (cuuint32_t)(kTileH + a.ksize - 1), 1};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        CUresult r = enc(plane ? &a.tm_in_lo : &a.tm_in, tc_act_type(a.fmt), 4,
                         const_cast<__nv_bfloat16*>(plane ? in_lo : in), dims, strides,
                         box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) {
            fprintf(stderr, "[b200pose] cuTensorMapEncodeTiled(in) failed: %d\n", (int)r);
            return cudaErrorInvalidValue;
        }
    }
    {
        const int cin_pad = a.cin_blocks * 64;
        const int rows = a.groups * a.n_tiles * a.n_tile;
        const int taps = a.ksize * a.ksize;
        // taps per weight stage: as many as leave kMinBStages stages in the ring (N = 128: 2 taps of 16 KB, N = 32: 8 taps of
        // 4 KB).  bf16x3 closes a 7x7 chunk at every filter-row end, which a stage must not straddle (fp8 chunks per tap).
        const int esz = tc_w_row_bytes(a.fmt) / 64;      // bytes per weight
        const int tap_bytes = a.n_tile * 64 * esz;
        int tps = (kNumBStages * kBStageBytes) / (kMinBStages * tap_bytes);
        if (tps < 1 || (tc_chunked(a.fmt) && tc_weights(a.fmt) != TcWeights::kE4m3 && a.ksize == 7)) tps = 1;
        if (tps > taps) tps = taps;
        a.tps = tps;
        cuuint64_t dims[3] = {(cuuint64_t)cin_pad, (cuuint64_t)rows, (cuuint64_t)tc_w_slices(a.fmt, taps)};
        cuuint64_t strides[2] = {(cuuint64_t)cin_pad * esz, (cuuint64_t)rows * cin_pad * esz};
        cuuint32_t box[3] = {64, (cuuint32_t)a.n_tile, (cuuint32_t)tps};
        cuuint32_t estr[3] = {1, 1, 1};
        CUresult r = enc(&a.tm_w, tc_w_type(a.fmt), 3, const_cast<void*>(w), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, tc_w_swizzle(a.fmt),
                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        if (r != CUDA_SUCCESS) {
            fprintf(stderr, "[b200pose] cuTensorMapEncodeTiled(w) failed: %d\n", (int)r);
            return cudaErrorInvalidValue;
        }
    }
    return cudaSuccess;
}

namespace {
// Programmatic dependent launch (a.pdl): the next layer's CTAs may start - barrier init, descriptor prefetch, weight loads -
// while this layer's last CTAs drain; they wait (griddepcontrol.wait) before touching activations.  Used by the SMALL-batch
// plans only, where the fixed cost per launch is most of a layer.
template <TcFormat F, int N>
cudaError_t launch_k(int grid, cudaStream_t stream, const ConvTcArgs& a) {
    // per kernel (uniform, ragged; PReLU) and device: a second net on another GPU of the same process needs its own opt-in
    static DynSmemOptIn optin[4];
    const bool ragged = a.ext != nullptr;
    const bool prelu = a.slope != nullptr;
    void (*kernel)(ConvTcArgs) = ragged ? conv_tc_kernel<F, N, true, false> : conv_tc_kernel<F, N, false, false>;
    if (prelu) {      // PReLU (OpenPose_Model's plans) in the formats those plans run: bf16, bf16x3
        if constexpr (tc_weights(F) == TcWeights::kBf16HiLo)
            kernel = ragged ? conv_tc_kernel<F, N, true, true> : conv_tc_kernel<F, N, false, true>;
        else
            return cudaErrorInvalidValue;
    }
    cudaError_t e = optin[2 * prelu + ragged].ensure(kernel, kConvTcSmemBytes);
    if (e != cudaSuccess) return e;
    if (a.pdl) {
        cudaLaunchConfig_t cfg = {};
        cfg.gridDim = dim3(grid);
        cfg.blockDim = dim3(kConvTcThreads);
        cfg.dynamicSmemBytes = kConvTcSmemBytes;
        cfg.stream = stream;
        cudaLaunchAttribute attr[1];
        attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        attr[0].val.programmaticStreamSerializationAllowed = 1;
        cfg.attrs = attr;
        cfg.numAttrs = 1;
        return cudaLaunchKernelEx(&cfg, kernel, a);
    }
    kernel<<<grid, kConvTcThreads, kConvTcSmemBytes, stream>>>(a);
    return cudaGetLastError();
}

// n-tiles 128 (not in the chunked formats), 64, 48 and 32
template <TcFormat F>
cudaError_t launch(int grid, cudaStream_t stream, const ConvTcArgs& a) {
    switch (a.n_tile) {
        case 128:
            if constexpr (tc_max_n_tile(F) >= 128) return launch_k<F, 128>(grid, stream, a);
            break;
        case 64: return launch_k<F, 64>(grid, stream, a);
        case 48: return launch_k<F, 48>(grid, stream, a);
        case 32: return launch_k<F, 32>(grid, stream, a);
    }
    return cudaErrorInvalidValue;
}
}  // namespace

cudaError_t conv_tc_launch(const ConvTcArgs& a, int num_sms, cudaStream_t stream) {
    if (a.pool && ((a.H | a.W) & 1)) return cudaErrorInvalidValue;
    if (a.tps < 1) return cudaErrorInvalidValue;                     // conv_tc_make_maps has not run
    if (tc_aux(a.fmt) == TcAux::kAmax && (a.amax_out == nullptr || a.amax_in[0] == nullptr || a.w_exp == nullptr))
        return cudaErrorInvalidValue;
    if (tc_aux(a.fmt) == TcAux::kOverflow && a.ovf_out == nullptr) return cudaErrorInvalidValue;
    const int tiles_x = (a.W + kTileW - 1) / kTileW;
    const int tiles_y = (a.H + kTileH - 1) / kTileH;
    const int total = a.n_img * tiles_y * tiles_x * a.groups * a.n_tiles;
    const int grid = total < num_sms ? total : num_sms;
    switch (a.fmt) {
        case TcFormat::kBf16: return launch<TcFormat::kBf16>(grid, stream, a);
        case TcFormat::kBf16x3: return launch<TcFormat::kBf16x3>(grid, stream, a);
        case TcFormat::kFp8: return launch<TcFormat::kFp8>(grid, stream, a);
        case TcFormat::kFp16: return launch<TcFormat::kFp16>(grid, stream, a);
    }
    return cudaErrorInvalidValue;
}

#ifdef B2P_CONV_TIMELINE
cudaError_t conv_tc_read_timeline(unsigned long long* out) {
    cudaError_t e = cudaMemcpyFromSymbol(out, g_conv_timeline, sizeof(g_conv_timeline));
    if (e != cudaSuccess) return e;
    void* p = nullptr;
    e = cudaGetSymbolAddress(&p, g_conv_timeline);
    if (e != cudaSuccess) return e;
    return cudaMemset(p, 0, sizeof(g_conv_timeline));
}
#endif

}  // namespace b2p
