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
//     of the k*k filter taps then reads its shifted window of that SAME patch with ldmatrix (the swizzle is undone in the
//     address: 16-byte chunk c of patch pixel p sits at chunk c ^ (p & 7)), so the activation tile is fetched from L2
//     once instead of k*k times.  The fragments feed wgmma with A in registers.
//   * TMA 3-D loads bring the [n_tile x 64] weight slices (K-major, SWIZZLE_128B) of `tps` consecutive taps per stage into
//     a 96 KB ring; wgmma reads them through a shared-memory descriptor.
//   * A warpgroup issues the four k16 steps of a tap as one wgmma group and waits for it before its ldmatrix overwrites
//     the A registers; the other warpgroup's MMAs fill the tensor cores meanwhile.
//   * The fp32 accumulators stay in registers: bias, ReLU, the optional 2x2 max-pool (vertical pair in-thread, horizontal
//     pair through one shuffle), conversion to bf16 and NHWC stores; the stage heads additionally emit fp32 NCHW outputs.
//   * Persistent grid (one CTA per SM), static round-robin tile schedule; warp 0 (patches) and warp 1 (weights) run
//     ahead of the consumers through mbarrier rings and prefetch the next tile's operands during the epilogue.
#include <cstdio>

#include "conv_tc.cuh"
#include "host_util.h"
#include "ptx.cuh"

namespace b2p {

#ifdef B2P_CONV_TIMELINE
__device__ unsigned long long g_conv_timeline[64 * kTlSlots];
#define B2P_TL(slot) do { if (blockIdx.x < 64) g_conv_timeline[blockIdx.x * kTlSlots + (slot)] = clock64(); } while (0)
#else
#define B2P_TL(slot) do { } while (0)
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

template <int N> struct Mma;
template <> struct Mma<128> {
    static __device__ __forceinline__ void run(float (&d)[64], const uint32_t (&a)[4], uint64_t b, uint32_t s) { wgmma_m64n128k16_rs(d, a, b, s); }
};
template <> struct Mma<64> {
    static __device__ __forceinline__ void run(float (&d)[32], const uint32_t (&a)[4], uint64_t b, uint32_t s) { wgmma_m64n64k16_rs(d, a, b, s); }
};
template <> struct Mma<48> {
    static __device__ __forceinline__ void run(float (&d)[24], const uint32_t (&a)[4], uint64_t b, uint32_t s) { wgmma_m64n48k16_rs(d, a, b, s); }
};
template <> struct Mma<32> {
    static __device__ __forceinline__ void run(float (&d)[16], const uint32_t (&a)[4], uint64_t b, uint32_t s) { wgmma_m64n32k16_rs(d, a, b, s); }
};

constexpr int kConsumerWarps = 8;

template <int N, bool kChunk>
__device__ __forceinline__ void conv_tc_body(const ConvTcArgs& a) {
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
    constexpr uint32_t b_tx = N * 128;                       // one tap's weight slice
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
        // ldmatrix: this lane addresses A row r (pixel (lh, lw) of the tile), 16-byte K chunk kc of each k16 step
        const int r = (lane & 7) + ((lane >> 3) & 1) * 8;
        const int kc = lane >> 4;
        const int lh = 8 * wg + 2 * wi + (r >> 3);
        const int lw = r & 7;
        // accumulators: this lane holds pixels (hA, wA) and (hA + 1, wA), columns 8 j + cq, 8 j + cq + 1
        const int hA = 8 * wg + 2 * wi;
        const int wA = lane >> 2;
        const int cq = 2 * (lane & 3);
        const uint32_t patch0 = smem_u32(patch_smem);
        const uint64_t bdesc_hi = make_sdesc_sw128(0, 1024);
        const uint32_t b_lo0 = (smem_u32(b_smem) & 0x3FFFFu) >> 4;
        const bool row_chunks = kChunk && a.ksize == 7;    // K-chunked mode: one chunk per filter row (7x7; tps == 1) ...
        const bool blk_chunks = kChunk && !row_chunks;     // ... or per (channel block, term)
        const int Ho = a.pool ? a.H >> 1 : a.H;
        const int Wo = a.pool ? a.W >> 1 : a.W;
        float acc[N / 2];
        float sum[kChunk ? N / 2 : 1];
#pragma unroll
        for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
        uint32_t pi = 0, pph = 0, bi = 0, bph = 0;
        for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
            const TileCoord tc = decode_tile(t, a.n_tiles, a.groups, tiles_x, tiles_y);
            if (kChunk) {
#pragma unroll
                for (int i = 0; i < N / 2; ++i) sum[i] = 0.f;
            }
            uint32_t scale = 0;       // 0: the next MMA overwrites the accumulators
            for (int cb = 0; cb < a.cin_blocks; ++cb) {
                for (int term = 0; term < nterms; ++term) {
                    // term 0 and 1 read the hi patch (against W_hi, W_lo), term 2 the residual patch (against W_hi)
                    if (term != 1) mbar_wait(&patch_full[pi], pph);
                    if (wi == 0 && lane == 0 && t == (int)blockIdx.x) B2P_TL(2 + (cb & 1));
                    const bool release_patch = (term == nterms - 1) || (term == 1);
                    if (blk_chunks) scale = 0;
                    const uint32_t pbase = patch0 + pi * kPatchBytes;
                    int dy = 0, dx = 0;
                    for (int tap0 = 0; tap0 < taps; tap0 += tps) {          // one weight stage = tps consecutive taps
                        const int cnt = taps - tap0 < tps ? taps - tap0 : tps;
                        if (row_chunks && dx == 0) scale = 0;
                        mbar_wait(&b_full[bi], bph);
                        const uint32_t b_lo = b_lo0 + bi * (b_stride >> 4);
                        for (int j = 0; j < cnt; ++j) {
                            const int p = (lh + dy) * kPatchPitch + lw + dx;     // patch pixel of this lane's A row
                            const uint32_t row_addr = pbase + p * 128;
                            const int sw = p & 7;
                            uint32_t af[4][4];
#pragma unroll
                            for (int k = 0; k < 4; ++k) ldmatrix_x4(row_addr + (((2 * k + kc) ^ sw) << 4), af[k]);
                            fence_regs(acc);
                            wgmma_fence();
#pragma unroll
                            for (int k = 0; k < 4; ++k) {
                                Mma<N>::run(acc, af[k], bdesc_hi | (b_lo + j * (b_tx >> 4) + k * 2), scale);
                                scale = 1;
                            }
                            wgmma_commit();
                            wgmma_wait_all();      // the next tap's ldmatrix reuses the A registers
                            fence_regs(acc);
                            if (++dx == a.ksize) { dx = 0; ++dy; }
                        }
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&b_empty[bi]);
                        if (++bi == nb) { bi = 0; bph ^= 1; }
                        if (row_chunks && dx == 0) {       // a filter row is complete: add the chunk in fp32
#pragma unroll
                            for (int i = 0; i < N / 2; ++i) sum[i] = __fadd_rn(sum[i], acc[i]);
                        }
                    }
                    if (blk_chunks) {
#pragma unroll
                        for (int i = 0; i < N / 2; ++i) sum[i] = __fadd_rn(sum[i], acc[i]);
                    }
                    if (release_patch) {
                        __syncwarp();
                        if (lane == 0) mbar_arrive(&patch_empty[pi]);
                        if (++pi == kNumPatchStages) { pi = 0; pph ^= 1; }
                    }
                }
            }
            if (wi == 0 && lane == 0 && t == (int)blockIdx.x) B2P_TL(5);

            // ---- epilogue
            const int ch_tile = tc.nt * N;                     // first channel of this n-tile within the group
            const float* bias = a.bias + (tc.g * a.n_tiles + tc.nt) * N;
            const int store_ch = a.store_ch[tc.g];
            float* of32 = a.out_f32[tc.g];
            const int f32_ch = a.f32_ch[tc.g];
            const int x = tc.x0 + wA;
            __nv_bfloat16* out_px[2] = {nullptr, nullptr};     // first channel of this n-tile at the lane's output pixel(s)
            int yo_px[2] = {0, 0}, xo = a.pool ? x >> 1 : x;
            bool wr[2];
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
                const int y = tc.y0 + hA + hh;
                // pooled: the lane with even w holds the 2x2 window (both rows) after the shuffle
                wr[hh] = (y < a.H) && (x < a.W) && (a.pool ? (hh == 0 && !(lane & 4)) : true);
                yo_px[hh] = a.pool ? y >> 1 : y;
                if (a.out != nullptr)
                    out_px[hh] = a.out + (static_cast<size_t>(tc.n * Ho + yo_px[hh]) * Wo + xo) * a.out_cstride +
                                 a.out_ch_off[tc.g] + ch_tile + cq;
            }
#pragma unroll
            for (int j = 0; j < N / 8; ++j) {
                const float2 b2 = __ldg(reinterpret_cast<const float2*>(bias + 8 * j + cq));
                float v[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    v[e] = (kChunk ? sum[4 * j + e] : acc[4 * j + e]) + ((e & 1) ? b2.y : b2.x);
                    if (a.relu) v[e] = fmaxf(v[e], 0.f);
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
                    const float lo = v[2 * hh], hi = v[2 * hh + 1];
                    if (out_px[hh] != nullptr && 8 * j < store_ch) {
                        *reinterpret_cast<uint32_t*>(out_px[hh] + 8 * j) = pack_bf16x2(lo, hi);
                        if (a.out_lo != nullptr) {      // split mode: residual plane v - bf16(v)
                            __nv_bfloat16* dlo = a.out_lo + (out_px[hh] - a.out) + 8 * j;
                            *reinterpret_cast<uint32_t*>(dlo) =
                                pack_bf16x2(lo - __bfloat162float(__float2bfloat16_rn(lo)), hi - __bfloat162float(__float2bfloat16_rn(hi)));
                        }
                    }
                    if (of32 != nullptr) {
                        const int c = ch_tile + 8 * j + cq;
                        if (c < f32_ch) of32[(static_cast<size_t>(tc.n * f32_ch + c) * Ho + yo_px[hh]) * Wo + xo] = lo;
                        if (c + 1 < f32_ch) of32[(static_cast<size_t>(tc.n * f32_ch + c + 1) * Ho + yo_px[hh]) * Wo + xo] = hi;
                    }
                }
            }
            if (wi == 0 && lane == 0 && t == (int)blockIdx.x) B2P_TL(7);
        }
    }
    if (threadIdx.x == 0) B2P_TL(9);
}

template <int N, bool kChunk>
__global__ void __launch_bounds__(kConvTcThreads, 1) conv_tc_kernel(const __grid_constant__ ConvTcArgs a) {
    conv_tc_body<N, kChunk>(a);
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

cudaError_t conv_tc_make_maps(ConvTcArgs& a, const __nv_bfloat16* in, int in_cstride, const __nv_bfloat16* w,
                              const __nv_bfloat16* in_lo) {
    PFN_encodeTiled enc = get_encode_fn();
    if (enc == nullptr) return cudaErrorNotSupported;
    if (a.ksize != 1 && a.ksize != 3 && a.ksize != 7) return cudaErrorInvalidValue;
    if (a.n_tile != 32 && a.n_tile != 48 && a.n_tile != 64 && a.n_tile != 128) return cudaErrorInvalidValue;
    if (a.groups < 1 || a.groups > 2 || in_cstride % 8 != 0) return cudaErrorInvalidValue;
    if (a.split && in_lo == nullptr) return cudaErrorInvalidValue;
    for (int plane = 0; plane <= (a.split ? 1 : 0); ++plane) {
        cuuint64_t dims[4] = {(cuuint64_t)in_cstride, (cuuint64_t)a.W, (cuuint64_t)a.H, (cuuint64_t)a.n_img};
        cuuint64_t strides[3] = {(cuuint64_t)in_cstride * 2, (cuuint64_t)a.W * in_cstride * 2,
                                 (cuuint64_t)a.H * a.W * in_cstride * 2};
        cuuint32_t box[4] = {64, (cuuint32_t)kPatchPitch, (cuuint32_t)(kTileH + a.ksize - 1), 1};
        cuuint32_t estr[4] = {1, 1, 1, 1};
        CUresult r = enc(plane ? &a.tm_in_lo : &a.tm_in, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4,
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
        // 4 KB).  The K-chunked 7x7 mode closes a chunk at every filter-row end, which a stage must not straddle.
        const int tap_bytes = a.n_tile * 128;
        int tps = (kNumBStages * kBStageBytes) / (kMinBStages * tap_bytes);
        if (tps < 1 || (a.chunk && a.ksize == 7)) tps = 1;
        if (tps > taps) tps = taps;
        a.tps = tps;
        cuuint64_t dims[3] = {(cuuint64_t)cin_pad, (cuuint64_t)rows, (cuuint64_t)(2 * taps)};
        cuuint64_t strides[2] = {(cuuint64_t)cin_pad * 2, (cuuint64_t)rows * cin_pad * 2};
        cuuint32_t box[3] = {64, (cuuint32_t)a.n_tile, (cuuint32_t)tps};
        cuuint32_t estr[3] = {1, 1, 1};
        CUresult r = enc(&a.tm_w, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, const_cast<__nv_bfloat16*>(w), dims, strides,
                         box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
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
template <int N, bool kChunk>
cudaError_t launch(int grid, cudaStream_t stream, const ConvTcArgs& a) {
    static DynSmemOptIn optin;   // per device: a second net on another GPU of the same process needs its own opt-in
    cudaError_t e = optin.ensure(conv_tc_kernel<N, kChunk>, kConvTcSmemBytes);
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
        return cudaLaunchKernelEx(&cfg, conv_tc_kernel<N, kChunk>, a);
    }
    conv_tc_kernel<N, kChunk><<<grid, kConvTcThreads, kConvTcSmemBytes, stream>>>(a);
    return cudaGetLastError();
}
}  // namespace

cudaError_t conv_tc_launch(const ConvTcArgs& a, int num_sms, cudaStream_t stream) {
    if (a.pool && ((a.H | a.W) & 1)) return cudaErrorInvalidValue;
    if (a.chunk && a.n_tile > 64) return cudaErrorInvalidValue;      // K-chunked mode keeps a second accumulator set
    if (a.tps < 1) return cudaErrorInvalidValue;                     // conv_tc_make_maps has not run
    const int tiles_x = (a.W + kTileW - 1) / kTileW;
    const int tiles_y = (a.H + kTileH - 1) / kTileH;
    const int total = a.n_img * tiles_y * tiles_x * a.groups * a.n_tiles;
    const int grid = total < num_sms ? total : num_sms;
    switch (a.n_tile) {
        case 128: return launch<128, false>(grid, stream, a);
        case 64: return a.chunk ? launch<64, true>(grid, stream, a) : launch<64, false>(grid, stream, a);
        case 48: return a.chunk ? launch<48, true>(grid, stream, a) : launch<48, false>(grid, stream, a);
        case 32: return a.chunk ? launch<32, true>(grid, stream, a) : launch<32, false>(grid, stream, a);
        default: return cudaErrorInvalidValue;
    }
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
