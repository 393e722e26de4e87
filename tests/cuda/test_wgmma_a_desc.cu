// Standalone GPU check of how conv_tc_kernel addresses its wgmma A operand in the halo patch (csrc/conv_tc.cu).
//
// A tap's window starts dx patch pixels (dx * 128 B) past a 1024-B boundary of the SWIZZLE_128B patch.  The matrix
// descriptor has a base-offset field (bits 49-51) for operands that do not start on the swizzle pattern's boundary; the
// kernel leaves it at 0, which is right if wgmma applies the swizzle of each row's absolute shared-memory address, as TMA
// did when it wrote the patch.  This check runs one tap (dy, dx) = (dx % 3, dx) for each dx of 0..6 on one 8 x 8 pixel
// half (M = 64, N = 64, K = 64: four k16 steps) three ways:
//   RS     A fragments from ldmatrix with the swizzle undone in the address (chunk c of pixel p at c ^ (p & 7)), the
//          register-A wgmma of conv_tc_kernel's fp8 path;
//   SS/0   A through a descriptor as conv_tc_kernel builds it: base offset 0;
//   SS/dx  the same with base offset dx & 7.
// SS/0 must equal RS bit for bit at every dx (same operands, same MMA order), and RS must match a float64 reference.
// SS/dx is reported, not required.  Build: see __graft_entry__.build().  Run on an H100: build/test_wgmma_a_desc
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include <cuda_bf16.h>

#include "../../pytorch_realtime_multi-person_pose_estimation_b200/csrc/ptx.cuh"

using namespace b2p;

#define CK(x)                                                                               \
    do {                                                                                    \
        cudaError_t e_ = (x);                                                               \
        if (e_ != cudaSuccess) {                                                            \
            printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
            exit(2);                                                                        \
        }                                                                                   \
    } while (0)

constexpr int kPitch = 16;                  // patch row pitch in pixels, as conv_tc_kernel's
constexpr int kRows = 8 + 2;                // the half's 8 pixel rows plus dy up to 2
constexpr int kPatchBytes = kRows * kPitch * 128;
constexpr int kN = 64;
constexpr int kTaps = 7;                    // dx = 0..6
constexpr int kVariants = 3;                // RS, SS/0, SS/dx
constexpr int kSmem = 1024 + kPatchBytes + kN * 128;

__device__ __forceinline__ void mma_rs(float (&d)[kN / 2], const uint32_t (&a)[4], uint64_t desc_b, uint32_t scale_d) {
    B2P_WGMMA_M64N64_RS("bf16", "16", ", 0");
}
__device__ __forceinline__ void mma_ss(float (&d)[kN / 2], uint64_t desc_a, uint64_t desc_b, uint32_t scale_d) {
    B2P_WGMMA_M64N64_SS("bf16");
}

// One CTA per dx, one warpgroup.  patch: [kRows * kPitch pixels][64 channels], w: [kN rows][64 k], both bf16 row-major;
// out[(variant * kTaps + dx) * 128 + thread][kN / 2]: the accumulator registers.
__global__ void __launch_bounds__(128) a_desc_probe(const __nv_bfloat16* patch, const __nv_bfloat16* w, float* out) {
    extern __shared__ uint8_t raw[];
    uint8_t* ps = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(raw) + 1023) & ~uintptr_t(1023));
    uint8_t* bs = ps + kPatchBytes;
    // SWIZZLE_128B placement, as TMA writes it into a 1024-B aligned buffer: 16-byte chunk c of row p at c ^ (p & 7)
    for (int i = threadIdx.x; i < kRows * kPitch * 8; i += blockDim.x) {
        const int p = i >> 3, c = i & 7;
        *reinterpret_cast<uint4*>(ps + p * 128 + ((c ^ (p & 7)) << 4)) = reinterpret_cast<const uint4*>(patch)[i];
    }
    for (int i = threadIdx.x; i < kN * 8; i += blockDim.x) {
        const int n = i >> 3, c = i & 7;
        *reinterpret_cast<uint4*>(bs + n * 128 + ((c ^ (n & 7)) << 4)) = reinterpret_cast<const uint4*>(w)[i];
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic-proxy stores -> wgmma reads
    __syncthreads();

    const int dx = blockIdx.x, dy = dx % 3;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint64_t bdesc = make_sdesc_sw128(smem_u32(bs), 1024);
    for (int v = 0; v < kVariants; ++v) {
        float acc[kN / 2];
#pragma unroll
        for (int i = 0; i < kN / 2; ++i) acc[i] = 0.f;
        if (v == 0) {
            const int r = (lane & 7) + ((lane >> 3) & 1) * 8, kc = lane >> 4;
            const int p = (2 * warp + (r >> 3) + dy) * kPitch + (r & 7) + dx;
            uint32_t af[4][4];
#pragma unroll
            for (int k = 0; k < 4; ++k) ldmatrix_x4(smem_u32(ps) + p * 128 + (((2 * k + kc) ^ (p & 7)) << 4), af[k]);
            fence_regs(acc);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) mma_rs(acc, af[k], bdesc + 2 * k, k > 0);
        } else {
            const uint64_t adesc = make_sdesc_sw128(smem_u32(ps) + (dy * kPitch + dx) * 128, kPitch * 128, v == 2 ? dx & 7 : 0);
            fence_regs(acc);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) mma_ss(acc, adesc + 2 * k, bdesc + 2 * k, k > 0);
        }
        wgmma_commit();
        wgmma_wait_all();
        fence_regs(acc);
        float* o = out + ((size_t)(v * kTaps + dx) * 128 + threadIdx.x) * (kN / 2);
#pragma unroll
        for (int i = 0; i < kN / 2; ++i) o[i] = acc[i];
    }
}

int main() {
    CK(cudaSetDevice(0));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    printf("device %s sm_%d%d\n", prop.name, prop.major, prop.minor);
    uint32_t rng = 777;
    auto frand = [&]() {
        rng = rng * 1664525u + 1013904223u;
        return ((rng >> 8) & 0xFFFF) / 65536.0f - 0.5f;
    };
    std::vector<__nv_bfloat16> patch(kRows * kPitch * 64), w(kN * 64);
    for (auto& x : patch) x = __float2bfloat16(frand());
    for (auto& x : w) x = __float2bfloat16(frand());
    __nv_bfloat16 *d_patch, *d_w;
    float* d_out;
    const size_t out_n = (size_t)kVariants * kTaps * 128 * (kN / 2);
    CK(cudaMalloc(&d_patch, patch.size() * 2));
    CK(cudaMalloc(&d_w, w.size() * 2));
    CK(cudaMalloc(&d_out, out_n * 4));
    CK(cudaMemcpy(d_patch, patch.data(), patch.size() * 2, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(d_w, w.data(), w.size() * 2, cudaMemcpyHostToDevice));
    CK(cudaMemset(d_out, 0xFF, out_n * 4));
    CK(cudaFuncSetAttribute(a_desc_probe, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
    a_desc_probe<<<kTaps, 128, kSmem>>>(d_patch, d_w, d_out);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    std::vector<float> out(out_n);
    CK(cudaMemcpy(out.data(), d_out, out_n * 4, cudaMemcpyDeviceToHost));

    int fails = 0;
    for (int dx = 0; dx < kTaps; ++dx) {
        const int dy = dx % 3;
        const float* rs = &out[(size_t)(0 * kTaps + dx) * 128 * (kN / 2)];
        int diff[kVariants] = {0, 0, 0};
        double worst = 0;      // RS against float64, in units of sum |a w|
        for (int t = 0; t < 128; ++t)
            for (int i = 0; i < kN / 2; ++i) {
                const size_t e = (size_t)t * (kN / 2) + i;
                for (int v = 1; v < kVariants; ++v)
                    if (memcmp(&rs[e], &out[(size_t)(v * kTaps + dx) * 128 * (kN / 2) + e], 4) != 0) ++diff[v];
                // accumulator register i of thread t: row m, column n of the 64 x N tile
                const int warp = t >> 5, lane = t & 31;
                const int m = 16 * warp + (lane >> 2) + 8 * ((i >> 1) & 1), n = 8 * (i >> 2) + 2 * (lane & 3) + (i & 1);
                const int p = (m / 8 + dy) * kPitch + m % 8 + dx;
                double r = 0, s = 0;
                for (int k = 0; k < 64; ++k) {
                    const double x = (double)__bfloat162float(patch[p * 64 + k]) * __bfloat162float(w[n * 64 + k]);
                    r += x;
                    s += std::fabs(x);
                }
                worst = std::fmax(worst, std::fabs(rs[e] - r) / s);
            }
        const bool ok = diff[1] == 0 && worst < 1e-4;
        printf("dx=%d dy=%d: RS vs float64 %.2e of sum|aw|; SS base offset 0: %d of %d words differ; SS base offset %d: %d "
               "differ  %s\n", dx, dy, worst, diff[1], 128 * kN / 2, dx & 7, diff[2], ok ? "OK" : "MISMATCH");
        fails += !ok;
    }
    cudaFree(d_patch); cudaFree(d_w); cudaFree(d_out);
    printf("wgmma A descriptor: %s\n", fails == 0 ? "ALL OK" : "FAILURES");
    return fails == 0 ? 0 : 1;
}
