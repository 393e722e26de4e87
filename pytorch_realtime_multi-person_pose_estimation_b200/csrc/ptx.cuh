// Thin inline-PTX wrappers for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), warpgroup MMA (wgmma), ldmatrix.
// Everything here is hand-written for this repo; no CUTLASS/CuTe types are used.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include <cuda.h>

namespace b2p {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------- programmatic dependent launch
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred P;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, P;\n\t}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a pipeline bug must trap (a reported launch error) instead of hanging the GPU.  No printf here: a function
// call between wgmmas makes ptxas serialise the wgmma pipeline.
#ifndef B2P_WAIT_LIMIT
#define B2P_WAIT_LIMIT (1u << 27)
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if (++spins > B2P_WAIT_LIMIT) __trap();
    }
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2) {
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2),
        "r"(c3)
        : "memory");
}

// ---------------------------------------------------------------- ldmatrix
// Four 8x8 bf16 matrices; lane l supplies the row address of row (l & 7) of matrix (l >> 3).  With matrices ordered
// (rows 0-7, k 0-7), (rows 8-15, k 0-7), (rows 0-7, k 8-15), (rows 8-15, k 8-15) the result is the A fragment of a
// 16 x 16 slice as mma.m16n8k16 and wgmma (A in registers) expect it.
__device__ __forceinline__ void ldmatrix_x4(uint32_t saddr, uint32_t (&r)[4]) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                 : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
                 : "r"(saddr)
                 : "memory");
}

// ---------------------------------------------------------------- wgmma
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// Waits until at most `kPending` of this warpgroup's committed wgmma groups are still in flight.
template <int kPending>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kPending) : "memory"); }
// Keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs.
template <int N>
__device__ __forceinline__ void fence_regs(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// Shared-memory matrix descriptor (sm_90 layout), K-major, 128-byte swizzle: rows are 128 B (64 bf16) apart inside an
// 8-row group, groups are `sbo_bytes` apart.  [0,14) addr>>4, [16,30) LBO>>4 (unused for SW128 K-major), [32,46) SBO>>4,
// [49,52) base offset, [62,64) layout (1 = SWIZZLE_128B).  conv_tc_kernel's operands were written by TMA with the
// swizzle of their absolute address and use base offset 0, also where they start past a 1024 B boundary
// (tests/cuda/test_wgmma_a_desc.cu checks that rule against ldmatrix fragments).
__device__ __forceinline__ uint64_t make_sdesc_sw128(uint32_t saddr, uint32_t sbo_bytes, uint32_t base_offset = 0) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);
    d |= 1ull << 16;
    d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
    d |= static_cast<uint64_t>(base_offset & 7u) << 49;
    d |= 1ull << 62;
    return d;
}

// D[64 x N] (+)= A[64 x K, registers] * B[K x N, shared memory descriptor] -> fp32, the statement for one N, used
// inside a function with the operands d (float[N / 2]), a (uint32_t[4]), desc_b and scale_d (0: D = A * B).
// TYPE, K: "bf16" or "f16" with K = "16" (the same A fragments and K-major B layout for both), or "e4m3" with
// K = "32".  TAIL: ", 0" (B not transposed) for the 16-bit types, "" for e4m3, which has no transpose operand.
#define B2P_WGMMA_M64N128_RS(TYPE, K, TAIL) \
    asm volatile( \
        "{\n\t.reg .pred p;\n\t" \
        "setp.ne.b32 p, %69, 0;\n\t" \
        "wgmma.mma_async.sync.aligned.m64n128k" K ".f32." TYPE "." TYPE " " \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, " \
        "{%64, %65, %66, %67}, %68, p, 1, 1" TAIL ";\n\t}\n" \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]) \
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(scale_d) \
        : "memory")

#define B2P_WGMMA_M64N64_RS(TYPE, K, TAIL) \
    asm volatile( \
        "{\n\t.reg .pred p;\n\t" \
        "setp.ne.b32 p, %37, 0;\n\t" \
        "wgmma.mma_async.sync.aligned.m64n64k" K ".f32." TYPE "." TYPE " " \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, " \
        "{%32, %33, %34, %35}, %36, p, 1, 1" TAIL ";\n\t}\n" \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]) \
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(scale_d) \
        : "memory")

#define B2P_WGMMA_M64N48_RS(TYPE, K, TAIL) \
    asm volatile( \
        "{\n\t.reg .pred p;\n\t" \
        "setp.ne.b32 p, %29, 0;\n\t" \
        "wgmma.mma_async.sync.aligned.m64n48k" K ".f32." TYPE "." TYPE " " \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, " \
        "{%24, %25, %26, %27}, %28, p, 1, 1" TAIL ";\n\t}\n" \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]) \
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(scale_d) \
        : "memory")

#define B2P_WGMMA_M64N32_RS(TYPE, K, TAIL) \
    asm volatile( \
        "{\n\t.reg .pred p;\n\t" \
        "setp.ne.b32 p, %21, 0;\n\t" \
        "wgmma.mma_async.sync.aligned.m64n32k" K ".f32." TYPE "." TYPE " " \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, " \
        "{%16, %17, %18, %19}, %20, p, 1, 1" TAIL ";\n\t}\n" \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]) \
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(scale_d) \
        : "memory")

// The same with A in shared memory too: D[64 x N] (+)= A[64 x K, descriptor desc_a] * B[K x N, descriptor desc_b], for
// the 16-bit types (TYPE "bf16" or "f16", K = 16), neither operand transposed.  Operands d (float[N / 2]), desc_a,
// desc_b, scale_d.
#define B2P_WGMMA_M64N128_SS(TYPE) \
    asm volatile( \
        "{\n\t.reg .pred p;\n\t" \
        "setp.ne.b32 p, %66, 0;\n\t" \
        "wgmma.mma_async.sync.aligned.m64n128k16.f32." TYPE "." TYPE " " \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, " \
        "%64, %65, p, 1, 1, 0, 0;\n\t}\n" \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]) \
        : "l"(desc_a), "l"(desc_b), "r"(scale_d) \
        : "memory")

#define B2P_WGMMA_M64N64_SS(TYPE) \
    asm volatile( \
        "{\n\t.reg .pred p;\n\t" \
        "setp.ne.b32 p, %34, 0;\n\t" \
        "wgmma.mma_async.sync.aligned.m64n64k16.f32." TYPE "." TYPE " " \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, " \
        "%32, %33, p, 1, 1, 0, 0;\n\t}\n" \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]) \
        : "l"(desc_a), "l"(desc_b), "r"(scale_d) \
        : "memory")

#define B2P_WGMMA_M64N48_SS(TYPE) \
    asm volatile( \
        "{\n\t.reg .pred p;\n\t" \
        "setp.ne.b32 p, %26, 0;\n\t" \
        "wgmma.mma_async.sync.aligned.m64n48k16.f32." TYPE "." TYPE " " \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, " \
        "%24, %25, p, 1, 1, 0, 0;\n\t}\n" \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]) \
        : "l"(desc_a), "l"(desc_b), "r"(scale_d) \
        : "memory")

#define B2P_WGMMA_M64N32_SS(TYPE) \
    asm volatile( \
        "{\n\t.reg .pred p;\n\t" \
        "setp.ne.b32 p, %18, 0;\n\t" \
        "wgmma.mma_async.sync.aligned.m64n32k16.f32." TYPE "." TYPE " " \
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, " \
        "%16, %17, p, 1, 1, 0, 0;\n\t}\n" \
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]) \
        : "l"(desc_a), "l"(desc_b), "r"(scale_d) \
        : "memory")

// ---------------------------------------------------------------- binary16 (fp16 mode)
// Two floats rounded to nearest even on the binary16 grid (subnormals kept, beyond 65504 + half an ulp: +-inf); lo in
// bits 0..15, hi in bits 16..31.
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
    uint32_t r;
    asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));     // cvt puts its first source in the upper half
    return r;
}
// Non-zero iff either half of a binary16 pair is +-inf or NaN: an all-ones exponent field plus 1 carries into the sign
// bit of its half (and no further), any other exponent does not.
__device__ __forceinline__ uint32_t f16x2_nonfinite(uint32_t v) {
    return ((v & 0x7c007c00u) + 0x04000400u) & 0x80008000u;
}

// ---------------------------------------------------------------- fp8 (e4m3)
// As make_sdesc_sw128 for 64-byte rows (64 e4m3) with the 64-byte swizzle: layout type 2.
__device__ __forceinline__ uint64_t make_sdesc_sw64(uint32_t saddr, uint32_t sbo_bytes) {
    uint64_t d = 0;
    d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);
    d |= 1ull << 16;
    d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
    d |= 2ull << 62;
    return d;
}

// e4m3x4 from two bf16x2 registers u (bytes 0, 1) and v (bytes 2, 3), each value multiplied by the power of two s first
// (exact), then rounded to nearest even on the e4m3 grid.
__device__ __forceinline__ uint32_t bf16x4_to_e4m3x4(uint32_t u, uint32_t v, float s) {
    const float u0 = __uint_as_float(u << 16) * s, u1 = __uint_as_float(u & 0xffff0000u) * s;
    const float v0 = __uint_as_float(v << 16) * s, v1 = __uint_as_float(v & 0xffff0000u) * s;
    uint16_t lo, hi;     // cvt puts its first source in the upper byte
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(u1), "f"(u0));
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(v1), "f"(v0));
    uint32_t r;
    asm("mov.b32 %0, {%1, %2};" : "=r"(r) : "h"(lo), "h"(hi));
    return r;
}

}  // namespace b2p
