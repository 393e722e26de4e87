// JPEG encoding kernels (DESIGN.md 2.14), five launches per batch in three phases:
//  1. coefficients: one thread per 8 x 8 block in scan order - its samples straight from the BGR frame (colour
//     conversion, edge replication and downsampling per sample), the forward DCT, quantisation into zig-zag order, and
//     the length of its AC codes.
//  2. scan: one CTA per image adds each block's DC code length (the predecessor's DC is in the coefficient buffer now)
//     and scans the lengths into bit offsets and the image's bit count.
// The host reads the bit counts back and sizes and zeroes the bit buffers exactly (wbase: each image's first word).
//  3. pack: one thread per block writes its codes at its offset: words it fills alone are stored, its first and last
//     word (shared with its neighbours) are ORed atomically.
//  4. count: one CTA per image counts the 0xFF bytes of its padded data: the stream's size.
// The host reads the sizes back and sizes the output exactly.
//  5. write: one CTA per image finds its place behind the streams before it and writes the header, the data with a
//     0x00 after every 0xFF (a block-wide scan of the bytes each thread's run of kStuffBytes becomes) and EOI.
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include "jpeg_enc.cuh"

namespace b2p {
namespace {

constexpr int kThreads = 256;
constexpr int kImageThreads = 512;      // the per-image kernels
constexpr int kStuffBytes = 8;          // bytes per thread and tile of the stuffing

__global__ void __launch_bounds__(kThreads) jpeg_enc_dct_kernel(const JencImage* __restrict__ ims,
                                                                const JencHuff* __restrict__ huff,
                                                                const unsigned char* __restrict__ frames,
                                                                short* __restrict__ coef, int* __restrict__ acbits) {
    const JencImage& im = ims[blockIdx.y];
    const unsigned char* frame = frames + im.src;
    for (long long g = blockIdx.x * (long long)kThreads + threadIdx.x; g < im.blocks; g += (long long)gridDim.x * kThreads) {
        short zz[64];
        jenc_block_coefs(im, frame, g, zz);
        const int t = im.comp[im.mcu_comp[g % im.bpm]].t;
        acbits[im.blk0 + g] = jenc_codes(zz, false, 0, huff[2 * t], huff[2 * t + 1], JencNoPut{});
        short* dst = coef + (im.blk0 + g) * 64;
#pragma unroll
        for (int k = 0; k < 64; k += 2) *reinterpret_cast<short2*>(dst + k) = make_short2(zz[k], zz[k + 1]);
    }
}

__global__ void __launch_bounds__(kImageThreads) jpeg_enc_scan_kernel(const JencImage* __restrict__ ims,
                                                                      const JencHuff* __restrict__ huff,
                                                                      const short* __restrict__ coef,
                                                                      const int* __restrict__ acbits,
                                                                      long long* __restrict__ off, long long* bits) {
    using Scan = cub::BlockScan<long long, kImageThreads>;
    __shared__ typename Scan::TempStorage tmp;
    const JencImage& im = ims[blockIdx.x];
    const short* c0 = coef + im.blk0 * 64;
    long long run = 0;
    for (long long t0 = 0; t0 < im.blocks; t0 += kImageThreads) {
        const long long g = t0 + threadIdx.x;
        long long v = 0;
        if (g < im.blocks) {
            const long long p = jenc_pred_block(im, g);
            const int t = im.comp[im.mcu_comp[g % im.bpm]].t;
            v = acbits[im.blk0 + g] +
                jenc_codes(c0 + g * 64, true, p < 0 ? 0 : c0[p * 64], huff[2 * t], huff[2 * t + 1], JencNoPut{});
        }
        long long excl, total;
        Scan(tmp).ExclusiveSum(v, excl, total);
        if (g < im.blocks) off[im.blk0 + g] = run + excl;
        run += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) bits[blockIdx.x] = run;
}

__global__ void __launch_bounds__(kThreads) jpeg_enc_pack_kernel(const JencImage* __restrict__ ims,
                                                                 const JencHuff* __restrict__ huff,
                                                                 const short* __restrict__ coef,
                                                                 const long long* __restrict__ off,
                                                                 const long long* __restrict__ wbase, unsigned* words) {
    const JencImage& im = ims[blockIdx.y];
    const short* c0 = coef + im.blk0 * 64;
    unsigned* w = words + wbase[blockIdx.y];
    auto store = [w](long long i, unsigned v) { w[i] = v; };
    auto shared = [w](long long i, unsigned v) { atomicOr(w + i, v); };
    for (long long g = blockIdx.x * (long long)kThreads + threadIdx.x; g < im.blocks; g += (long long)gridDim.x * kThreads) {
        const long long p = jenc_pred_block(im, g);
        const int t = im.comp[im.mcu_comp[g % im.bpm]].t;
        JencBitWriter<decltype(store), decltype(shared)> wr(off[im.blk0 + g], store, shared);
        const short* zz = c0 + g * 64;
        jenc_codes(zz, true, p < 0 ? 0 : c0[p * 64], huff[2 * t], huff[2 * t + 1], [&wr](unsigned b, int l) { wr(b, l); });
        jenc_codes(zz, false, 0, huff[2 * t], huff[2 * t + 1], [&wr](unsigned b, int l) { wr(b, l); });
        wr.finish();
    }
}

__global__ void __launch_bounds__(kImageThreads) jpeg_enc_count_kernel(const JencImage* __restrict__ ims,
                                                                       const long long* __restrict__ wbase,
                                                                       const unsigned* __restrict__ words,
                                                                       const long long* __restrict__ bits,
                                                                       long long* __restrict__ sizes) {
    using Reduce = cub::BlockReduce<long long, kImageThreads>;
    __shared__ typename Reduce::TempStorage tmp;
    const JencImage& im = ims[blockIdx.x];
    const unsigned* w = words + wbase[blockIdx.x];
    const long long nb = bits[blockIdx.x], bytes = jenc_data_bytes(nb);
    long long ff = 0;
    for (long long k = threadIdx.x; k < bytes; k += kImageThreads) ff += jenc_byte(w, nb, k) == 0xFFu;
    const long long total = Reduce(tmp).Sum(ff);
    if (threadIdx.x == 0) sizes[blockIdx.x] = im.hdr_len + bytes + total + 2;
}

__global__ void __launch_bounds__(kImageThreads) jpeg_enc_write_kernel(const JencImage* __restrict__ ims,
                                                                       const long long* __restrict__ wbase,
                                                                       const unsigned* __restrict__ words,
                                                                       const long long* __restrict__ bits,
                                                                       const long long* __restrict__ sizes,
                                                                       unsigned char* __restrict__ out) {
    using Reduce = cub::BlockReduce<long long, kImageThreads>;
    using Scan = cub::BlockScan<long long, kImageThreads>;
    __shared__ union {
        typename Reduce::TempStorage r;
        typename Scan::TempStorage s;
    } tmp;
    __shared__ long long base;
    const JencImage& im = ims[blockIdx.x];
    long long before = 0;
    for (int i = threadIdx.x; i < (int)blockIdx.x; i += kImageThreads) before += sizes[i];
    before = Reduce(tmp.r).Sum(before);
    if (threadIdx.x == 0) base = before;
    __syncthreads();
    unsigned char* dst = out + base;
    for (int k = threadIdx.x; k < im.hdr_len; k += kImageThreads) dst[k] = im.hdr[k];
    const unsigned* w = words + wbase[blockIdx.x];
    const long long nb = bits[blockIdx.x], bytes = jenc_data_bytes(nb);
    long long at = im.hdr_len;
    for (long long t0 = 0; t0 < bytes; t0 += (long long)kImageThreads * kStuffBytes) {
        const long long b0 = t0 + (long long)threadIdx.x * kStuffBytes;
        unsigned long long v = 0;     // byte k in bits 8k .. 8k + 7
        long long len = 0;
#pragma unroll
        for (int k = 0; k < kStuffBytes; ++k)
            if (b0 + k < bytes) {
                const unsigned c = jenc_byte(w, nb, b0 + k);
                v |= (unsigned long long)c << (8 * k);
                len += 1 + (c == 0xFFu);
            }
        long long excl, total;
        Scan(tmp.s).ExclusiveSum(len, excl, total);
        long long o = at + excl;
#pragma unroll
        for (int k = 0; k < kStuffBytes; ++k)
            if (b0 + k < bytes) o += jenc_put_stuffed(dst + o, (unsigned)(v >> (8 * k)) & 0xFFu);
        at += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        dst[at] = 0xFF;
        dst[at + 1] = 0xD9;
    }
}

unsigned grid_for(long long items, int n) {
    long long bx = (items + kThreads - 1) / kThreads;
    const long long cap = (132LL * 8 + n - 1) / n;      // about one wave of 8 blocks per SM over the whole batch
    if (bx > cap) bx = cap;
    return (unsigned)(bx < 1 ? 1 : bx);
}

}  // namespace

cudaError_t jpeg_encode_launch(const JencBatch& b, int phase, cudaStream_t s) {
    if (b.n < 1 || b.n > 65535 || b.max_blocks < 1 || phase < 0 || phase > 2) return cudaErrorInvalidValue;
    const dim3 grid(grid_for(b.max_blocks, b.n), b.n);
    if (phase == 0) {
        jpeg_enc_dct_kernel<<<grid, kThreads, 0, s>>>(b.ims, b.huff, b.frames, b.coef, b.acbits);
        jpeg_enc_scan_kernel<<<b.n, kImageThreads, 0, s>>>(b.ims, b.huff, b.coef, b.acbits, b.off, b.bits);
    } else if (phase == 1) {
        jpeg_enc_pack_kernel<<<grid, kThreads, 0, s>>>(b.ims, b.huff, b.coef, b.off, b.wbase, b.words);
        jpeg_enc_count_kernel<<<b.n, kImageThreads, 0, s>>>(b.ims, b.wbase, b.words, b.bits, b.sizes);
    } else {
        jpeg_enc_write_kernel<<<b.n, kImageThreads, 0, s>>>(b.ims, b.wbase, b.words, b.bits, b.sizes, b.out);
    }
    return cudaGetLastError();
}

}  // namespace b2p
