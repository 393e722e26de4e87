// PNG encoding kernels (DESIGN.md 2.15), nine launches per batch in two phases:
//  1. filter: one thread per 8 filtered bytes of a 2 KB tile - the bytes, straight from the BGR frame, the tile's first
//     and last run start, and the Adler-32 sums (atomics per warp).
//  2. runs: one CTA per image scans the tiles: the last run start before each tile and the first after it.
//  3. count: one thread per 8 bytes finds each byte's run (block-wide scans of the run starts, the tile's neighbours
//     from step 2) and the symbol deflate_rle starts there, if any: the tile's symbol count.
//  4. symbol scan: one CTA per image scans the tile counts into symbol offsets; symbols and blocks of the image.
//  5. symbols: as 3, and writes each symbol at its place.
//  6. trees: one CTA per deflate block counts its symbols in shared memory; one thread builds zlib's trees and picks
//     the block type.
//  7. layout: one thread per image places its blocks (a stored block starts on a byte) and sizes the file.
// The host reads the sizes back and sizes the deflate words and the output exactly.
//  8. pack: one CTA per block: one thread writes the block header and tree description, each thread a group of its
//     symbols (or stored bytes) at offsets from a block-wide scan; words a group fills alone are stored, its first and
//     last word ORed atomically.
//  9. write: one warp per IDAT chunk behind the images before: length, type, the zlib bytes and the CRC (a CRC per
//     lane, combined); the first CTA of an image writes the signature, IHDR and IEND.
#include <climits>
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include "png_enc.cuh"

namespace b2p {
namespace {

constexpr int kThreads = 256;
constexpr int kPer = kPngTile / kThreads;   // filtered bytes per thread
constexpr int kImageThreads = 512;          // the per-image scans
constexpr int kWarps = kThreads / 32;
static_assert(kPer == 8, "one 64-bit word of filtered bytes per thread");

struct MaxOp {
    __device__ long long operator()(long long a, long long b) const { return a > b ? a : b; }
};
struct MinOp {
    __device__ long long operator()(long long a, long long b) const { return a < b ? a : b; }
};

__global__ void __launch_bounds__(kThreads) png_enc_filter_kernel(const PngImage* __restrict__ ims,
                                                                  const unsigned char* __restrict__ frames,
                                                                  unsigned char* __restrict__ filt,
                                                                  long long* __restrict__ tfirst,
                                                                  long long* __restrict__ tlast, PngImageOut* outs) {
    using Reduce = cub::BlockReduce<long long, kThreads>;
    __shared__ typename Reduce::TempStorage tmp;
    const PngImage& im = ims[blockIdx.y];
    const unsigned char* frame = frames + im.src;
    unsigned long long a = 0, b = 0;
    for (long long t = blockIdx.x; t < im.tiles; t += gridDim.x) {
        const long long p0 = t * kPngTile + threadIdx.x * kPer;
        long long first = LLONG_MAX, last = -1;
        unsigned prev = p0 > 0 && p0 < im.n ? png_filtered(frame, im.w, p0 - 1) : 0u;
        unsigned long long word = 0;
#pragma unroll
        for (int k = 0; k < kPer; ++k) {
            const long long p = p0 + k;
            if (p >= im.n) break;
            const unsigned v = png_filtered(frame, im.w, p);
            word |= (unsigned long long)v << (8 * k);
            if (p == 0 || v != prev) {
                if (first == LLONG_MAX) first = p;
                last = p;
            }
            prev = v;
            a += v;
            b += (unsigned long long)((im.n - p) % kPngAdlerMod) * v;
        }
        if (p0 + kPer <= im.n) {
            *reinterpret_cast<unsigned long long*>(filt + im.f0 + p0) = word;
        } else {
            for (int k = 0; p0 + k < im.n; ++k) filt[im.f0 + p0 + k] = (unsigned char)(word >> (8 * k));
        }
        first = Reduce(tmp).Reduce(first, MinOp());
        __syncthreads();
        last = Reduce(tmp).Reduce(last, MaxOp());
        __syncthreads();
        if (threadIdx.x == 0) {
            tfirst[im.tile0 + t] = first;
            tlast[im.tile0 + t] = last;
        }
    }
    a %= kPngAdlerMod;
    b %= kPngAdlerMod;
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_down_sync(0xffffffffu, a, o);
        b += __shfl_down_sync(0xffffffffu, b, o);
    }
    if ((threadIdx.x & 31) == 0 && (a | b)) {
        atomicAdd(&outs[blockIdx.y].adler[0], a);
        atomicAdd(&outs[blockIdx.y].adler[1], b);
    }
}

__global__ void __launch_bounds__(kImageThreads) png_enc_runs_kernel(const PngImage* __restrict__ ims,
                                                                     const long long* __restrict__ tfirst,
                                                                     const long long* __restrict__ tlast,
                                                                     long long* __restrict__ tstart,
                                                                     long long* __restrict__ tend) {
    using Scan = cub::BlockScan<long long, kImageThreads>;
    __shared__ typename Scan::TempStorage tmp;
    const PngImage& im = ims[blockIdx.x];
    long long carry = -1;
    for (long long t0 = 0; t0 < im.tiles; t0 += kImageThreads) {
        const long long t = t0 + threadIdx.x;
        long long excl, agg;
        Scan(tmp).ExclusiveScan(t < im.tiles ? tlast[im.tile0 + t] : -1LL, excl, carry, MaxOp(), agg);
        if (t < im.tiles) tstart[im.tile0 + t] = excl;
        carry = carry > agg ? carry : agg;
        __syncthreads();
    }
    carry = im.n;
    for (long long t0 = 0; t0 < im.tiles; t0 += kImageThreads) {     // from the last tile down
        const long long t = im.tiles - 1 - (t0 + threadIdx.x);
        long long excl, agg;
        Scan(tmp).ExclusiveScan(t >= 0 ? tfirst[im.tile0 + t] : LLONG_MAX, excl, carry, MinOp(), agg);
        if (t >= 0) tend[im.tile0 + t] = excl;
        carry = carry < agg ? carry : agg;
        __syncthreads();
    }
}

// Steps 3 and 5 on tile t: each byte's run from the run starts (own bytes, then the threads before and after, then the
// tiles before and after), the symbols starting at the thread's bytes; counts them (kWrite false: the tile's count
// to tcount) or writes them at the tile's offset.
template <bool kWrite>
__device__ __forceinline__ void png_tile_symbols(const PngImage& im, long long t, const unsigned char* __restrict__ filt,
                                                 const PngBatch& B, long long* lo, long long* hi) {
    using Scan = cub::BlockScan<int, kThreads>;
    __shared__ typename Scan::TempStorage tmp;
    const int tid = threadIdx.x;
    const long long p0 = t * kPngTile + tid * kPer;
    const unsigned char* f = filt + im.f0;
    unsigned v[kPer];
    bool start[kPer];
    long long last = -1, first = LLONG_MAX;
    unsigned prev = p0 > 0 && p0 < im.n ? f[p0 - 1] : 0u;
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
        const long long p = p0 + k;
        v[k] = p < im.n ? f[p] : 0u;
        start[k] = p < im.n && (p == 0 || v[k] != prev);
        prev = v[k];
        if (start[k]) {
            if (first == LLONG_MAX) first = p;
            last = p;
        }
    }
    lo[tid] = last;
    hi[tid] = first;
    __syncthreads();
    for (int d = 1; d < kThreads; d <<= 1) {      // inclusive max-scan forward, min-scan backward
        const long long x = tid >= d ? lo[tid - d] : -1, y = tid + d < kThreads ? hi[tid + d] : LLONG_MAX;
        __syncthreads();
        if (x > lo[tid]) lo[tid] = x;
        if (y < hi[tid]) hi[tid] = y;
        __syncthreads();
    }
    long long s = B.tstart[im.tile0 + t], e = B.tend[im.tile0 + t];
    if (tid > 0 && lo[tid - 1] > s) s = lo[tid - 1];
    if (tid + 1 < kThreads && hi[tid + 1] < e) e = hi[tid + 1];
    long long ends[kPer];
#pragma unroll
    for (int k = kPer - 1; k >= 0; --k) {
        ends[k] = e;
        if (start[k]) e = p0 + k;
    }
    int sym[kPer], cnt = 0;
#pragma unroll
    for (int k = 0; k < kPer; ++k) {
        const long long p = p0 + k;
        if (start[k]) s = p;
        sym[k] = p < im.n ? png_symbol_at(p, s, ends[k], v[k]) : -1;
        cnt += sym[k] >= 0;
    }
    int excl, total;
    Scan(tmp).ExclusiveSum(cnt, excl, total);
    if (!kWrite) {
        if (tid == 0) B.tcount[im.tile0 + t] = total;
    } else {
        unsigned short* dst = B.sym + im.f0 + B.tbase[im.tile0 + t] + excl;
#pragma unroll
        for (int k = 0; k < kPer; ++k)
            if (sym[k] >= 0) *dst++ = (unsigned short)sym[k];
    }
    __syncthreads();
}

__global__ void __launch_bounds__(kThreads) png_enc_count_kernel(const PngBatch B) {
    __shared__ long long lo[kThreads], hi[kThreads];
    const PngImage& im = B.ims[blockIdx.y];
    for (long long t = blockIdx.x; t < im.tiles; t += gridDim.x) png_tile_symbols<false>(im, t, B.filt, B, lo, hi);
}

__global__ void __launch_bounds__(kThreads) png_enc_symbols_kernel(const PngBatch B) {
    __shared__ long long lo[kThreads], hi[kThreads];
    const PngImage& im = B.ims[blockIdx.y];
    for (long long t = blockIdx.x; t < im.tiles; t += gridDim.x) png_tile_symbols<true>(im, t, B.filt, B, lo, hi);
}

__global__ void __launch_bounds__(kImageThreads) png_enc_symscan_kernel(const PngImage* __restrict__ ims,
                                                                        const long long* __restrict__ tcount,
                                                                        long long* __restrict__ tbase,
                                                                        PngImageOut* __restrict__ outs) {
    using Scan = cub::BlockScan<long long, kImageThreads>;
    __shared__ typename Scan::TempStorage tmp;
    const PngImage& im = ims[blockIdx.x];
    long long run = 0;
    for (long long t0 = 0; t0 < im.tiles; t0 += kImageThreads) {
        const long long t = t0 + threadIdx.x;
        long long excl, total;
        Scan(tmp).ExclusiveSum(t < im.tiles ? tcount[im.tile0 + t] : 0LL, excl, total);
        if (t < im.tiles) tbase[im.tile0 + t] = run + excl;
        run += total;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        outs[blockIdx.x].symbols = run;
        outs[blockIdx.x].blocks = (int)png_blocks(run);
    }
}

__global__ void __launch_bounds__(kThreads) png_enc_tree_kernel(const PngImage* __restrict__ ims,
                                                                const unsigned short* __restrict__ sym,
                                                                const PngImageOut* __restrict__ outs,
                                                                PngBlock* __restrict__ blocks) {
    __shared__ PngTrees work;
    __shared__ unsigned lfreq[kPngLCodes], nmatch;
    __shared__ unsigned long long bytes;
    const PngImage& im = ims[blockIdx.y];
    const long long nsym = outs[blockIdx.y].symbols;
    const int nb = outs[blockIdx.y].blocks;
    for (int b = blockIdx.x; b < nb; b += gridDim.x) {
        for (int i = threadIdx.x; i < kPngLCodes; i += kThreads) lfreq[i] = 0;
        if (threadIdx.x == 0) nmatch = 0, bytes = 0;
        __syncthreads();
        const long long s0 = (long long)b * kPngBlockSymbols, s1 = b + 1 < nb ? s0 + kPngBlockSymbols : nsym;
        unsigned long long by = 0;
        for (long long i = s0 + threadIdx.x; i < s1; i += kThreads) {
            const int s = sym[im.f0 + i];
            by += png_sym_bytes(s);
            if (s < 256) {
                atomicAdd(&lfreq[s], 1u);
            } else {
                atomicAdd(&lfreq[257 + png_len_code(s - 256)], 1u);
                atomicAdd(&nmatch, 1u);
            }
        }
        atomicAdd(&bytes, by);
        __syncthreads();
        if (threadIdx.x == 0) {
            lfreq[256] = 1;
            PngBlock& B = blocks[im.blk0 + b];
            B.sym0 = s0;
            B.nsym = s1 - s0;
            png_block_trees(lfreq, nmatch, (long long)bytes, b + 1 == nb, work, B);
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(128) png_enc_layout_kernel(const PngImage* __restrict__ ims, int n,
                                                             PngBlock* __restrict__ blocks, PngImageOut* __restrict__ outs) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    PngBlock* blk = blocks + ims[i].blk0;
    long long off = 0, byte0 = 0;
    for (int k = 0; k < outs[i].blocks; ++k) {
        blk[k].off = off;
        blk[k].byte0 = byte0;
        off = png_block_end(blk[k], off);
        byte0 += blk[k].bytes;
    }
    const long long z = png_zlib_bytes(off);
    outs[i].bits = off;
    outs[i].size = png_file_bytes(z);
    outs[i].chunks = (int)png_chunks(z);
}

__global__ void __launch_bounds__(kThreads) png_enc_pack_kernel(const PngImage* __restrict__ ims,
                                                                const unsigned char* __restrict__ filt,
                                                                const unsigned short* __restrict__ sym,
                                                                const PngBlock* __restrict__ blocks,
                                                                const PngImageOut* __restrict__ outs,
                                                                const long long* __restrict__ wbase, unsigned* words) {
    using Scan = cub::BlockScan<long long, kThreads>;
    __shared__ typename Scan::TempStorage tmp;
    const PngImage& im = ims[blockIdx.y];
    unsigned* w = words + wbase[blockIdx.y];
    auto store = [w](long long i, unsigned v) { w[i] = v; };
    auto shared = [w](long long i, unsigned v) { atomicOr(w + i, v); };
    using Writer = PngBitWriter<decltype(store), decltype(shared)>;
    const unsigned short* s = sym + im.f0;
    for (int b = blockIdx.x; b < outs[blockIdx.y].blocks; b += gridDim.x) {
        const PngBlock& B = blocks[im.blk0 + b];
        if (threadIdx.x == 0) {
            Writer head(B.off, store, shared);
            png_put_head(B, B.off, head);
            head.finish();
        }
        if (B.type == kPngStored) {
            const long long at = ((B.off + 3 + 7) & ~7LL) + 32, per = (B.bytes + kThreads - 1) / kThreads;
            const long long i0 = threadIdx.x * per, i1 = i0 + per < B.bytes ? i0 + per : B.bytes;
            Writer wr(at + 8 * i0, store, shared);
            for (long long i = i0; i < i1; ++i) wr(filt[im.f0 + B.byte0 + i], 8);
            if (i0 < i1) wr.finish();
            continue;
        }
        // the symbols and END in groups of `per`
        const long long items = B.nsym + 1, per = (items + kThreads - 1) / kThreads;
        const long long i0 = threadIdx.x * per, i1 = i0 + per < items ? i0 + per : items;
        long long bits = 0;
        for (long long i = i0; i < i1; ++i) bits += i < B.nsym ? png_sym_bits(B, s[B.sym0 + i]) : B.llen[256];
        long long excl;
        Scan(tmp).ExclusiveSum(bits, excl);
        __syncthreads();
        if (i0 >= i1) continue;
        Writer wr(B.off + 3 + B.tree_bits + excl, store, shared);
        for (long long i = i0; i < i1; ++i) {
            if (i < B.nsym) png_put_sym(B, s[B.sym0 + i], wr);
            else wr(B.lcode[256], B.llen[256]);
        }
        wr.finish();
    }
}

__global__ void __launch_bounds__(kThreads) png_enc_write_kernel(const PngImage* __restrict__ ims,
                                                                 const PngImageOut* __restrict__ outs,
                                                                 const long long* __restrict__ wbase,
                                                                 const unsigned* __restrict__ words,
                                                                 unsigned char* __restrict__ out) {
    using Reduce = cub::BlockReduce<long long, kThreads>;
    __shared__ typename Reduce::TempStorage tmp;
    __shared__ long long base;
    __shared__ unsigned table[256], part_crc[kThreads];
    __shared__ int part_len[kThreads];
    const PngImage& im = ims[blockIdx.y];
    const PngImageOut& o = outs[blockIdx.y];
    long long before = 0;
    for (int i = threadIdx.x; i < (int)blockIdx.y; i += kThreads) before += outs[i].size;
    before = Reduce(tmp).Sum(before);
    if (threadIdx.x == 0) base = before;
    table[threadIdx.x] = png_crc_entry(threadIdx.x);
    __syncthreads();
    unsigned char* dst = out + base;
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        png_head(im.h, im.w, dst);
        png_tail(dst + o.size - 12);
    }
    const unsigned* wd = words + wbase[blockIdx.y];
    const long long dbytes = (o.bits + 7) / 8, zbytes = png_zlib_bytes(o.bits);
    const unsigned adler = png_adler(im.n, o.adler[0], o.adler[1]);
    const int lane = threadIdx.x & 31;
    constexpr unsigned kIdat = 0x49444154u;    // "IDAT"
    for (int c = blockIdx.x * kWarps + threadIdx.x / 32; c < o.chunks; c += gridDim.x * kWarps) {
        const long long k0 = (long long)c * kPngChunk;
        const int len = (int)(zbytes - k0 < kPngChunk ? zbytes - k0 : kPngChunk);
        unsigned char* ch = dst + 33 + (long long)c * (kPngChunk + 12);
        if (lane < 4) ch[lane] = (unsigned char)(len >> (24 - 8 * lane));
        else if (lane < 8) ch[lane] = (unsigned char)(kIdat >> (56 - 8 * lane));
        for (int k = lane; k < len; k += 32) ch[8 + k] = (unsigned char)png_zbyte(im.zhdr, wd, dbytes, adler, k0 + k);
        // CRC of the type and data: lane l takes bytes [l seg, (l + 1) seg), lane 0 combines them in order
        const int m = 4 + len, seg = (m + 31) / 32, q0 = min(lane * seg, m), q1 = min(q0 + seg, m);
        unsigned crc = 0xFFFFFFFFu;
        for (int q = q0; q < q1; ++q) {
            const unsigned byte = q < 4 ? (kIdat >> (24 - 8 * q)) & 0xFFu : png_zbyte(im.zhdr, wd, dbytes, adler, k0 + q - 4);
            crc = table[(crc ^ byte) & 0xFFu] ^ (crc >> 8);
        }
        part_crc[threadIdx.x] = crc ^ 0xFFFFFFFFu;
        part_len[threadIdx.x] = q1 - q0;
        __syncwarp();
        if (lane == 0) {
            unsigned total = 0;
            for (int l = 0; l < 32; ++l) total = png_crc_combine(total, part_crc[threadIdx.x + l], part_len[threadIdx.x + l]);
            for (int i = 0; i < 4; ++i) ch[8 + len + i] = (unsigned char)(total >> (24 - 8 * i));
        }
        __syncwarp();
    }
}

unsigned grid_for(long long items, int n) {
    const long long cap = (132LL * 8 + n - 1) / n;      // about one wave of 8 CTAs per SM over the whole batch
    const long long bx = items > cap ? cap : items;
    return (unsigned)(bx < 1 ? 1 : bx);
}

}  // namespace

cudaError_t png_encode_launch(const PngBatch& b, int phase, cudaStream_t s) {
    if (b.n < 1 || b.n > 65535 || b.max_tiles < 1 || phase < 0 || phase > 1) return cudaErrorInvalidValue;
    if (phase == 0) {
        const dim3 tiles(grid_for(b.max_tiles, b.n), b.n), blks(grid_for(b.max_blocks, b.n), b.n);
        png_enc_filter_kernel<<<tiles, kThreads, 0, s>>>(b.ims, b.frames, b.filt, b.tfirst, b.tlast, b.outs);
        png_enc_runs_kernel<<<b.n, kImageThreads, 0, s>>>(b.ims, b.tfirst, b.tlast, b.tstart, b.tend);
        png_enc_count_kernel<<<tiles, kThreads, 0, s>>>(b);
        png_enc_symscan_kernel<<<b.n, kImageThreads, 0, s>>>(b.ims, b.tcount, b.tbase, b.outs);
        png_enc_symbols_kernel<<<tiles, kThreads, 0, s>>>(b);
        png_enc_tree_kernel<<<blks, kThreads, 0, s>>>(b.ims, b.sym, b.outs, b.blocks);
        png_enc_layout_kernel<<<(b.n + 127) / 128, 128, 0, s>>>(b.ims, b.n, b.blocks, b.outs);
    } else {
        const dim3 blks(grid_for(b.max_blocks, b.n), b.n);
        const dim3 chunks(grid_for((b.max_chunks + kWarps - 1) / kWarps, b.n), b.n);
        png_enc_pack_kernel<<<blks, kThreads, 0, s>>>(b.ims, b.filt, b.sym, b.blocks, b.outs, b.wbase, b.words);
        png_enc_write_kernel<<<chunks, kThreads, 0, s>>>(b.ims, b.outs, b.wbase, b.words, b.out);
    }
    return cudaGetLastError();
}

}  // namespace b2p
