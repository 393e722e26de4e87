// JPEG decoding kernels (DESIGN.md 2.13), five launches per batch:
//  1. unstuff: one CTA per image compacts its scan - drops fill bytes, the 0x00 after a data 0xFF and the restart
//     markers - with a block-wide scan of the bytes each thread keeps.
//  2. Huffman: parallel decoding by self-synchronisation (Weissenberger & Schmidt, ICPP 2018).  Each thread owns a
//     chunk of kJpegChunkBits bits of one segment and decodes it speculatively from the state the previous chunk's
//     thread reported at the boundary (bit position, coefficient in the block, block in the MCU); the first chunk of a
//     segment starts from the true state.  Rounds repeat until no boundary state changes: chunk k is right after at
//     most k + 1 rounds, and the code usually resynchronises within a few symbols.  A segmented scan of the blocks
//     each chunk began gives every chunk its first block, and a last pass writes the coefficients.  A CTA takes whole
//     segments, in windows of kThreads chunks, carrying the state and block count from one window to the next.
//  3. DC: per (image, component), the DC differences are prefix-summed in decode order, restarting at each restart
//     interval (a segmented scan in 32-bit ints, stored as 16-bit coefficients as jdhuff.c does).
//  4. IDCT: one thread per 8 x 8 block into the component's sample plane.
//  5. colour: one thread per output pixel - upsampling, YCbCr -> BGR and orientation - into the packed output.
// Progressive images (DESIGN.md 2.18) are unstuffed per scan by the same kernel, skip steps 2 and 3 (the DC kernel's
// prefix sums run before their coefficients are written, over zeros) and are decoded by jpeg_prog_kernel between
// steps 3 and 4: one CTA per image walks its scans in stream order, each scan's restart segments spread over the
// threads, each segment decoded serially by jdphuff.c's loop (refinement scans consume bits by the coefficients of
// earlier scans, so they cannot be self-synchronised as the Huffman kernel's chunks are).  Launches whose grid would be
// empty (no baseline image) are skipped.
#include "jpeg.cuh"

namespace b2p {
namespace {

constexpr int kThreads = 256;
constexpr int kUnstuffBytes = 16;       // bytes per thread and tile of the unstuffing

// Inclusive sum over the CTA (kThreads threads); every thread must call it.
template <class T> __device__ T block_inclusive_sum(T v, T* warp_tot, T* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const T u = __shfl_up_sync(0xffffffffu, v, o);
        if (lane >= o) v += u;
    }
    if (lane == 31) warp_tot[warp] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        T run = 0;
        for (int w = 0; w < kThreads / 32; ++w) {
            const T t = warp_tot[w];
            warp_tot[w] = run;
            run += t;
        }
        *total = run;
    }
    __syncthreads();
    v += warp_tot[warp];
    __syncthreads();
    return v;
}

// Inclusive segmented sum over the CTA: a segment starts at every thread with head set.
template <class T> __device__ T block_segmented_sum(T v, bool head, T* sv, int* sf) {
    int f = head;
    for (int o = 1; o < kThreads; o <<= 1) {
        sv[threadIdx.x] = v;
        sf[threadIdx.x] = f;
        __syncthreads();
        if ((int)threadIdx.x >= o && !f) {
            v += sv[threadIdx.x - o];
            f = sf[threadIdx.x - o];
        }
        __syncthreads();
    }
    return v;
}

__device__ __forceinline__ bool jp_keep(const unsigned char* raw, long long i, long long beg, long long end) {
    const unsigned char b = raw[i];
    if (b != 0xFF) return !(i > beg && raw[i - 1] == 0xFF);
    return i + 1 < end && raw[i + 1] == 0x00;
}

__global__ void __launch_bounds__(kThreads) jpeg_unstuff_kernel(const JpegUnstuffJob* __restrict__ jobs,
                                                                const unsigned char* __restrict__ raw,
                                                                unsigned char* __restrict__ data) {
    __shared__ long long warp_tot[kThreads / 32], total;
    const JpegUnstuffJob j = jobs[blockIdx.x];
    long long at = j.out;
    for (long long t0 = j.raw_beg; t0 < j.raw_end; t0 += (long long)kThreads * kUnstuffBytes) {
        const long long b0 = t0 + (long long)threadIdx.x * kUnstuffBytes;
        long long kept = 0;
        for (int k = 0; k < kUnstuffBytes; ++k)
            if (b0 + k < j.raw_end) kept += jp_keep(raw, b0 + k, j.raw_beg, j.raw_end);
        const long long incl = block_inclusive_sum(kept, warp_tot, &total);
        long long o = at + incl - kept;
        for (int k = 0; k < kUnstuffBytes; ++k)
            if (b0 + k < j.raw_end && jp_keep(raw, b0 + k, j.raw_beg, j.raw_end)) data[o++] = raw[b0 + k];
        at += total;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kThreads) jpeg_huff_kernel(const JpegImage* __restrict__ ims,
                                                             const JpegSeg* __restrict__ segs,
                                                             const int* __restrict__ chunk_seg,
                                                             const long long* __restrict__ work,
                                                             const unsigned char* __restrict__ data, short* coef,
                                                             unsigned* status) {
    __shared__ JpegState exits[kThreads];
    __shared__ long long sv[kThreads];
    __shared__ int sf[kThreads];
    __shared__ JpegState carry;
    __shared__ long long carry_g;
    const long long c0 = work[blockIdx.x], c1 = work[blockIdx.x + 1];
    const int t = threadIdx.x;
    for (long long w0 = c0; w0 < c1; w0 += kThreads) {
        const long long c = w0 + t;
        const bool active = c < c1;
        JpegSeg sg{};
        long long cb = 0, ce = 0;
        bool head = true, last = false;
        if (active) {
            sg = segs[chunk_seg[c]];
            const long long bits = (sg.end - sg.beg) * 8, q = c - sg.chunk0;
            const long long chunks = bits > 0 ? (bits + kJpegChunkBits - 1) / kJpegChunkBits : 1;
            cb = q * kJpegChunkBits;
            ce = cb + kJpegChunkBits < bits ? cb + kJpegChunkBits : bits;
            head = q == 0;
            last = q == chunks - 1;
        }
        const JpegImage& im = ims[sg.img];
        const unsigned char* d = data + sg.beg;
        const long long nbytes = sg.end - sg.beg;
        JpegState entry = head ? JpegState{0, 0, 0} : (t == 0 ? carry : JpegState{cb, 0, 0});
        JpegState used{-1, 0, 0};
        int blocks = 0;
        for (;;) {
            if (active && !jp_same(entry, used)) {
                JpegState s = entry;
                blocks = jp_sync_chunk(im, s, d, nbytes, ce);
                exits[t] = s;
                used = entry;
            }
            __syncthreads();
            JpegState ne = entry;
            if (active && !head && t > 0) ne = exits[t - 1];
            const bool changed = !jp_same(ne, entry);
            entry = ne;
            if (!__syncthreads_or(changed)) break;
        }
        // first block of each chunk: segmented scan of the blocks the chunks began (thread 0 continues the carry)
        const long long v = (active ? blocks : 0) + (t == 0 && !head ? carry_g : 0);
        const long long incl = block_segmented_sum(v, head || t == 0, sv, sf);
        const long long g = incl - (active ? blocks : 0) - (entry.k > 0 ? 1 : 0);
        if (active) {
            const unsigned bad = jp_write_chunk(im, sg, entry, g, ce, last, d, coef);
            if (bad) atomicOr(status + sg.img, bad);
        }
        if (t == kThreads - 1) {
            carry = exits[t];
            carry_g = incl;
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kThreads) jpeg_dc_kernel(const JpegImage* __restrict__ ims, short* coef) {
    __shared__ unsigned sv[kThreads];
    __shared__ int sf[kThreads];
    __shared__ unsigned carry;
    const JpegImage& im = ims[blockIdx.x];
    const int c = blockIdx.y;
    if (c >= im.ncomp) return;
    const long long total = (long long)im.comp[c].bw * im.comp[c].bh;
    for (long long t0 = 0; t0 < total; t0 += kThreads) {
        const long long i = t0 + threadIdx.x;
        bool head = true;
        short* blk = nullptr;
        unsigned v = 0;
        if (i < total) {
            blk = jp_dc_block(im, coef, c, i, &head);
            v = (unsigned)(int)blk[0];
        }
        if (threadIdx.x == 0 && !head) v += carry;
        const unsigned incl = block_segmented_sum(v, head || threadIdx.x == 0, sv, sf);
        if (blk) blk[0] = (short)(int)incl;
        if (threadIdx.x == kThreads - 1) carry = incl;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kThreads) jpeg_idct_kernel(const JpegImage* __restrict__ ims,
                                                             const short* __restrict__ coef,
                                                             unsigned char* __restrict__ planes) {
    const JpegImage& im = ims[blockIdx.y];
    const int c = blockIdx.z;
    if (c >= im.ncomp) return;
    const JpegComp& cp = im.comp[c];
    const long long total = (long long)cp.bw * cp.bh, pitch = (long long)cp.bw * 8;
    for (long long b = blockIdx.x * (long long)kThreads + threadIdx.x; b < total; b += (long long)gridDim.x * kThreads) {
        const long long by = b / cp.bw, bx = b - by * cp.bw;
        jp_idct_block(coef + (cp.coef + b) * 64, im.qt[c], planes + cp.plane + by * 8 * pitch + bx * 8, pitch);
    }
}

__global__ void __launch_bounds__(kThreads) jpeg_color_kernel(const JpegImage* __restrict__ ims,
                                                              const unsigned char* __restrict__ planes,
                                                              unsigned char* __restrict__ out) {
    const JpegImage& im = ims[blockIdx.y];
    const long long px = (long long)im.oh * im.ow;
    unsigned char* dst = out + im.out;
    for (long long p = blockIdx.x * (long long)kThreads + threadIdx.x; p < px; p += (long long)gridDim.x * kThreads) {
        const int y = (int)(p / im.ow), x = (int)(p - (long long)y * im.ow);
        unsigned char bgr[3];
        jpeg_px(im, planes, y, x, bgr);
        dst[3 * p + 0] = bgr[0];
        dst[3 * p + 1] = bgr[1];
        dst[3 * p + 2] = bgr[2];
    }
}

constexpr int kProgThreads = 128;

__global__ void __launch_bounds__(kProgThreads) jpeg_prog_kernel(const JpegImage* __restrict__ ims,
                                                                 const JpegProgImage* __restrict__ prog,
                                                                 const JpegScan* __restrict__ scans,
                                                                 const JpegSeg* __restrict__ segs,
                                                                 const unsigned char* __restrict__ data, short* coef,
                                                                 unsigned* status) {
    const JpegProgImage pi = prog[blockIdx.x];
    const JpegImage& im = ims[pi.img];
    unsigned bad = 0;
    for (int s = pi.scan0; s < pi.scan0 + pi.nscans; ++s) {
        const JpegScan& sc = scans[s];
        for (int k = threadIdx.x; k < sc.nseg; k += kProgThreads) bad |= jp_prog_segment(im, sc, segs[sc.seg0 + k], data, coef);
        __syncthreads();
    }
    if (bad) atomicOr(status + pi.img, bad);
}

unsigned grid_for(long long items, int n) {
    long long bx = (items + kThreads - 1) / kThreads;
    const long long cap = (132LL * 8 + n - 1) / n;      // about one wave of 8 blocks per SM over the whole batch
    if (bx > cap) bx = cap;
    return (unsigned)(bx < 1 ? 1 : bx);
}

}  // namespace

int jpeg_decode_launches(const JpegBatch& b) {
    return b.nprog == 0 ? kJpegLaunches : b.nwork > 0 ? kJpegProgLaunches : kJpegProgOnlyLaunches;
}

cudaError_t jpeg_decode_launch(const JpegBatch& b, cudaStream_t s) {
    if (b.n < 1 || b.n > 65535 || b.nwork < (b.nprog ? 0 : 1) || b.max_px < 1 || b.max_blocks < 1 || b.nprog < 0 ||
        b.nprog > b.n || b.njobs < 1)
        return cudaErrorInvalidValue;
    jpeg_unstuff_kernel<<<b.njobs, kThreads, 0, s>>>(b.jobs, b.raw, b.data);
    if (b.nwork > 0) {
        jpeg_huff_kernel<<<b.nwork, kThreads, 0, s>>>(b.ims, b.segs, b.chunk_seg, b.work, b.data, b.coef, b.status);
        jpeg_dc_kernel<<<dim3(b.n, 3), kThreads, 0, s>>>(b.ims, b.coef);
    }
    if (b.nprog > 0)
        jpeg_prog_kernel<<<b.nprog, kProgThreads, 0, s>>>(b.ims, b.prog, b.scans, b.pseg, b.data, b.coef, b.status);
    jpeg_idct_kernel<<<dim3(grid_for(b.max_blocks, 3 * b.n), b.n, 3), kThreads, 0, s>>>(b.ims, b.coef, b.planes);
    jpeg_color_kernel<<<dim3(grid_for(b.max_px, b.n), b.n), kThreads, 0, s>>>(b.ims, b.planes, b.out);
    return cudaGetLastError();
}

}  // namespace b2p
