// PNG decoding kernels (DESIGN.md 2.17), four launches per batch:
//  1. gather: one warp per IDAT chunk copies its data to its place in the image's zlib stream and checks the chunk's
//     CRC-32 (each lane a slice, joined by crc32_combine).
//  2. inflate: one warp per image.  Lane 0 decodes Huffman symbols into a buffer of tokens in shared memory; the warp
//     then writes them: literals and stored runs at once, each match in order as out[p + j] = out[p - d + (j mod d)]
//     (correct for overlapping copies: [p - d, p) exists already).  The Adler-32 of the output is summed by the warp.
//  3. unfilter: one warp per image, row after row of every pass: Up over all lanes, Sub, Average and Paeth along the
//     row with one lane per byte of the pixel.
//  4. colour: one thread per output pixel - Adam7 position, unpacking, palette, 16 -> 8 bits, gray -> BGR, alpha
//     dropped and orientation - into the packed output.
#include "png.cuh"

namespace b2p {
namespace {

constexpr int kThreads = 256;
constexpr unsigned kFull = 0xffffffffu;

__global__ void __launch_bounds__(32) png_gather_kernel(const PngDecImage* __restrict__ ims,
                                                        const PngIdat* __restrict__ idat,
                                                        const unsigned char* __restrict__ raw,
                                                        unsigned char* __restrict__ zlib, unsigned* status) {
    __shared__ unsigned table[256];
    const int lane = threadIdx.x;
    for (int i = lane; i < 256; i += 32) table[i] = png_crc_entry((unsigned)i);
    __syncwarp();
    const PngIdat c = idat[blockIdx.x];
    const unsigned char* src = raw + c.src;      // chunk type, then data
    unsigned char* dst = zlib + ims[c.img].z0 + c.dst;
    for (long long i = lane; i < c.len; i += 32) dst[i] = src[4 + i];
    const long long total = c.len + 4, per = (total + 31) / 32;
    const long long b0 = lane * per < total ? lane * per : total, b1 = b0 + per < total ? b0 + per : total;
    unsigned crc = 0xFFFFFFFFu;
    for (long long i = b0; i < b1; ++i) crc = table[(crc ^ src[i]) & 0xFFu] ^ (crc >> 8);
    crc ^= 0xFFFFFFFFu;
    long long len = b1 - b0;
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned oc = __shfl_down_sync(kFull, crc, o);
        const long long ol = __shfl_down_sync(kFull, len, o);
        if ((lane & (2 * o - 1)) == 0) {
            crc = png_crc_combine(crc, oc, ol);
            len += ol;
        }
    }
    if (lane == 0 && crc != c.crc) atomicOr(status + c.img, kPngBadCrc);
}

__global__ void __launch_bounds__(32) png_inflate_kernel(const PngDecImage* __restrict__ ims,
                                                         const PngIdat* __restrict__ idat,
                                                         const unsigned char* __restrict__ zlib,
                                                         unsigned char* __restrict__ rows, unsigned* status) {
    __shared__ PngInflate s;
    __shared__ PngToken tok[kPngTokens];
    __shared__ int nt;
    const PngDecImage& im = ims[blockIdx.x];
    const unsigned char* z = zlib + im.z0;
    unsigned char* out = rows + im.f0;
    const int lane = threadIdx.x;
    if (lane == 0) pn_zlib_header(s, z, im.zlen);
    __syncwarp();
    for (;;) {
        if (lane == 0) nt = s.state == kPnDone ? -1 : pn_inflate_round(s, z, im.zlen, im.flen, idat + im.idat0, im.nidat, tok);
        __syncwarp();
        const int m = nt;
        if (m < 0) break;
        for (int t = 0; t < m; ++t) {
            const PngToken k = tok[t];
            if (k.kind == 0 && lane == (t & 31)) out[k.pos] = (unsigned char)k.src;
            if (k.kind == 2)
                for (int j = lane; j < k.len; j += 32) pn_token_byte(k, j, z, out);
        }
        __syncwarp();
        for (int t = 0; t < m; ++t) {
            const PngToken k = tok[t];
            if (k.kind != 1) continue;
            for (int j = lane; j < k.len; j += 32) pn_token_byte(k, j, z, out);
            __syncwarp();
        }
        __syncwarp();      // every lane is done with tok before lane 0 refills it
    }
    unsigned long long a = 0, b = 0;
    const bool check = s.ended && s.status == 0;
    if (check) {
        const long long n = im.flen, per = (n + 31) / 32;
        const long long b0 = lane * per < n ? lane * per : n, b1 = b0 + per < n ? b0 + per : n;
        for (long long p = b0; p < b1; ++p) {
            a += out[p];
            b += (unsigned long long)((n - p) % kPngAdlerMod) * out[p];
            if (((p - b0) & 4095) == 4095) {
                a %= kPngAdlerMod;
                b %= kPngAdlerMod;
            }
        }
        a %= kPngAdlerMod;
        b %= kPngAdlerMod;
        for (int o = 16; o > 0; o >>= 1) {
            a += __shfl_down_sync(kFull, a, o);
            b += __shfl_down_sync(kFull, b, o);
        }
    }
    if (lane == 0) {
        unsigned st = s.status;
        if (check && png_adler(im.flen, a % kPngAdlerMod, b % kPngAdlerMod) != s.adler) st |= kPngBadAdler;
        if (st) atomicOr(status + blockIdx.x, st);
    }
}

__global__ void __launch_bounds__(32) png_unfilter_kernel(const PngDecImage* __restrict__ ims,
                                                          unsigned char* __restrict__ rows, unsigned* status) {
    const PngDecImage& im = ims[blockIdx.x];
    const int lane = threadIdx.x;
    unsigned char* at = rows + im.f0;
    for (int p = 0; p < (im.interlace ? 7 : 1); ++p) {
        int ph, pw;
        pn_pass(im.interlace, p, im.h, im.w, &ph, &pw);
        const long long rb = pn_rowbytes(im, pw);
        for (int r = 0; r < ph; ++r, at += rb + 1) {
            const int type = at[0];
            if (type > 4) {
                if (lane == 0) atomicOr(status + blockIdx.x, kPngBadFilter);
                continue;
            }
            if (type) pn_unfilter_lane(at + 1, r ? at - rb : nullptr, rb, im.bpp, type, lane, 32);
            __syncwarp();
        }
    }
}

__global__ void __launch_bounds__(kThreads) png_color_kernel(const PngDecImage* __restrict__ ims,
                                                             const unsigned char* __restrict__ rows,
                                                             unsigned char* __restrict__ out) {
    const PngDecImage& im = ims[blockIdx.y];
    const long long px = (long long)im.oh * im.ow;
    unsigned char* dst = out + im.out;
    for (long long p = blockIdx.x * (long long)kThreads + threadIdx.x; p < px; p += (long long)gridDim.x * kThreads) {
        const int y = (int)(p / im.ow), x = (int)(p - (long long)y * im.ow);
        unsigned char bgr[3];
        png_px(im, rows + im.f0, y, x, bgr);
        dst[3 * p + 0] = bgr[0];
        dst[3 * p + 1] = bgr[1];
        dst[3 * p + 2] = bgr[2];
    }
}

unsigned grid_for(long long items, int n) {
    long long bx = (items + kThreads - 1) / kThreads;
    const long long cap = (132LL * 8 + n - 1) / n;      // about one wave of 8 blocks per SM over the whole batch
    if (bx > cap) bx = cap;
    return (unsigned)(bx < 1 ? 1 : bx);
}

}  // namespace

cudaError_t png_decode_launch(const PngDecBatch& b, cudaStream_t s) {
    if (b.n < 1 || b.n > 65535 || b.nidat < 1 || b.max_px < 1) return cudaErrorInvalidValue;
    png_gather_kernel<<<b.nidat, 32, 0, s>>>(b.ims, b.idat, b.raw, b.zlib, b.status);
    png_inflate_kernel<<<b.n, 32, 0, s>>>(b.ims, b.idat, b.zlib, b.rows, b.status);
    png_unfilter_kernel<<<b.n, 32, 0, s>>>(b.ims, b.rows, b.status);
    png_color_kernel<<<dim3(grid_for(b.max_px, b.n), b.n), kThreads, 0, s>>>(b.ims, b.rows, b.out);
    return cudaGetLastError();
}

}  // namespace b2p
