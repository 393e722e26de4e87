// JPEG encoding, host/device shared core: packed uint8 HWC BGR frames -> baseline JPEG streams, byte for byte
//   cv2.imencode('.jpg', frame, [IMWRITE_JPEG_QUALITY, q, IMWRITE_JPEG_SAMPLING_FACTOR, s])
//   (OpenCV 4.13 with libjpeg-turbo 3.1: jpeg_set_defaults, jpeg_set_quality(q, force_baseline), the standard Huffman
//   tables, no restart interval).  What libjpeg-turbo computes on the path cv2 takes, restated (DESIGN.md 2.14):
//  * the header: SOI, JFIF APP0 (1.01, density units 0, 1:1), one DQT per table (luma, chroma; zig-zag order), SOF0,
//    four DHT segments (DC 0, AC 0, DC 1, AC 1), SOS;
//  * jccolor.c's JCS_EXT_BGR -> YCbCr tables (SCALEBITS 16; Cb / Cr rounded with ONE_HALF - 1);
//  * the edges: samples are replicated right to the block-padded component width (expand_right_edge on the full-size
//    rows), the last row to a whole row group (max v factor rows) before downsampling, and the last downsampled row to
//    the iMCU height (jcprepct.c);
//  * jcsample.c: h2v1 / h2v2 averages with the alternating bias (0, 1 / 1, 2 by output column), int_downsample
//    (rounded mean) for 4:4:0 and 4:1:1;
//  * the accurate integer forward DCT (jfdctint.c, CONST_BITS 13, PASS1_BITS 2) on samples - 128;
//  * quantisation by jcdctmgr.c's reciprocals of q << 3 (the SIMD quantiser cv2 runs on x86-64: (|x| + corr) * recip
//    >> 16, then * scale >> 16, sign restored, which equals (|x| + corr) * recip >> r);
//  * jccoefct.c's dummy blocks of a partial MCU: AC zero, DC that of the block to the left (right edge) or of the
//    MCU's last block of the row above (bottom edge);
//  * jchuff.c's baseline coding: DC differences per component, ZRL for runs of 16 zeros, EOB, 0xFF bytes followed by
//    0x00, and the last byte padded with 1-bits, then EOI.
// The work is split the way the kernels of jpeg_enc.cu run it: per block the coefficients and their AC code length,
// per image a scan of the block lengths (with the DC codes, which need the predecessor's DC), per block the packing of
// its codes into 32-bit words, per image the stuffing.  tests/cuda/jpeg_enc_core_host.cpp runs the same steps.
#pragma once

#include "jpeg_core.h"

namespace b2p {

constexpr int kJencMaxBlocksPerMcu = 6;
constexpr int kJencHeaderCap = 640;                    // the header of a three-component image is 623 bytes
constexpr long long kJencBlockBitsMax = 22 + 63 * 26;  // DC: 11-bit code + 11 bits; 63 AC: 16-bit code + 10 bits

// cv2's IMWRITE_JPEG_SAMPLING_FACTOR values the encoder takes (luma h, v in the top two nibbles, chroma 1 x 1)
constexpr int kJencSampling[5] = {0x221111, 0x211111, 0x121111, 0x411111, 0x111111};

// A Huffman table in encoding form.
struct JencHuff {
    unsigned short code[256];
    unsigned char len[256];
};

struct JencComp {
    int h, v;          // sampling factors
    int fx, fy;        // downsampling: hmax / h, vmax / v
    int wib, hib;      // blocks that hold samples (width_in_blocks, height_in_blocks)
    int rows;          // rows made from the frame's row groups; the iMCU's later rows repeat the last of them
    int t;             // tables: 0 luma, 1 chroma
};

// One image of an encode batch (device-resident descriptor).
struct JencImage {
    int h, w, hmax, vmax, mcux, mcuy, bpm;
    int mcu_comp[kJencMaxBlocksPerMcu], mcu_bx[kJencMaxBlocksPerMcu], mcu_by[kJencMaxBlocksPerMcu];
    JencComp comp[3];
    unsigned short recip[2][64], corr[2][64];   // jcdctmgr.c's divisors of q << 3, natural order
    unsigned char shift[2][64];                 // r - 16
    long long src;                              // byte offset of the BGR frame in the input
    long long blk0, blocks;                     // its blocks in the batch (scan order), and how many
    int hdr_len;
    unsigned char hdr[kJencHeaderCap];
};

// The standard tables of the JPEG specification (K.3), as jpeg_std_huff_table installs them: BITS then HUFFVAL.
constexpr unsigned char kJencDcBits[2][16] = {{0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0},
                                              {0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0}};
constexpr unsigned char kJencAcBits[2][16] = {{0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d},
                                              {0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77}};
constexpr unsigned char kJencAcVals[2][162] = {
    {0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14,
     0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09,
     0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a,
     0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65,
     0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88,
     0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9,
     0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca,
     0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea,
     0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa},
    {0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71, 0x13, 0x22, 0x32,
     0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0, 0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16,
     0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39,
     0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64,
     0x65, 0x66, 0x67, 0x68, 0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86,
     0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
     0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8,
     0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9,
     0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8, 0xf9, 0xfa}};

// ---------------------------------------------------------------------------------------------- samples
// rgb_ycc_convert's fixed-point weights: FIX(0.29900), FIX(0.58700), FIX(0.11400), FIX(0.16874), FIX(0.33126),
// FIX(0.50000), FIX(0.41869), FIX(0.08131) at SCALEBITS 16.
constexpr int kJencScaleBits = 16;
constexpr int kJencFixYR = 19595, kJencFixYG = 38470, kJencFixYB = 7471, kJencFixCbR = 11059, kJencFixCbG = 21709,
              kJencFixHalf = 32768, kJencFixCrG = 27439, kJencFixCrB = 5329;

// Component c (0 Y, 1 Cb, 2 Cr) of one BGR pixel.
B2P_JP_HD int jenc_ycc(const unsigned char* bgr, int c) {
    const int b = bgr[0], g = bgr[1], r = bgr[2];
    const int one_half = 1 << (kJencScaleBits - 1), offset = 128 << kJencScaleBits;
    if (c == 0) return (kJencFixYR * r + kJencFixYG * g + kJencFixYB * b + one_half) >> kJencScaleBits;
    if (c == 1) return (-kJencFixCbR * r - kJencFixCbG * g + kJencFixHalf * b + offset + one_half - 1) >> kJencScaleBits;
    return (kJencFixHalf * r - kJencFixCrG * g - kJencFixCrB * b + offset + one_half - 1) >> kJencScaleBits;
}

// Sample (y, x) of component c's padded plane, from the frame (h x w x 3, pitch 3w).
B2P_JP_HD int jenc_sample(const JencImage& im, const unsigned char* frame, int c, int y, int x) {
    const JencComp& cp = im.comp[c];
    const int cy = y < cp.rows ? y : cp.rows - 1;
    int sum = 0;
    for (int k = 0; k < cp.fy; ++k) {
        const int sy = cy * cp.fy + k < im.h ? cy * cp.fy + k : im.h - 1;
        for (int j = 0; j < cp.fx; ++j) {
            const int sx = x * cp.fx + j < im.w ? x * cp.fx + j : im.w - 1;
            sum += jenc_ycc(frame + 3 * ((long long)sy * im.w + sx), c);
        }
    }
    if (cp.fx == 1 && cp.fy == 1) return sum;                       // fullsize_downsample
    if (cp.fx == 2 && cp.fy == 1) return (sum + (x & 1)) >> 1;      // h2v1_downsample: bias 0, 1, 0, 1, ...
    if (cp.fx == 2 && cp.fy == 2) return (sum + 1 + (x & 1)) >> 2;  // h2v2_downsample: bias 1, 2, 1, 2, ...
    const int n = cp.fx * cp.fy;                                    // int_downsample
    return (sum + n / 2) / n;
}

// ---------------------------------------------------------------------------------------------- transform
constexpr int kFdctConst = 13, kFdctPass1 = 2;
constexpr int kFdct0298631336 = 2446, kFdct0390180644 = 3196, kFdct0541196100 = 4433, kFdct0765366865 = 6270,
              kFdct0899976223 = 7373, kFdct1175875602 = 9633, kFdct1501321110 = 12299, kFdct1847759065 = 15137,
              kFdct1961570560 = 16069, kFdct2053119869 = 16819, kFdct2562915447 = 20995, kFdct3072711026 = 25172;

B2P_JP_HD int jenc_descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }

// One 1-D pass of jpeg_fdct_islow on d[0], d[st], .. d[7 st]; pass 1 scales up by PASS1_BITS, pass 2 removes it.
B2P_JP_HD void jenc_fdct_1d(int* d, int st, bool pass1) {
    const int tmp0 = d[0] + d[7 * st], tmp7 = d[0] - d[7 * st], tmp1 = d[st] + d[6 * st], tmp6 = d[st] - d[6 * st];
    const int tmp2 = d[2 * st] + d[5 * st], tmp5 = d[2 * st] - d[5 * st], tmp3 = d[3 * st] + d[4 * st],
              tmp4 = d[3 * st] - d[4 * st];
    const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    const int sh = pass1 ? kFdctConst - kFdctPass1 : kFdctConst + kFdctPass1;
    d[0] = pass1 ? (tmp10 + tmp11) * (1 << kFdctPass1) : jenc_descale(tmp10 + tmp11, kFdctPass1);
    d[4 * st] = pass1 ? (tmp10 - tmp11) * (1 << kFdctPass1) : jenc_descale(tmp10 - tmp11, kFdctPass1);
    const int z1e = (tmp12 + tmp13) * kFdct0541196100;
    d[2 * st] = jenc_descale(z1e + tmp13 * kFdct0765366865, sh);
    d[6 * st] = jenc_descale(z1e + tmp12 * -kFdct1847759065, sh);
    const int z5 = (tmp4 + tmp5 + tmp6 + tmp7) * kFdct1175875602;
    const int z1 = (tmp4 + tmp7) * -kFdct0899976223, z2 = (tmp5 + tmp6) * -kFdct2562915447;
    const int z3 = (tmp4 + tmp6) * -kFdct1961570560 + z5, z4 = (tmp5 + tmp7) * -kFdct0390180644 + z5;
    d[7 * st] = jenc_descale(tmp4 * kFdct0298631336 + z1 + z3, sh);
    d[5 * st] = jenc_descale(tmp5 * kFdct2053119869 + z2 + z4, sh);
    d[3 * st] = jenc_descale(tmp6 * kFdct3072711026 + z2 + z3, sh);
    d[st] = jenc_descale(tmp7 * kFdct1501321110 + z1 + z4, sh);
}

// jcdctmgr.c's quantisation of one coefficient by the reciprocal of its divisor.
B2P_JP_HD int jenc_quant(int v, unsigned recip, unsigned corr, int shift) {
    const unsigned a = (unsigned)(v < 0 ? -v : v);
    const int q = (int)(((unsigned long long)(a + corr) * recip) >> (shift + 16));
    return v < 0 ? -q : q;
}

// Block (bx, by) of component c and its position in the scan.
B2P_JP_HD void jenc_block_pos(const JencImage& im, long long g, int* c, int* bx, int* by) {
    const long long m = g / im.bpm;
    const int b = (int)(g - m * im.bpm);
    *c = im.mcu_comp[b];
    const JencComp& cp = im.comp[*c];
    *bx = (int)(m % im.mcux) * cp.h + im.mcu_bx[b];
    *by = (int)(m / im.mcux) * cp.v + im.mcu_by[b];
}

// The quantised coefficients of block g (scan order) in zig-zag order.  A dummy block of a partial MCU has zero AC
// and the DC of its source: the last real block of its row (right edge), or the MCU's last block of the last real
// row (bottom edge) - the same block jccoefct.c copies from, whose DC is the sum of its samples - 8 * 8 * 128.
B2P_JP_HD void jenc_block_coefs(const JencImage& im, const unsigned char* frame, long long g, short* zz) {
    int c, bx, by;
    jenc_block_pos(im, g, &c, &bx, &by);
    const JencComp& cp = im.comp[c];
    const unsigned short* recip = im.recip[cp.t];
    const unsigned short* corr = im.corr[cp.t];
    const unsigned char* shift = im.shift[cp.t];
    if (bx >= cp.wib || by >= cp.hib) {
        int sx = cp.wib - 1, sy = by;
        if (by >= cp.hib) {
            sy = cp.hib - 1;
            const int last = (bx / cp.h) * cp.h + cp.h - 1;
            sx = last < cp.wib - 1 ? last : cp.wib - 1;
        }
        int sum = 0;
        for (int y = 0; y < 8; ++y)
            for (int x = 0; x < 8; ++x) sum += jenc_sample(im, frame, c, sy * 8 + y, sx * 8 + x) - 128;
        zz[0] = (short)jenc_quant(sum, recip[0], corr[0], shift[0]);
        for (int k = 1; k < 64; ++k) zz[k] = 0;
        return;
    }
    int d[64];
    for (int y = 0; y < 8; ++y)
        for (int x = 0; x < 8; ++x) d[y * 8 + x] = jenc_sample(im, frame, c, by * 8 + y, bx * 8 + x) - 128;
    for (int r = 0; r < 8; ++r) jenc_fdct_1d(d + r * 8, 1, true);
    for (int k = 0; k < 8; ++k) jenc_fdct_1d(d + k, 8, false);
    for (int k = 0; k < 64; ++k) {
        const int n = jp_natural(k);
        zz[k] = (short)jenc_quant(d[n], recip[n], corr[n], shift[n]);
    }
}

// ---------------------------------------------------------------------------------------------- entropy coding
B2P_JP_HD int jenc_nbits(int v) {
    int a = v < 0 ? -v : v, n = 0;
    while (a) {
        ++n;
        a >>= 1;
    }
    return n;
}

// The value bits of v in nbits bits (a negative v as v - 1, jchuff.c).
B2P_JP_HD unsigned jenc_value(int v, int nbits) {
    return (unsigned)(v < 0 ? v - 1 : v) & ((1u << nbits) - 1u);
}

// The codes of block zz (zig-zag order): the AC part, or with dc set the DC difference from `pred` first; each code is
// handed to put(bits, length).  Returns the bits emitted.
template <class Put>
B2P_JP_HD int jenc_codes(const short* zz, bool dc, int pred, const JencHuff& dct, const JencHuff& act, Put put) {
    int total = 0;
    if (dc) {
        const int diff = zz[0] - pred, nb = jenc_nbits(diff);
        put(dct.code[nb], dct.len[nb]);
        total += dct.len[nb];
        if (nb) put(jenc_value(diff, nb), nb);
        total += nb;
        return total;
    }
    int run = 0;
    for (int k = 1; k < 64; ++k) {
        const int v = zz[k];
        if (v == 0) {
            ++run;
            continue;
        }
        while (run > 15) {
            put(act.code[0xF0], act.len[0xF0]);
            total += act.len[0xF0];
            run -= 16;
        }
        const int nb = jenc_nbits(v), s = (run << 4) + nb;
        put(act.code[s], act.len[s]);
        put(jenc_value(v, nb), nb);
        total += act.len[s] + nb;
        run = 0;
    }
    if (run > 0) {
        put(act.code[0], act.len[0]);
        total += act.len[0];
    }
    return total;
}

struct JencNoPut {
    B2P_JP_HD void operator()(unsigned, int) const {}
};

// The block of the same component coded before block g in the scan (its DC predicts g's), or -1 for the first.
B2P_JP_HD long long jenc_pred_block(const JencImage& im, long long g) {
    const long long m = g / im.bpm;
    const int b = (int)(g - m * im.bpm), c = im.mcu_comp[b];
    if (b > 0 && im.mcu_comp[b - 1] == c) return g - 1;
    if (m == 0) return -1;
    int last = b;
    while (last + 1 < im.bpm && im.mcu_comp[last + 1] == c) ++last;
    return (m - 1) * im.bpm + last;
}

// Bit writer of one block's codes starting at bit `off` of an image's word buffer (32-bit words, most significant bit
// first).  Words the block fills alone are stored; its first and last word may be shared with its neighbours and go
// to store_shared (an OR into a zeroed word).
template <class Store, class StoreShared> struct JencBitWriter {
    unsigned long long acc;
    int n;
    long long wi;
    bool first;
    Store store;
    StoreShared shared;
    B2P_JP_HD JencBitWriter(long long off, Store s, StoreShared ss)
        : acc(0), n((int)(off & 31)), wi(off >> 5), first(true), store(s), shared(ss) {}
    B2P_JP_HD void operator()(unsigned bits, int len) {
        acc = (acc << len) | bits;
        n += len;
        if (n >= 32) {
            const unsigned word = (unsigned)(acc >> (n - 32));
            n -= 32;
            acc &= (1ull << n) - 1ull;
            if (first) shared(wi, word);
            else store(wi, word);
            first = false;
            ++wi;
        }
    }
    B2P_JP_HD void finish() {
        if (n > 0) shared(wi, (unsigned)(acc << (32 - n)));
    }
};

// Byte k of an image's entropy-coded data before stuffing: `bits` bits in words, the last byte padded with 1-bits.
B2P_JP_HD unsigned jenc_byte(const unsigned* words, long long bits, long long k) {
    unsigned b = (words[k >> 2] >> (24 - 8 * (k & 3))) & 0xFFu;
    if (k == (bits - 1) >> 3 && (bits & 7)) b |= 0xFFu >> (bits & 7);
    return b;
}

B2P_JP_HD long long jenc_data_bytes(long long bits) { return (bits + 7) >> 3; }

// Byte b of the data in the stream at dst: 0xFF is followed by a stuffed 0x00.  Returns the bytes written.
B2P_JP_HD int jenc_put_stuffed(unsigned char* dst, unsigned b) {
    dst[0] = (unsigned char)b;
    if (b != 0xFFu) return 1;
    dst[1] = 0;
    return 2;
}

}  // namespace b2p

// ================================================================================================ host-side set-up
#include <cstring>

namespace b2p {

// jpeg_quality_scaling + jpeg_add_quant_table(force_baseline): the quantisation tables, natural order.
inline void jenc_quant_tables(int quality, int qt[2][64]) {
    static const int base[2][64] = {
        {16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
         14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
         49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99},
        {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
         47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
         99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99}};
    const int scale = quality < 50 ? 5000 / quality : 200 - quality * 2;
    for (int t = 0; t < 2; ++t)
        for (int i = 0; i < 64; ++i) {
            long v = ((long)base[t][i] * scale + 50L) / 100L;
            qt[t][i] = (int)(v <= 0 ? 1 : (v > 255 ? 255 : v));
        }
}

// compute_reciprocal(q << 3): the divisor's reciprocal, rounding correction and shift (r - 16).
inline void jenc_reciprocal(int q, unsigned short* recip, unsigned short* corr, unsigned char* shift) {
    const unsigned divisor = (unsigned)q << 3;
    int b = 0;
    while ((divisor >> (b + 1)) != 0) ++b;           // flss(divisor) - 1
    int r = 16 + b;
    unsigned long long fq = (1ull << r) / divisor, fr = (1ull << r) % divisor;
    unsigned c = divisor / 2;
    if (fr == 0) {
        fq >>= 1;
        --r;
    } else if (fr <= divisor / 2u) {
        ++c;
    } else {
        ++fq;
    }
    *recip = (unsigned short)fq;
    *corr = (unsigned short)c;
    *shift = (unsigned char)(r - 16);
}

// jpeg_make_c_derived_tbl for table t (0 DC luma, 1 AC luma, 2 DC chroma, 3 AC chroma).
inline void jenc_huff_table(int t, JencHuff* out) {
    const bool ac = t & 1;
    const int cls = t >> 1;
    const unsigned char* bits = ac ? kJencAcBits[cls] : kJencDcBits[cls];
    memset(out, 0, sizeof(*out));
    int code = 0, k = 0;
    for (int l = 1; l <= 16; ++l) {
        for (int i = 0; i < bits[l - 1]; ++i, ++k, ++code) {
            const int sym = ac ? kJencAcVals[cls][k] : k;
            out->code[sym] = (unsigned short)code;
            out->len[sym] = (unsigned char)l;
        }
        code <<= 1;
    }
}

inline bool jenc_sampling_ok(int s) {
    for (int v : kJencSampling)
        if (v == s) return true;
    return false;
}

// The descriptor of an h x w frame at `quality` (1 .. 100) and sampling (one of kJencSampling), header included;
// src and blk0 are left for the caller.
inline void jenc_image(int h, int w, int quality, int sampling, JencImage* im) {
    memset(im, 0, sizeof(*im));
    im->h = h;
    im->w = w;
    im->hmax = (sampling >> 20) & 15;
    im->vmax = (sampling >> 16) & 15;
    im->mcux = (w + 8 * im->hmax - 1) / (8 * im->hmax);
    im->mcuy = (h + 8 * im->vmax - 1) / (8 * im->vmax);
    for (int c = 0; c < 3; ++c) {
        JencComp& cp = im->comp[c];
        cp.h = c ? 1 : im->hmax;
        cp.v = c ? 1 : im->vmax;
        cp.fx = im->hmax / cp.h;
        cp.fy = im->vmax / cp.v;
        cp.wib = (int)(((long long)w * cp.h + 8 * im->hmax - 1) / (8 * im->hmax));
        cp.hib = (int)(((long long)h * cp.v + 8 * im->vmax - 1) / (8 * im->vmax));
        cp.rows = (h + im->vmax - 1) / im->vmax * cp.v;
        cp.t = c ? 1 : 0;
        for (int y = 0; y < cp.v; ++y)
            for (int x = 0; x < cp.h; ++x, ++im->bpm) {
                im->mcu_comp[im->bpm] = c;
                im->mcu_bx[im->bpm] = x;
                im->mcu_by[im->bpm] = y;
            }
    }
    im->blocks = (long long)im->mcux * im->mcuy * im->bpm;
    int qt[2][64];
    jenc_quant_tables(quality, qt);
    for (int t = 0; t < 2; ++t)
        for (int i = 0; i < 64; ++i) jenc_reciprocal(qt[t][i], &im->recip[t][i], &im->corr[t][i], &im->shift[t][i]);
    // the header, as jcmarker.c writes it
    unsigned char* p = im->hdr;
    auto u8 = [&](int v) { *p++ = (unsigned char)v; };
    auto u16 = [&](int v) { u8(v >> 8); u8(v & 255); };
    u16(0xFFD8);
    u16(0xFFE0); u16(16);
    for (char ch : {'J', 'F', 'I', 'F', '\0'}) u8(ch);
    u8(1); u8(1); u8(0); u16(1); u16(1); u8(0); u8(0);
    for (int t = 0; t < 2; ++t) {
        u16(0xFFDB); u16(67); u8(t);
        for (int k = 0; k < 64; ++k) u8(qt[t][jp_natural(k)]);
    }
    u16(0xFFC0); u16(17); u8(8); u16(h); u16(w); u8(3);
    for (int c = 0; c < 3; ++c) {
        u8(c + 1);
        u8((im->comp[c].h << 4) | im->comp[c].v);
        u8(im->comp[c].t);
    }
    for (int t = 0; t < 4; ++t) {
        const bool ac = t & 1;
        const int cls = t >> 1, nv = ac ? 162 : 12;
        const unsigned char* bits = ac ? kJencAcBits[cls] : kJencDcBits[cls];
        u16(0xFFC4); u16(2 + 1 + 16 + nv); u8((ac << 4) | cls);
        for (int l = 0; l < 16; ++l) u8(bits[l]);
        for (int k = 0; k < nv; ++k) u8(ac ? kJencAcVals[cls][k] : k);
    }
    u16(0xFFDA); u16(12); u8(3);
    for (int c = 0; c < 3; ++c) {
        u8(c + 1);
        u8(c ? 0x11 : 0x00);
    }
    u8(0); u8(63); u8(0);
    im->hdr_len = (int)(p - im->hdr);
}

// The 32-bit words a bit buffer of `bits` bits spans (and a spare word), and the stream bytes that always suffice for
// an image: the header, every block at its longest codes, each byte stuffed, and EOI.
inline long long jenc_words(long long bits) { return bits / 32 + 2; }
inline long long jenc_stream_bound(const JencImage& im) {
    return im.hdr_len + 2 * ((im.blocks * kJencBlockBitsMax + 7) / 8) + 2;
}

}  // namespace b2p
