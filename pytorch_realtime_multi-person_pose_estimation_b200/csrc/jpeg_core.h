// JPEG decoding, host/device shared core: baseline / extended sequential Huffman JPEG -> uint8 HWC BGR, oriented.
//   cv2.imdecode(buf, cv2.IMREAD_COLOR)   (OpenCV 4.13 with libjpeg-turbo 3.1)
// What libjpeg-turbo computes on the path cv2 takes, restated (DESIGN.md 2.13):
//  * entropy decoding as jdhuff.c: a run past coefficient 63 stores at 63 (jpeg_natural_order's guard entries), DC
//    predictors in 32-bit ints reset at every restart marker, coefficients stored as 16-bit JCOEF;
//  * the accurate integer IDCT (CONST_BITS 13, PASS1_BITS 2) as libjpeg-turbo's SIMD islow computes it on x86-64,
//    not the plain-C jidctint.c: 16-bit dequantisation and word sums, pass 1 saturated to 16 bits with its zero-row
//    shortcut, output saturated to 0 .. 255 (the C build's range-limit table wraps instead);
//  * jdsample.c's upsampling: the "fancy" triangular filters h2v1 / h2v2 (for a downsampled width > 2) and h1v2, plain
//    replication otherwise (h2v1 / h2v2 with width <= 2, and 4:1:1, for which libjpeg-turbo has no fancy path); the
//    first and last sample row / column are repeated outwards, as jdmainct.c's context rows and the filters' edge
//    cases do;
//  * jdcolor.c's YCbCr -> RGB tables (SCALEBITS 16, ONE_HALF rounding), written out as JCS_EXT_BGR; grayscale is
//    replicated into B, G and R;
//  * OpenCV's EXIF orientation (ExifReader + ApplyExifOrientation): the first orientation entry of IFD0 among the APP1
//    segments that begin "Exif\0\0" (a TIFF header from byte 6), mapped through frame_core.h's rotation plus a mirror
//    for 2, 4, 5 and 7.
// Progressive (SOF2) streams are parsed scan by scan when jpeg_parse's `progressive` is set, and their scans decoded as
// jdphuff.c does into the same coefficient buffer (DESIGN.md 2.18); the steps above then run unchanged.
// The parse (host only) validates every length, table and dimension; streams the device does not decode are reported
// as unsupported with the reason.  The decode steps are the functions the kernels of jpeg.cu run, and the host build of
// the tests (tests/cuda/jpeg_core_host.cpp) runs them in the same order.
#pragma once

#include "frame_core.h"

#if defined(__CUDACC__)
#define B2P_JP_HD __host__ __device__ __forceinline__
#else
#define B2P_JP_HD inline
#endif

namespace b2p {

constexpr int kJpegLutBits = 9;
constexpr int kJpegMaxBlocksPerMcu = 6;     // 4:2:0 / 4:2:2-like luma 2x2 / 4x1 + two chroma blocks
constexpr int kJpegChunkBits = 1024;        // bits of entropy data one thread decodes per round (jpeg.cu)

// per-image status bits of the entropy decoding (b200pose_post_jpeg_status)
constexpr unsigned kJpegBadCode = 1u, kJpegShortData = 2u, kJpegExtraData = 4u, kJpegBadRestart = 8u;

// A Huffman table in decoding form: lut[next 9 bits] = (length << 8) | symbol for codes of <= 9 bits (0: longer);
// maxcode[l] the largest code of length l (-1: none), valoff[l] + code = index in vals of a code of length l.
struct JpegHuff {
    unsigned short lut[1 << kJpegLutBits];
    int maxcode[18];
    int valoff[17];
    unsigned char vals[256];
};

struct JpegComp {
    int h, v;            // sampling factors as decoded (1 x 1 for a one-component image)
    int bw, bh;          // blocks per row / column in the coefficient and sample planes
    int dw, dh;          // downsampled_width / _height: the component's meaningful samples
    int dc, ac;          // Huffman tables (index into JpegImage::huff: DC 0..3, AC 4..7)
    long long coef;      // first block's index in the batch's coefficient buffer (64 int16 each)
    long long plane;     // byte offset of the sample plane (pitch bw * 8)
};

// One image of a decode batch (device-resident descriptor).
struct JpegImage {
    int h, w;                    // decoded (stored) frame
    int oh, ow, rot, mirror;     // oriented frame: output (y, x) shows stored fr_source_pixel(y, ow - 1 - x if mirror)
    int ncomp, hmax, vmax, mcux, mcuy, bpm, restart;
    int mcu_comp[kJpegMaxBlocksPerMcu], mcu_bx[kJpegMaxBlocksPerMcu], mcu_by[kJpegMaxBlocksPerMcu];
    JpegComp comp[3];
    int qt[3][64];               // dequantisation table of each component, natural order
    unsigned char zz[80];        // jpeg_natural_order with its 16 guard entries (a run past 63 stores at 63)
    JpegHuff huff[8];
    long long out;               // byte offset of the oriented BGR frame in the output
};

// One entropy-coded segment (a restart interval): bytes [beg, end) of the unstuffed data, MCUs mcu0 .. mcu0 + mcus - 1.
struct JpegSeg {
    int img;
    int mcu0, mcus;
    long long beg, end;
    long long chunk0;            // global index of its first chunk
};

// Decoder state at a chunk boundary: next symbol at bit p of the segment, coefficient k of block b of the MCU.
struct JpegState {
    long long p;
    int k, b;
};

B2P_JP_HD bool jp_same(const JpegState& a, const JpegState& b) { return a.p == b.p && a.k == b.k && a.b == b.b; }

// jpeg_natural_order: zig-zag index -> natural (row-major) index
B2P_JP_HD int jp_natural(int k) {
    const unsigned char t[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                 41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
    return t[k > 63 ? 63 : k];
}

// ---------------------------------------------------------------------------------------------- entropy decoding
// 32 bits of segment data [beg, end) starting at bit p; bytes past the end read as zeros (libjpeg's fill at a marker).
B2P_JP_HD unsigned jp_peek32(const unsigned char* data, long long nbytes, long long p) {
    const long long i = p >> 3;
    unsigned long long v = 0;
    for (int j = 0; j < 5; ++j) v = (v << 8) | (i + j < nbytes ? data[i + j] : 0u);
    return (unsigned)(v >> (8 - (p & 7)));
}

// HUFF_EXTEND
B2P_JP_HD int jp_extend(unsigned x, int s) { return s == 0 ? 0 : ((int)x < (1 << (s - 1)) ? (int)x + (int)(~0u << s) + 1 : (int)x); }

// Decodes one Huffman code at the top of `bits`: the symbol, and its length in *len (0: no such code).
B2P_JP_HD int jp_huff(const JpegHuff& t, unsigned bits, int* len) {
    const int e = t.lut[bits >> (32 - kJpegLutBits)];
    if (e) {
        *len = e >> 8;
        return e & 255;
    }
    int l = kJpegLutBits + 1;
    int code = (int)(bits >> (32 - l));
    while (l <= 16 && code > t.maxcode[l]) {
        ++l;
        code = (int)(bits >> (32 - l));
    }
    if (l > 16) {
        *len = 0;
        return 0;
    }
    *len = l;
    return t.vals[(t.valoff[l] + code) & 255];
}

// Decodes the symbol at state s (DC when s.k == 0, else AC) and advances s.  Writes the value into `block` (64
// coefficients, natural order; DC: the difference) when block is non-null.  Returns false on an invalid code.
// *done: the symbol ended its block (s.k is back to 0 and s.b advanced).
B2P_JP_HD bool jp_symbol(const JpegImage& im, JpegState& s, const unsigned char* data, long long nbytes, short* block,
                         bool* done) {
    const int c = im.mcu_comp[s.b];
    const unsigned bits = jp_peek32(data, nbytes, s.p);
    int len;
    if (s.k == 0) {
        const int t = jp_huff(im.huff[im.comp[c].dc], bits, &len);
        if (len == 0 || t > 15) return false;
        const unsigned v = t ? (bits << len) >> (32 - t) : 0u;
        if (block) block[0] = (short)jp_extend(v, t);
        s.p += len + t;
        s.k = 1;
    } else {
        const int rs = jp_huff(im.huff[im.comp[c].ac], bits, &len);
        if (len == 0) return false;
        const int r = rs >> 4, sz = rs & 15;
        if (sz) {
            s.k += r;
            const unsigned v = (bits << len) >> (32 - sz);
            if (block) block[im.zz[s.k]] = (short)jp_extend(v, sz);
            s.k += 1;
        } else {
            s.k = r == 15 ? s.k + 16 : 64;
        }
        s.p += len + sz;
    }
    *done = s.k >= 64;
    if (*done) {
        s.k = 0;
        s.b = s.b + 1 == im.bpm ? 0 : s.b + 1;
    }
    return true;
}

// Speculative decoding of a chunk: symbols from state s while s.p < end (bits of the segment).  Returns the blocks
// whose DC symbol this chunk decoded; s becomes the state at the chunk's exit.  An invalid code means the entry state
// was a wrong guess (the writing pass reports those of the true path): decoding resumes at the next bit as a fresh
// guess, so that the exit can still agree with the true path's and stop the next round there.
B2P_JP_HD int jp_sync_chunk(const JpegImage& im, JpegState& s, const unsigned char* data, long long nbytes, long long end) {
    int blocks = 0;
    while (s.p < end) {
        const bool dc = s.k == 0;
        bool done;
        if (!jp_symbol(im, s, data, nbytes, nullptr, &done)) {
            s = JpegState{s.p + 1, 0, 0};
            continue;
        }
        blocks += dc;
    }
    return blocks;
}

// The coefficients of block g (decode order) of a segment starting at MCU mcu0: a pointer into the coefficient buffer.
B2P_JP_HD short* jp_block_ptr(const JpegImage& im, short* coef, int mcu0, long long g) {
    const long long m = mcu0 + g / im.bpm;
    const int b = (int)(g % im.bpm), c = im.mcu_comp[b];
    const JpegComp& cp = im.comp[c];
    const long long bx = (m % im.mcux) * cp.h + im.mcu_bx[b], by = (m / im.mcux) * cp.v + im.mcu_by[b];
    return coef + (cp.coef + by * cp.bw + bx) * 64;
}

// The writing pass of a chunk: from its final entry state s, block index g (decode order within the segment), until
// the chunk's end (last: the segment's last block).  Returns the status bits it found.
B2P_JP_HD unsigned jp_write_chunk(const JpegImage& im, const JpegSeg& sg, JpegState s, long long g, long long end,
                                  bool last, const unsigned char* data, short* coef) {
    const long long nbytes = sg.end - sg.beg, total = (long long)sg.mcus * im.bpm, bits = nbytes * 8;
    while (last ? g < total : s.p < end) {
        if (g >= total) return kJpegExtraData;
        if (s.p >= bits) return kJpegShortData;
        bool done;
        if (!jp_symbol(im, s, data, nbytes, jp_block_ptr(im, coef, sg.mcu0, g), &done)) return kJpegBadCode;
        g += done;
    }
    if (last && s.p > bits) return kJpegShortData;
    if (last && bits - s.p >= 8) return kJpegExtraData;
    return 0;
}

// ---------------------------------------------------------------------------------------------- samples
constexpr int kIdctConst = 13, kIdctPass1 = 2;
constexpr long long kFix0298631336 = 2446, kFix0390180644 = 3196, kFix0541196100 = 4433, kFix0765366865 = 6270,
                    kFix0899976223 = 7373, kFix1175875602 = 9633, kFix1501321110 = 12299, kFix1847759065 = 15137,
                    kFix1961570560 = 16069, kFix2053119869 = 16819, kFix2562915447 = 20995, kFix3072711026 = 25172;

B2P_JP_HD long long jp_descale(long long x, int n) { return (x + (1LL << (n - 1))) >> n; }

// The low 16 bits of x as a signed word (pmullw, paddw, psllw), and signed saturation to 16 bits (packssdw).
B2P_JP_HD long long jp_w16(long long x) { return (long long)(short)(unsigned short)(x & 0xFFFF); }
B2P_JP_HD long long jp_clamp64(long long x, long long lo, long long hi) { return x < lo ? lo : (x > hi ? hi : x); }

// One 1-D pass of the SIMD islow IDCT (jidctint-avx2.asm / -sse2.asm) on 16-bit words in[0], in[st], .. in[7 st]:
// out[0..7] before the descale.  The products are jidctint.c's, regrouped into pmaddwd pairs (exact in 32 bits), but
// in0 + in4, in0 - in4, in7 + in3 and in5 + in1 are 16-bit word sums that wrap.
B2P_JP_HD void jp_idct_1d(const short* in, int st, long long* out) {
    const long long i0 = in[0], i1 = in[st], i2 = in[2 * st], i3 = in[3 * st], i4 = in[4 * st], i5 = in[5 * st],
                    i6 = in[6 * st], i7 = in[7 * st];
    const long long tmp0 = jp_w16(i0 + i4) * (1LL << kIdctConst), tmp1 = jp_w16(i0 - i4) * (1LL << kIdctConst);
    const long long tmp2 = i2 * kFix0541196100 + i6 * (kFix0541196100 - kFix1847759065);
    const long long tmp3 = i2 * (kFix0541196100 + kFix0765366865) + i6 * kFix0541196100;
    const long long tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    const long long z3 = jp_w16(i7 + i3), z4 = jp_w16(i5 + i1);
    const long long z3p = z3 * (kFix1175875602 - kFix1961570560) + z4 * kFix1175875602;
    const long long z4p = z3 * kFix1175875602 + z4 * (kFix1175875602 - kFix0390180644);
    const long long o0 = i7 * (kFix0298631336 - kFix0899976223) + i1 * -kFix0899976223 + z3p;
    const long long o1 = i5 * (kFix2053119869 - kFix2562915447) + i3 * -kFix2562915447 + z4p;
    const long long o2 = i5 * -kFix2562915447 + i3 * (kFix3072711026 - kFix2562915447) + z3p;
    const long long o3 = i7 * -kFix0899976223 + i1 * (kFix1501321110 - kFix0899976223) + z4p;
    out[0] = tmp10 + o3;
    out[7] = tmp10 - o3;
    out[1] = tmp11 + o2;
    out[6] = tmp11 - o2;
    out[2] = tmp12 + o1;
    out[5] = tmp12 - o1;
    out[3] = tmp13 + o0;
    out[4] = tmp13 - o0;
}

// jsimd_idct_islow of one block, what libjpeg-turbo runs on x86-64 in place of jpeg_idct_islow: coefficients (natural
// order) times qt as 16-bit products (pmullw); pass 1 over columns, its results saturated to 16 bits, except that a
// block whose rows 1 .. 7 are all zero takes the shortcut (row 0 << PASS1_BITS as a 16-bit shift, which wraps);
// pass 2 over rows, saturated to -128 .. 127 (packssdw, packsswb) plus 128.  -> 8 x 8 samples at out (pitch `pitch`).
B2P_JP_HD void jp_idct_block(const short* coef, const int* qt, unsigned char* out, long long pitch) {
    short deq[64], ws[64];
    long long o[8];
    bool ac_rows_zero = true;
    for (int i = 0; i < 64; ++i) {
        deq[i] = (short)jp_w16((long long)coef[i] * qt[i]);
        if (i >= 8 && coef[i]) ac_rows_zero = false;
    }
    for (int c = 0; c < 8; ++c) {
        if (ac_rows_zero) {
            for (int r = 0; r < 8; ++r) ws[r * 8 + c] = (short)jp_w16((long long)deq[c] * (1 << kIdctPass1));
            continue;
        }
        jp_idct_1d(deq + c, 8, o);
        for (int r = 0; r < 8; ++r) ws[r * 8 + c] = (short)jp_clamp64(jp_descale(o[r], kIdctConst - kIdctPass1), -32768, 32767);
    }
    for (int r = 0; r < 8; ++r) {
        jp_idct_1d(ws + r * 8, 1, o);
        for (int c = 0; c < 8; ++c)
            out[r * pitch + c] = (unsigned char)(jp_clamp64(jp_descale(o[c], kIdctConst + kIdctPass1 + 3), -128, 127) + 128);
    }
}

B2P_JP_HD int jp_clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// Upsampled sample (y, x) of component c (full-resolution coordinates of the stored frame).
B2P_JP_HD int jp_chroma(const JpegImage& im, const unsigned char* planes, int c, int y, int x) {
    const JpegComp& cp = im.comp[c];
    const unsigned char* pl = planes + cp.plane;
    const long long pitch = (long long)cp.bw * 8;
    const int fx = im.hmax / cp.h, fy = im.vmax / cp.v;
    if (fx == 1 && fy == 1) return pl[y * pitch + x];
    const bool fancy_h = fx == 2 && cp.dw > 2;
    if (fx == 2 && fy == 1 && fancy_h) {      // h2v1_fancy_upsample
        const int cx = x >> 1, nx = jp_clampi(x & 1 ? cx + 1 : cx - 1, 0, cp.dw - 1);
        const unsigned char* row = pl + y * pitch;
        return (3 * row[cx] + row[nx] + (x & 1 ? 2 : 1)) >> 2;
    }
    if (fx == 2 && fy == 2 && fancy_h) {      // h2v2_fancy_upsample
        const int cy = y >> 1, ny = jp_clampi(y & 1 ? cy + 1 : cy - 1, 0, cp.dh - 1);
        const int cx = x >> 1, nx = jp_clampi(x & 1 ? cx + 1 : cx - 1, 0, cp.dw - 1);
        const unsigned char *r0 = pl + cy * pitch, *r1 = pl + ny * pitch;
        const int this_sum = 3 * r0[cx] + r1[cx], next_sum = 3 * r0[nx] + r1[nx];
        return (3 * this_sum + next_sum + (x & 1 ? 7 : 8)) >> 4;
    }
    if (fx == 1 && fy == 2) {                 // h1v2_fancy_upsample
        const int cy = y >> 1, ny = jp_clampi(y & 1 ? cy + 1 : cy - 1, 0, cp.dh - 1);
        return (3 * pl[cy * pitch + x] + pl[ny * pitch + x] + (y & 1 ? 2 : 1)) >> 2;
    }
    return pl[(y / fy) * pitch + x / fx];      // h2v1_upsample / h2v2_upsample / int_upsample: replication
}

constexpr int kJpegScaleBits = 16;
constexpr int kJpegFixCrR = 91881, kJpegFixCbB = 116130, kJpegFixCrG = 46802, kJpegFixCbG = 22554;

B2P_JP_HD unsigned char jp_sat(int v) { return (unsigned char)(v < 0 ? 0 : (v > 255 ? 255 : v)); }

// ycc_rgb_convert for one pixel, stored B, G, R.
B2P_JP_HD void jp_ycc_to_bgr(int y, int cb, int cr, unsigned char* bgr) {
    const int half = 1 << (kJpegScaleBits - 1);
    const int xcb = cb - 128, xcr = cr - 128;
    const int cr_r = (kJpegFixCrR * xcr + half) >> kJpegScaleBits;
    const int cb_b = (kJpegFixCbB * xcb + half) >> kJpegScaleBits;
    const int g = (-kJpegFixCbG * xcb + half + -kJpegFixCrG * xcr) >> kJpegScaleBits;
    bgr[0] = jp_sat(y + cb_b);
    bgr[1] = jp_sat(y + g);
    bgr[2] = jp_sat(y + cr_r);
}

// Output pixel (y, x) of the oriented frame.
B2P_JP_HD void jpeg_px(const JpegImage& im, const unsigned char* planes, int y, int x, unsigned char* bgr) {
    int sy, sx;
    fr_source_pixel(im.h, im.w, im.rot, y, im.mirror ? im.ow - 1 - x : x, &sy, &sx);
    const int Y = jp_chroma(im, planes, 0, sy, sx);
    if (im.ncomp == 1) {
        bgr[0] = bgr[1] = bgr[2] = (unsigned char)Y;
        return;
    }
    jp_ycc_to_bgr(Y, jp_chroma(im, planes, 1, sy, sx), jp_chroma(im, planes, 2, sy, sx), bgr);
}

// The component-c block of decode-order index i of an image: its coefficients, and whether it starts a restart
// interval (the DC predictor is reset there).
B2P_JP_HD short* jp_dc_block(const JpegImage& im, short* coef, int c, long long i, bool* head) {
    const JpegComp& cp = im.comp[c];
    const int per = cp.h * cp.v;
    const long long m = i / per;
    const int j = (int)(i % per);
    *head = j == 0 && (im.restart ? m % im.restart == 0 : m == 0);
    const long long bx = (m % im.mcux) * cp.h + j % cp.h, by = (m / im.mcux) * cp.v + j / cp.h;
    return coef + (cp.coef + by * cp.bw + bx) * 64;
}

// ---------------------------------------------------------------------------------------------- progressive scans
// Progressive (SOF2) streams, jdphuff.c restated (DESIGN.md 2.18).  Every scan is decoded into the same coefficient
// buffer in stream order; the IDCT, upsampling and colour steps above then run unchanged.  A scan's unit is a block
// of its one component (component's own ceil(dw / 8) x ceil(dh / 8) blocks in raster order, not the MCU-padded plane)
// or, for an interleaved DC scan, an MCU of the frame; its restart interval counts units.
constexpr int kJpegMaxScans = 256;      // scans per image; more are refused as unsupported

// One scan of a progressive image (device-resident).  DC first scans decode component k of the scan with huff[k], AC
// first and refinement scans with huff[0]; DC refinement scans read no table.
struct JpegScan {
    int ncomp, comp[3];          // frame components of the scan, in frame order
    int ss, se, ah, al;          // spectral band and successive-approximation bits
    int units, restart;          // units of the scan; units per segment (0: one segment)
    int seg0, nseg;              // its segments in the batch's segment table (JpegSeg::mcu0 / mcus count units)
    JpegHuff huff[3];
};

// One progressive image of a decode batch: JpegImage img of the batch, its scans scan0 .. scan0 + nscans - 1.
struct JpegProgImage {
    int img, scan0, nscans;
};

// The next n (0 .. 16) bits at bit *p of the segment, advancing *p.
B2P_JP_HD unsigned jp_getbits(const unsigned char* d, long long nbytes, long long* p, int n) {
    if (n == 0) return 0;
    const unsigned v = jp_peek32(d, nbytes, *p) >> (32 - n);
    *p += n;
    return v;
}

// The block of unit u of scan sc holding its k-th block (k < the unit's blocks), and the scan component it belongs to.
B2P_JP_HD short* jp_prog_block(const JpegImage& im, const JpegScan& sc, short* coef, long long u, int k, int* ci) {
    if (sc.ncomp == 1) {
        const JpegComp& cp = im.comp[sc.comp[0]];
        const long long wb = (cp.dw + 7) / 8;
        *ci = 0;
        return coef + (cp.coef + (u / wb) * cp.bw + u % wb) * 64;
    }
    int c = 0;
    for (;; ++c) {
        const int per = im.comp[sc.comp[c]].h * im.comp[sc.comp[c]].v;
        if (k < per) break;
        k -= per;
    }
    const JpegComp& cp = im.comp[sc.comp[c]];
    *ci = c;
    const long long bx = (u % im.mcux) * cp.h + k % cp.h, by = (u / im.mcux) * cp.v + k / cp.h;
    return coef + (cp.coef + by * cp.bw + bx) * 64;
}

// jdphuff.c's decode_mcu_AC_refine for one block: correction bits for the band's nonzero coefficients passed over,
// new coefficients +-p1 at the r-th zero-history position, EOB runs.  16-bit JCOEF arithmetic.
B2P_JP_HD bool jp_ac_refine(const JpegImage& im, const JpegScan& sc, short* blk, const unsigned char* d, long long nbytes,
                            long long* p, int* eobrun) {
    const int p1 = 1 << sc.al, m1 = (int)(~0u << sc.al);
    int k = sc.ss;
    if (*eobrun == 0) {
        for (; k <= sc.se; ++k) {
            int len;
            const int rs = jp_huff(sc.huff[0], jp_peek32(d, nbytes, *p), &len);
            if (len == 0) return false;
            *p += len;
            int r = rs >> 4, s = rs & 15;
            if (s) {
                s = jp_getbits(d, nbytes, p, 1) ? p1 : m1;       // a size other than 1: libjpeg warns, reads one bit
            } else if (r != 15) {
                *eobrun = (1 << r) + (int)jp_getbits(d, nbytes, p, r);
                break;
            }
            do {
                short* c = blk + im.zz[k];
                if (*c != 0) {
                    if (jp_getbits(d, nbytes, p, 1) && (*c & p1) == 0) *c = (short)(*c >= 0 ? *c + p1 : *c + m1);
                } else if (--r < 0) {
                    break;
                }
                ++k;
            } while (k <= sc.se);
            if (s) blk[im.zz[k]] = (short)s;
        }
    }
    if (*eobrun > 0) {
        for (; k <= sc.se; ++k) {
            short* c = blk + im.zz[k];
            if (*c != 0 && jp_getbits(d, nbytes, p, 1) && (*c & p1) == 0) *c = (short)(*c >= 0 ? *c + p1 : *c + m1);
        }
        --*eobrun;
    }
    return true;
}

// Decodes segment sg of scan sc of image im (unstuffed bytes [sg.beg, sg.end) of data) into coef, as libjpeg's loop
// runs it from a restart: DC predictors and EOBRUN start at 0.  Returns the kJpeg* status bits it found.
B2P_JP_HD unsigned jp_prog_segment(const JpegImage& im, const JpegScan& sc, const JpegSeg& sg, const unsigned char* data,
                                   short* coef) {
    const unsigned char* d = data + sg.beg;
    const long long nbytes = sg.end - sg.beg, bits = nbytes * 8;
    long long p = 0;
    int pred[3] = {0, 0, 0}, eobrun = 0;
    int bpu = 1;                 // blocks per unit
    if (sc.ncomp > 1) {
        bpu = 0;
        for (int c = 0; c < sc.ncomp; ++c) bpu += im.comp[sc.comp[c]].h * im.comp[sc.comp[c]].v;
    }
    for (long long u = sg.mcu0; u < (long long)sg.mcu0 + sg.mcus; ++u) {
        for (int k = 0; k < bpu; ++k) {
            int ci;
            short* blk = jp_prog_block(im, sc, coef, u, k, &ci);
            if (sc.ss == 0 && sc.ah == 0) {              // DC first
                int len;
                const int t = jp_huff(sc.huff[ci], jp_peek32(d, nbytes, p), &len);
                if (len == 0 || t > 15) return kJpegBadCode;
                p += len;
                pred[ci] += jp_extend(jp_getbits(d, nbytes, &p, t), t);
                blk[0] = (short)(int)((unsigned)pred[ci] << sc.al);
            } else if (sc.ss == 0) {                     // DC refinement
                if (jp_getbits(d, nbytes, &p, 1)) blk[0] = (short)(blk[0] | (1 << sc.al));
            } else if (sc.ah == 0) {                     // AC first
                if (eobrun > 0) {
                    --eobrun;
                    continue;
                }
                for (int j = sc.ss; j <= sc.se; ++j) {
                    int len;
                    const int rs = jp_huff(sc.huff[0], jp_peek32(d, nbytes, p), &len);
                    if (len == 0) return kJpegBadCode;
                    p += len;
                    const int r = rs >> 4, s = rs & 15;
                    if (s) {
                        j += r;
                        blk[im.zz[j]] = (short)(int)((unsigned)jp_extend(jp_getbits(d, nbytes, &p, s), s) << sc.al);
                    } else if (r == 15) {
                        j += 15;
                    } else {
                        eobrun = (1 << r) + (int)jp_getbits(d, nbytes, &p, r) - 1;
                        break;
                    }
                }
            } else if (!jp_ac_refine(im, sc, blk, d, nbytes, &p, &eobrun)) {
                return kJpegBadCode;
            }
        }
        if (p > bits) return kJpegShortData;
    }
    if (bits - p >= 8) return kJpegExtraData;
    return 0;
}

}  // namespace b2p

// ================================================================================================ host-side parse
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <vector>

namespace b2p {

// Orientation value (1 .. 8, anything else: 1) -> rotation clockwise and mirror of the output x (applied first).
inline void jpeg_orientation(int o, int* rot, int* mirror) {
    const int r[9] = {0, 0, 0, 180, 180, 90, 90, 270, 270}, m[9] = {0, 0, 1, 0, 1, 1, 0, 1, 0};
    if (o < 1 || o > 8) o = 1;
    *rot = r[o];
    *mirror = m[o];
}

// OpenCV's ExifReader on an Exif APP1 segment's bytes from offset 6: IFD0's first orientation entry, -1 when there is
// none.  Byte order "II" is little-endian, anything else big-endian (as ExifReader reads a format it does not know);
// a read past the data ends the walk.
inline int jpeg_exif_orientation(const unsigned char* d, size_t n) {
    const bool intel = n > 1 && d[0] == d[1] && d[0] == 'I';
    bool ok = true;
    auto u16 = [&](size_t o) -> unsigned {
        if (o + 1 >= n) { ok = false; return 0; }
        return intel ? d[o] + (d[o + 1] << 8) : (d[o] << 8) + d[o + 1];
    };
    auto u32 = [&](size_t o) -> size_t {
        if (o + 3 >= n) { ok = false; return 0; }
        return intel ? d[o] + (d[o + 1] << 8) + (d[o + 2] << 16) + ((size_t)d[o + 3] << 24)
                     : ((size_t)d[o] << 24) + (d[o + 1] << 16) + (d[o + 2] << 8) + d[o + 3];
    };
    if (u16(2) != 0x2A || !ok) return -1;
    size_t off = u32(4);
    const size_t entries = ok ? u16(off) : 0;
    off += 2;
    for (size_t e = 0; e < entries && ok; ++e, off += 12)
        if (u16(off) == 0x0112 && ok) {
            const unsigned v = u16(off + 8);
            return ok ? (int)v : -1;
        }
    return -1;
}

// A parsed stream: its descriptor, and where its entropy-coded segments are in the stream and once unstuffed.
struct JpegParsed {
    bool supported = false;
    char reason[200] = {0};        // why a stream is malformed, or unsupported
    int h = 0, w = 0, orientation = 0;
    JpegImage im{};
    unsigned status = 0;           // what the marker walk found: kJpegBadRestart
    long long scan_beg = 0, scan_end = 0;                  // the scan's bytes [scan_beg, scan_end) of the stream
    std::vector<long long> seg_beg, seg_end;              // per segment, unstuffed bytes from the scan's start
    // Progressive streams (jpeg_parse's `progressive`): every scan with its tables, and its bytes [scan_raw[2s],
    // scan_raw[2s + 1]) of the stream; seg_beg / seg_end then hold the segments of all scans one after another, each in
    // unstuffed bytes from its own scan's start (JpegScan::seg0, nseg).  bits[c][k]: the Al of the last scan that
    // coded zig-zag coefficient k of component c (-1: none did), libjpeg's coef_bits.
    bool progressive = false;
    std::vector<JpegScan> scans;
    std::vector<long long> scan_raw;
    int bits[3][64];
};

inline bool jp_fail(JpegParsed* P, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(P->reason, sizeof(P->reason), fmt, ap);
    va_end(ap);
    return false;
}

inline bool jp_unsupported(JpegParsed* P, const char* what) {
    snprintf(P->reason, sizeof(P->reason), "unsupported: %s", what);
    return true;
}

// A decoding table from BITS / HUFFVAL, with jdhuff.c jpeg_make_d_derived_tbl's checks.
inline bool jpeg_build_huff(const unsigned char* counts, const unsigned char* vals, int nvals, bool dc, JpegHuff* t) {
    memset(t, 0, sizeof(*t));
    memcpy(t->vals, vals, nvals);
    int code = 0, k = 0;
    for (int l = 1; l <= 16; ++l) {
        t->valoff[l] = k - code;
        for (int i = 0; i < counts[l - 1]; ++i, ++k, ++code)
            if (l <= kJpegLutBits)
                for (int f = 0; f < (1 << (kJpegLutBits - l)); ++f)
                    t->lut[(code << (kJpegLutBits - l)) | f] = (unsigned short)((l << 8) | vals[k]);
        t->maxcode[l] = counts[l - 1] ? code - 1 : -1;
        if (code >= (1 << l)) return false;      // no code may be all ones
        code <<= 1;
    }
    t->maxcode[17] = 0x7fffffff;
    for (int i = 0; dc && i < nvals; ++i)
        if (vals[i] > 15) return false;
    return true;
}

// The entropy-coded data of a scan from byte beg: every 0xFF is a stuffed byte (FF 00), a restart marker (RSTn, ending
// a segment) or the marker after the scan; fill bytes (more 0xFF) may precede any of them.  Appends each segment's
// unstuffed [begin, end) from beg to sb / se and ORs kJpegBadRestart into *status for a misnumbered restart marker.
// Returns where the scan ends (the marker's first 0xFF, or n); *code: the marker after the scan (-1: none).
inline long long jpeg_scan_walk(const unsigned char* d, long long n, long long beg, std::vector<long long>* sb,
                                std::vector<long long>* se, unsigned* status, int* code) {
    long long dropped = 0, pos = beg, rst = 0, end = n;     // dropped: the bytes unstuffing removes
    *code = -1;
    sb->push_back(0);
    while (pos < n) {
        const void* f = memchr(d + pos, 0xFF, (size_t)(n - pos));
        if (!f) break;
        const long long a = (const unsigned char*)f - d;
        long long j = a + 1;
        while (j < n && d[j] == 0xFF) ++j;
        if (j >= n) {
            end = a;
            break;
        }
        const int c = d[j];
        pos = j + 1;
        if (c == 0x00) {
            dropped += j - a;
        } else if (c >= 0xD0 && c <= 0xD7) {
            if (c != 0xD0 + (rst & 7)) *status |= kJpegBadRestart;
            ++rst;
            se->push_back(a - beg - dropped);
            dropped += j - a + 1;
            sb->push_back(j + 1 - beg - dropped);
        } else {
            *code = c;
            end = a;
            break;
        }
    }
    se->push_back(end - beg - dropped);
    return end;
}

// One SOS of a progressive stream (payload s, ns components): the scan's checks, tables and progression, appended to
// P->scans.  Returns false for a malformed scan (reason set), true otherwise (P->reason set: unsupported).
struct JpegProgTables {
    const int (*qt)[64];
    const unsigned char (*counts)[16];
    const unsigned char (*vals)[256];
    const int* nvals;
    int qt_have, huff_have, restart;
    const int *ids, *tq;
    bool latched[3];
};

inline bool jp_prog_sos(JpegParsed* P, const unsigned char* s, int ns, JpegProgTables& T) {
    JpegImage& im = P->im;
    const int nf = im.ncomp;
    const int Ss = s[1 + 2 * ns], Se = s[2 + 2 * ns], Ah = s[3 + 2 * ns] >> 4, Al = s[3 + 2 * ns] & 15;
    const int scan = (int)P->scans.size();
    // jdphuff.c start_pass_phuff_decoder's JERR_BAD_PROGRESSION: cv2.imdecode returns None
    const bool dc = Ss == 0;
    if ((dc && Se != 0) || (!dc && (Ss > Se || Se > 63 || ns != 1)) || (Ah != 0 && Al != Ah - 1) || Al > 13)
        return jp_fail(P, "malformed scan %d: Ss %d, Se %d, Ah %d, Al %d with %d components is not a valid progression",
                       scan, Ss, Se, Ah, Al, ns);
    if (scan >= kJpegMaxScans) return jp_unsupported(P, "more than 256 scans");
    P->scans.emplace_back();
    JpegScan& sc = P->scans.back();
    memset(&sc, 0, sizeof(sc));
    sc.ncomp = ns;
    sc.ss = Ss;
    sc.se = Se;
    sc.ah = Ah;
    sc.al = Al;
    int prev = -1;
    for (int k = 0; k < ns; ++k) {
        int c = 0;
        while (c < nf && T.ids[c] != s[1 + 2 * k]) ++c;
        if (c == nf || c <= prev) return jp_unsupported(P, "scan components not in the frame's order");
        prev = c;
        sc.comp[k] = c;
        if (!T.latched[c]) {     // latch_quant_tables: a component keeps the table it had at its first scan
            if (!(T.qt_have >> T.tq[c] & 1)) return jp_fail(P, "malformed header: component %d has no quantisation table", c);
            memcpy(im.qt[c], T.qt[T.tq[c]], sizeof(im.qt[c]));
            T.latched[c] = true;
        }
        const int td = s[2 + 2 * k] >> 4, ta = s[2 + 2 * k] & 15;
        if (dc && Ah == 0) {     // DC refinement reads no table
            if (td > 3) return jp_fail(P, "malformed header: SOS DC table id %d", td);
            if (!(T.huff_have >> td & 1)) return jp_unsupported(P, "a scan with an undefined Huffman table");
            if (!jpeg_build_huff(T.counts[td], T.vals[td], T.nvals[td], true, &sc.huff[k]))
                return jp_fail(P, "malformed header: Huffman table DC %d is not a valid code", td);
        } else if (!dc) {
            if (ta > 3) return jp_fail(P, "malformed header: SOS AC table id %d", ta);
            if (!(T.huff_have >> (4 + ta) & 1)) return jp_unsupported(P, "a scan with an undefined Huffman table");
            if (!jpeg_build_huff(T.counts[4 + ta], T.vals[4 + ta], T.nvals[4 + ta], false, &sc.huff[0]))
                return jp_fail(P, "malformed header: Huffman table AC %d is not a valid code", ta);
        }
        // libjpeg only warns about a bogus progression (JWRN_BOGUS_PROGRESSION) and decodes on: left to cv2
        int* bits = P->bits[c];
        if (!dc && bits[0] < 0) return jp_unsupported(P, "a bogus progression (an AC scan before the component's DC)");
        for (int q = Ss; q <= Se; ++q) {
            if (Ah != (bits[q] < 0 ? 0 : bits[q]))
                return jp_unsupported(P, "a bogus progression (Ah differs from the bits already coded)");
            bits[q] = Al;
        }
    }
    if (ns == 1) {
        const JpegComp& cp = im.comp[sc.comp[0]];
        sc.units = ((cp.dw + 7) / 8) * ((cp.dh + 7) / 8);
    } else {
        sc.units = im.mcux * im.mcuy;
    }
    sc.restart = T.restart;
    return true;
}

// The frame geometry of a JpegImage: sizes, MCUs, per component its sampling, planes and downsampled size, and the
// blocks of an interleaved MCU.
inline void jpeg_geometry(JpegImage* im, int h, int w, int nf, const int* hs, const int* vs) {
    for (int k = 0; k < 80; ++k) im->zz[k] = (unsigned char)jp_natural(k);
    im->h = h;
    im->w = w;
    im->ncomp = nf;
    im->hmax = nf == 3 ? hs[0] : 1;
    im->vmax = nf == 3 ? vs[0] : 1;
    im->mcux = (im->w + 8 * im->hmax - 1) / (8 * im->hmax);
    im->mcuy = (im->h + 8 * im->vmax - 1) / (8 * im->vmax);
    im->bpm = 0;
    for (int c = 0; c < nf; ++c) {
        JpegComp& cp = im->comp[c];
        cp.h = nf == 3 ? hs[c] : 1;
        cp.v = nf == 3 ? vs[c] : 1;
        cp.bw = im->mcux * cp.h;
        cp.bh = im->mcuy * cp.v;
        cp.dw = (int)(((long long)im->w * cp.h + im->hmax - 1) / im->hmax);
        cp.dh = (int)(((long long)im->h * cp.v + im->vmax - 1) / im->vmax);
        for (int y = 0; y < cp.v; ++y)
            for (int x = 0; x < cp.h; ++x, ++im->bpm) {
                im->mcu_comp[im->bpm] = c;
                im->mcu_bx[im->bpm] = x;
                im->mcu_by[im->bpm] = y;
            }
    }
}

// The entropy-coded data of the progressive scan just parsed (P->scans.back()), from byte *i: its bytes, segments and
// restart status.  *i becomes the scan's end; returns false when the data ends there (no marker follows).
inline bool jpeg_prog_walk(const unsigned char* d, long long n, long long* i, JpegParsed* P) {
    JpegScan& sc = P->scans.back();
    sc.seg0 = (int)P->seg_beg.size();
    int code;
    const long long end = jpeg_scan_walk(d, n, *i, &P->seg_beg, &P->seg_end, &P->status, &code);
    const long long found = (long long)P->seg_beg.size() - sc.seg0;
    const long long expect = sc.restart ? (sc.units + (long long)sc.restart - 1) / sc.restart : 1;
    if (found != expect) P->status |= kJpegBadRestart;
    sc.nseg = (int)(found < expect ? found : expect);
    P->scan_raw.push_back(*i);
    P->scan_raw.push_back(end);
    *i = end;
    return code >= 0;
}

// Parses a whole stream: the headers up to the scan, then the scan's markers.  Returns false for a malformed stream
// (reason set); else P->supported tells whether the device decodes it (reason: why not).  max_pixels bounds h * w.
// progressive: progressive (SOF2) streams with 8-bit samples are parsed scan by scan (DESIGN.md 2.18) instead of being
// refused as unsupported.
inline bool jpeg_parse(const unsigned char* d, long long n, long long max_pixels, JpegParsed* P, bool progressive = false) {
    *P = JpegParsed{};
    if (!d || n < 4 || d[0] != 0xFF || d[1] != 0xD8) return jp_fail(P, "not a JPEG stream (no SOI marker)");
    struct Tables {
        int qt[4][64];
        unsigned char counts[8][16], vals[8][256];
        int nvals[8];
    } T{};
    int qt_have = 0, huff_have = 0, nf = 0, restart = 0, adobe = -1, sof = -1, prec = 8;
    bool jfif = false, exif_found = false;
    int ids[4] = {0}, hs[4] = {0}, vs[4] = {0}, tq[4] = {0};
    long long i = 2;
    JpegProgTables PT{T.qt, T.counts, T.vals, T.nvals, 0, 0, 0, ids, tq, {false, false, false}};
    for (;;) {
        // between the scans of a progressive stream, the end of the data stands for EOI (libjpeg's fill_input_buffer)
        if (P->progressive && i >= n) break;
        if (i >= n || d[i] != 0xFF) return jp_fail(P, "malformed header: no marker at byte %lld", i);
        while (i < n && d[i] == 0xFF) ++i;
        if (P->progressive && i >= n) break;
        if (i >= n) return jp_fail(P, "malformed header: the stream ends before the scan");
        const int m = d[i++];
        if (P->progressive && m == 0xD9) break;
        if (m == 0xD8 || m == 0xD9) return jp_fail(P, "malformed header: marker 0xFF%02X before the scan", m);
        if ((m >= 0xD0 && m <= 0xD7) || m == 0x01) continue;        // parameterless markers
        if (P->progressive && (i + 2 > n || i + ((d[i] << 8) | d[i + 1]) > n))
            return jp_unsupported(P, "a marker segment cut off between scans");
        if (i + 2 > n) return jp_fail(P, "malformed header: the stream ends in marker 0xFF%02X", m);
        const long long len = (d[i] << 8) | d[i + 1];
        if (len < 2 || i + len > n) return jp_fail(P, "malformed header: segment 0xFF%02X of length %lld runs past the data", m, len);
        const unsigned char* s = d + i + 2;
        const long long sl = len - 2;
        i += len;
        if (m >= 0xC0 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC) {        // SOFn
            if (sof >= 0) return jp_fail(P, "malformed header: a second SOF marker");
            sof = m;
            if (sl < 6) return jp_fail(P, "malformed header: SOF segment of %lld bytes", sl);
            prec = s[0];
            P->h = (s[1] << 8) | s[2];
            P->w = (s[3] << 8) | s[4];
            nf = s[5];
            if (nf < 1 || sl != 6 + 3 * nf) return jp_fail(P, "malformed header: SOF length %lld for %d components", len, nf);
            for (int c = 0; c < nf && c < 4; ++c) {
                ids[c] = s[6 + 3 * c];
                hs[c] = s[7 + 3 * c] >> 4;
                vs[c] = s[7 + 3 * c] & 15;
                tq[c] = s[8 + 3 * c];
                if (hs[c] < 1 || hs[c] > 4 || vs[c] < 1 || vs[c] > 4 || tq[c] > 3)
                    return jp_fail(P, "malformed header: component %d sampling %dx%d, table %d", c, hs[c], vs[c], tq[c]);
            }
            if (P->w < 1) return jp_fail(P, "malformed header: width 0");
        } else if (m == 0xC4) {                                                      // DHT
            for (long long o = 0; o < sl;) {
                if (o + 17 > sl) return jp_fail(P, "malformed header: truncated DHT segment");
                const int tc = s[o] >> 4, th = s[o] & 15;
                if (tc > 1 || th > 3) return jp_fail(P, "malformed header: DHT class / id 0x%02X", s[o]);
                int cnt = 0;
                for (int l = 0; l < 16; ++l) cnt += s[o + 1 + l];
                if (cnt > 256 || o + 17 + cnt > sl) return jp_fail(P, "malformed header: DHT table of %d symbols", cnt);
                const int t = tc * 4 + th;
                memcpy(T.counts[t], s + o + 1, 16);
                memcpy(T.vals[t], s + o + 17, cnt);
                T.nvals[t] = cnt;
                huff_have |= 1 << t;
                o += 17 + cnt;
            }
        } else if (m == 0xDB) {                                                      // DQT
            for (long long o = 0; o < sl;) {
                const int pq = s[o] >> 4, t = s[o] & 15;
                if (pq > 1 || t > 3) return jp_fail(P, "malformed header: DQT precision / id 0x%02X", s[o]);
                if (o + 1 + 64 * (pq + 1) > sl) return jp_fail(P, "malformed header: truncated DQT segment");
                for (int k = 0; k < 64; ++k)     // ISLOW_MULT_TYPE is a short in libjpeg-turbo's SIMD builds
                    T.qt[t][jp_natural(k)] = (short)(pq ? (s[o + 1 + 2 * k] << 8) | s[o + 2 + 2 * k] : s[o + 1 + k]);
                qt_have |= 1 << t;
                o += 1 + 64 * (pq + 1);
            }
        } else if (m == 0xDD) {                                                      // DRI
            if (sl != 2) return jp_fail(P, "malformed header: DRI segment of %lld bytes", sl);
            restart = (s[0] << 8) | s[1];
        } else if (m == 0xE0) {
            if (sl >= 14 && !memcmp(s, "JFIF\0", 5)) jfif = true;
        } else if (m == 0xE1) {
            // cv2 4.13: the first orientation entry of the APP1 segments that begin "Exif\0\0", in stream order;
            // other APP1 segments (XMP, ...) are passed over
            if (!exif_found && sl > 6 && !memcmp(s, "Exif\0\0", 6)) {
                const int o = jpeg_exif_orientation(s + 6, (size_t)(sl - 6));
                if (o >= 0) {
                    P->orientation = o;
                    exif_found = true;
                }
            }
        } else if (m == 0xEE) {
            if (sl >= 12 && !memcmp(s, "Adobe", 5)) adobe = s[11];
        } else if (m == 0xDA) {                                                      // SOS
            if (sof < 0) return jp_fail(P, "malformed header: SOS before SOF");
            const int ns = sl >= 1 ? s[0] : 0;
            if (ns < 1 || ns > 4 || sl != 4 + 2 * ns) return jp_fail(P, "malformed header: SOS segment of %lld bytes", sl);
            if (P->progressive) {      // a later scan of a progressive stream
                PT.qt_have = qt_have;
                PT.huff_have = huff_have;
                PT.restart = restart;
                if (!jp_prog_sos(P, s, ns, PT)) return false;
                if (P->reason[0]) return true;
                if (!jpeg_prog_walk(d, n, &i, P)) break;
                continue;
            }
            P->scan_beg = i;
            if (P->h < 1 || (long long)P->h * P->w > max_pixels)
                return jp_fail(P, "%d x %d pixels: a frame has 1 .. %lld pixels", P->h, P->w, max_pixels);
            jpeg_orientation(P->orientation, &P->im.rot, &P->im.mirror);
            fr_rotated_size(P->h, P->w, P->im.rot, &P->im.oh, &P->im.ow);
            char why[96];
            why[0] = 0;
            const bool prog = progressive && sof == 0xC2;
            if ((sof == 0xC2 && !prog) || sof == 0xC6) snprintf(why, sizeof(why), "progressive (SOF%d)", sof - 0xC0);
            else if (sof == 0xC3 || sof == 0xC7) snprintf(why, sizeof(why), "lossless (SOF%d)", sof - 0xC0);
            else if (sof >= 0xC9) snprintf(why, sizeof(why), "arithmetic-coded (SOF%d)", sof - 0xC0);
            else if (sof == 0xC5) snprintf(why, sizeof(why), "hierarchical (SOF5)");
            else if (prec != 8) snprintf(why, sizeof(why), "%d-bit samples", prec);
            else if (nf == 4) snprintf(why, sizeof(why), "4 components (CMYK / YCCK)");
            else if (nf != 1 && nf != 3) snprintf(why, sizeof(why), "%d components", nf);
            if (why[0]) return jp_unsupported(P, why);
            if (nf == 3 && !jfif && adobe == 0) return jp_unsupported(P, "Adobe RGB (transform 0)");
            if (nf == 3 && !jfif && adobe < 0 && ids[0] == 'R' && ids[1] == 'G' && ids[2] == 'B')
                return jp_unsupported(P, "R/G/B component ids");
            const int hv = hs[0] * 10 + vs[0];
            if (nf == 3 && (!(hv == 11 || hv == 21 || hv == 22 || hv == 12 || hv == 41) || hs[1] != 1 || vs[1] != 1 ||
                            hs[2] != 1 || vs[2] != 1))
                return jp_unsupported(P, "sampling other than luma 1x1, 2x1, 2x2, 1x2 or 4x1 with chroma 1x1");
            JpegImage& im = P->im;
            if (prog) {                // the first scan of a progressive stream
                jpeg_geometry(&im, P->h, P->w, nf, hs, vs);
                P->progressive = true;
                memset(P->bits, 0xFF, sizeof(P->bits));
                PT.qt_have = qt_have;
                PT.huff_have = huff_have;
                PT.restart = restart;
                if (!jp_prog_sos(P, s, ns, PT)) return false;
                if (P->reason[0]) return true;
                if (!jpeg_prog_walk(d, n, &i, P)) break;
                continue;
            }
            if (ns != nf) return jp_unsupported(P, "a scan without every component (multi-scan sequential)");
            for (int c = 0; c < ns; ++c) {
                const int td = s[2 + 2 * c] >> 4, ta = s[2 + 2 * c] & 15;
                if (s[1 + 2 * c] != ids[c]) return jp_unsupported(P, "scan components in another order than the frame's");
                if (td > 3 || ta > 3) return jp_fail(P, "malformed header: SOS table ids 0x%02X", s[2 + 2 * c]);
                if (!(huff_have >> td & 1) || !(huff_have >> (4 + ta) & 1))
                    return jp_unsupported(P, "a scan with an undefined Huffman table");
                if (!(qt_have >> tq[c] & 1)) return jp_fail(P, "malformed header: component %d has no quantisation table", c);
                im.comp[c].dc = td;
                im.comp[c].ac = 4 + ta;
                if (!jpeg_build_huff(T.counts[td], T.vals[td], T.nvals[td], true, &im.huff[td]) ||
                    !jpeg_build_huff(T.counts[4 + ta], T.vals[4 + ta], T.nvals[4 + ta], false, &im.huff[4 + ta]))
                    return jp_fail(P, "malformed header: Huffman table DC %d / AC %d is not a valid code", td, ta);
                memcpy(im.qt[c], T.qt[tq[c]], sizeof(im.qt[c]));
            }
            jpeg_geometry(&im, P->h, P->w, nf, hs, vs);
            im.restart = restart;
            break;
        } else if (m == 0xDC || (m >= 0xE2 && m <= 0xEF) || m == 0xFE) {
            // DNL, other APPn, COM: skipped
        } else {
            return jp_fail(P, "malformed header: unknown marker 0xFF%02X", m);
        }
    }
    if (P->progressive) {
        // jdcoefct.c's block smoothing changes the output where bits of zig-zag coefficients 0 .. 9 are still unknown
        // after the last scan; such streams are left to cv2
        for (int c = 0; c < P->im.ncomp; ++c)
            for (int k = 0; k < 10; ++k)
                if (P->bits[c][k] != 0) {
                    char why[120];
                    snprintf(why, sizeof(why), "an incomplete progression (component %d, zig-zag coefficient %d: %s), "
                             "which libjpeg smooths", c, k, P->bits[c][k] < 0 ? "never coded" : "low bits not coded");
                    return jp_unsupported(P, why);
                }
        P->scan_beg = P->scan_raw.front();
        P->scan_end = P->scan_raw.back();
        P->supported = true;
        return true;
    }
    const long long mcus = (long long)P->im.mcux * P->im.mcuy;
    const long long expect = P->im.restart ? (mcus + P->im.restart - 1) / P->im.restart : 1;
    int code;
    P->scan_end = jpeg_scan_walk(d, n, P->scan_beg, &P->seg_beg, &P->seg_end, &P->status, &code);
    if (code == 0xDA) return jp_unsupported(P, "more than one scan");
    if ((long long)P->seg_beg.size() != expect) P->status |= kJpegBadRestart;
    P->supported = true;
    return true;
}

// Splits the segments of one parsed image into JpegSeg entries (the first `expect` of them; MCU ranges by the restart
// interval), with unstuffed offsets from `base` and chunk indices from `chunk0`.  Returns the chunks used.
inline long long jpeg_segments(const JpegParsed& P, int img, long long base, long long chunk0, std::vector<JpegSeg>* out) {
    const JpegImage& im = P.im;
    const long long mcus = (long long)im.mcux * im.mcuy;
    const long long per = im.restart ? im.restart : mcus;
    long long chunks = 0;
    for (size_t k = 0; k < P.seg_beg.size() && (long long)k * per < mcus; ++k) {
        JpegSeg s;
        s.img = img;
        s.mcu0 = (int)(k * per);
        s.mcus = (int)((mcus - s.mcu0) < per ? mcus - s.mcu0 : per);
        s.beg = base + P.seg_beg[k];
        s.end = base + P.seg_end[k];
        s.chunk0 = chunk0 + chunks;
        const long long bits = (s.end - s.beg) * 8;
        chunks += bits > 0 ? (bits + kJpegChunkBits - 1) / kJpegChunkBits : 1;
        out->push_back(s);
    }
    return chunks;
}

// The scans of one parsed progressive image appended to *scans and their segments to *segs as JpegSeg entries (units
// by the scan's restart interval), scan s's unstuffed data starting at scan_base[s]; seg0 indexes *segs.
inline void jpeg_prog_segments(const JpegParsed& P, int img, const long long* scan_base, std::vector<JpegScan>* scans,
                               std::vector<JpegSeg>* segs) {
    for (size_t s = 0; s < P.scans.size(); ++s) {
        JpegScan sc = P.scans[s];
        const long long per = sc.restart ? sc.restart : sc.units;
        const int first = sc.seg0;
        sc.seg0 = (int)segs->size();
        for (int k = 0; k < sc.nseg; ++k) {
            JpegSeg g{};
            g.img = img;
            g.mcu0 = (int)(k * per);
            g.mcus = (int)(sc.units - g.mcu0 < per ? sc.units - g.mcu0 : per);
            g.beg = scan_base[s] + P.seg_beg[first + k];
            g.end = scan_base[s] + P.seg_end[first + k];
            segs->push_back(g);
        }
        scans->push_back(sc);
    }
}

// The Huffman kernel's work for segments holding `chunks` chunks in all: the segment of every chunk, and runs of whole
// segments of at least kJpegWorkChunks chunks (the last may be shorter), one CTA each: work[w] .. work[w + 1].
constexpr long long kJpegWorkChunks = 1024;
inline void jpeg_work(const std::vector<JpegSeg>& segs, long long chunks, std::vector<int>* chunk_seg,
                      std::vector<long long>* work) {
    chunk_seg->assign((size_t)chunks, 0);
    work->assign(1, 0);
    for (size_t k = 0; k < segs.size(); ++k) {
        const long long c1 = k + 1 < segs.size() ? segs[k + 1].chunk0 : chunks;
        for (long long c = segs[k].chunk0; c < c1; ++c) (*chunk_seg)[c] = (int)k;
        if (c1 - work->back() >= kJpegWorkChunks || k + 1 == segs.size()) work->push_back(c1);
    }
}

}  // namespace b2p
