// PNG decoding, host/device shared core: PNG streams -> uint8 HWC BGR, oriented.
//   cv2.imdecode(buf, cv2.IMREAD_COLOR)   (OpenCV 4.13 with libpng 1.6 and zlib 1.3)
// What libpng and zlib compute on the path cv2 takes, restated (DESIGN.md 2.17):
//  * the chunk walk: signature, IHDR first, CRCs of critical chunks, PLTE before IDAT, consecutive IDATs, IEND; an
//    ancillary chunk with a bad CRC is passed over; eXIf's orientation is applied as for JPEG (jpeg_core.h's IFD0 walk,
//    frame_core.h's rotation plus a mirror);
//  * inflate as zlib's: the zlib header (CM 8, CINFO <= 7, FCHECK, no dictionary), stored / fixed / dynamic blocks,
//    inflate_table's rules for a code set (over-subscribed: invalid; incomplete: invalid, except a literal/length or
//    distance code of one symbol of length 1; empty: invalid once a symbol is decoded), the fixed code's invalid
//    symbols 286, 287 and distances 30, 31, distances past the output or the window, Adler-32 at the stream's end;
//  * libpng's reading of the inflated rows (png_read_IDAT_data, png_read_finish_IDAT): a stream that ends or fails
//    before the last row fails; after it, what counts depends on where the IDAT data reaches inflate - the call that
//    completed the last row goes on to the end of its piece (errors and the Adler-32 there are fatal), then inflate
//    reads on piece by piece into a scratch buffer, where errors are warnings, and fails only when it needs data that
//    the IDATs do not hold (pn_tail);
//  * the five filters, Paeth with libpng's a / b / c tie order, per Adam7 pass (empty passes have no rows);
//  * the transforms cv2 asks for: 16-bit samples keep their high byte (png_set_strip_16), gray below 8 bits is
//    replicated to 8 (png_set_expand_gray_1_2_4_to_8), palette indices map through PLTE with missing entries black,
//    alpha is dropped without compositing (png_set_strip_alpha; tRNS changes nothing), gray is replicated to B, G, R.
// The parse (host only) validates the chunk structure; damage inside the zlib data is found on the device and reported
// per image.  The decode steps are the functions the kernels of png.cu run, and the host build of the tests
// (tests/cuda/png_core_host.cpp) runs them in the same order.
#pragma once

#include "jpeg_core.h"
#include "png_enc_core.h"

namespace b2p {

// per-image status bits of the device decoding (b200pose_post_png_status); each is a stream cv2.imdecode refuses
constexpr unsigned kPngBadDeflate = 1u, kPngShortData = 2u, kPngBadAdler = 4u, kPngBadCrc = 8u, kPngBadFilter = 16u;
constexpr int kPngLutBits = 9;
constexpr int kPngTokens = 256;          // tokens the decoding lane hands the warp per round (png.cu)

// One image of a decode batch (device-resident descriptor).
struct PngDecImage {
    int h, w;                    // stored frame
    int oh, ow, rot, mirror;     // oriented frame: output (y, x) shows stored fr_source_pixel(y, ow - 1 - x if mirror)
    int ctype, depth, interlace, channels, bpp;
    long long z0, zlen;          // its zlib stream in the gathered buffer
    long long f0, flen;          // its filtered rows (every pass) in the inflate buffer
    long long out;               // byte offset of the oriented BGR frame in the output
    int idat0, nidat;            // its IDAT chunks in the batch's chunk table
    unsigned char pal[256 * 3];  // PLTE as R, G, B; entries past the chunk are 0
};

// One IDAT chunk: its type and data at src (length len + 4) in the upload, its data to dst in the zlib buffer.
struct PngIdat {
    int img;
    unsigned crc;
    long long src, len, dst;
};

// ---------------------------------------------------------------------------------------------- rows and passes
B2P_PN_HD int pn_channels(int ctype) { return ctype == 0 || ctype == 3 ? 1 : ctype == 2 ? 3 : ctype == 4 ? 2 : 4; }

// Adam7 pass p (0 .. 6) of an interlaced image, or the whole image (p = 0, interlace 0): its size in pixels.
B2P_PN_HD void pn_pass(int interlace, int p, int h, int w, int* ph, int* pw) {
    if (!interlace) {
        *ph = h;
        *pw = w;
        return;
    }
    const int xs[7] = {0, 4, 0, 2, 0, 1, 0}, ys[7] = {0, 0, 4, 0, 2, 0, 1}, dx[7] = {8, 8, 4, 4, 2, 2, 1},
              dy[7] = {8, 8, 8, 4, 4, 2, 2};
    *pw = w > xs[p] ? (w - xs[p] + dx[p] - 1) / dx[p] : 0;
    *ph = h > ys[p] ? (h - ys[p] + dy[p] - 1) / dy[p] : 0;
    if (*pw == 0 || *ph == 0) *pw = *ph = 0;
}

// Bytes of a row of pw pixels (filter byte apart).
B2P_PN_HD long long pn_rowbytes(const PngDecImage& im, int pw) { return ((long long)pw * im.channels * im.depth + 7) / 8; }

// Filtered bytes of pass p, and of the whole image.
B2P_PN_HD long long pn_pass_bytes(const PngDecImage& im, int p) {
    int ph, pw;
    pn_pass(im.interlace, p, im.h, im.w, &ph, &pw);
    return ph ? (long long)ph * (pn_rowbytes(im, pw) + 1) : 0;
}
B2P_PN_HD long long pn_filtered_bytes(const PngDecImage& im) {
    long long n = 0;
    for (int p = 0; p < (im.interlace ? 7 : 1); ++p) n += pn_pass_bytes(im, p);
    return n;
}

// The stored pixel (sy, sx): its pass, and its row and column in that pass.
B2P_PN_HD void pn_locate(int interlace, int sy, int sx, int* p, int* r, int* c) {
    if (!interlace) {
        *p = 0;
        *r = sy;
        *c = sx;
        return;
    }
    // pass of (sy % 8, sx % 8) in the Adam7 pattern
    const unsigned char pat[8][8] = {{0, 5, 3, 5, 1, 5, 3, 5}, {6, 6, 6, 6, 6, 6, 6, 6}, {4, 5, 4, 5, 4, 5, 4, 5},
                                     {6, 6, 6, 6, 6, 6, 6, 6}, {2, 5, 3, 5, 2, 5, 3, 5}, {6, 6, 6, 6, 6, 6, 6, 6},
                                     {4, 5, 4, 5, 4, 5, 4, 5}, {6, 6, 6, 6, 6, 6, 6, 6}};
    const int xs[7] = {0, 4, 0, 2, 0, 1, 0}, ys[7] = {0, 0, 4, 0, 2, 0, 1}, dx[7] = {8, 8, 4, 4, 2, 2, 1},
              dy[7] = {8, 8, 8, 4, 4, 2, 2};
    const int q = pat[sy & 7][sx & 7];
    *p = q;
    *r = (sy - ys[q]) / dy[q];
    *c = (sx - xs[q]) / dx[q];
}

// ---------------------------------------------------------------------------------------------- unfiltering
B2P_PN_HD unsigned pn_paeth(int a, int b, int c) {
    const int p = a + b - c;
    const int pa = p > a ? p - a : a - p, pb = p > b ? p - b : b - p, pc = p > c ? p - c : c - p;
    if (pa <= pb && pa <= pc) return (unsigned)a;
    if (pb <= pc) return (unsigned)b;
    return (unsigned)c;
}

// Reconstructs the bytes of one row that lane `lane` of `lanes` owns, in place: row[0 .. rb) follows its filter byte
// `type` (1 .. 4), prior is the row above, already reconstructed (null for a pass's first row).  Sub, Average and
// Paeth run along the row in steps of bpp, lane j < bpp owning bytes j, j + bpp, ...; Up is split over every lane.
B2P_PN_HD void pn_unfilter_lane(unsigned char* row, const unsigned char* prior, long long rb, int bpp, int type, int lane,
                                int lanes) {
    if (type == 2) {
        for (long long x = lane; x < rb; x += lanes) row[x] = (unsigned char)(row[x] + (prior ? prior[x] : 0));
        return;
    }
    if (lane >= bpp) return;
    for (long long x = lane; x < rb; x += bpp) {
        const int a = x >= bpp ? row[x - bpp] : 0, b = prior ? prior[x] : 0, c = prior && x >= bpp ? prior[x - bpp] : 0;
        unsigned v = row[x];
        if (type == 1) v += a;
        else if (type == 3) v += (unsigned)((a + b) >> 1);
        else v += pn_paeth(a, b, c);
        row[x] = (unsigned char)v;
    }
}

// ---------------------------------------------------------------------------------------------- colour
// Sample k of pixel c of a reconstructed row, as the 8-bit value cv2's transforms make of it (palette indices as read).
B2P_PN_HD unsigned pn_sample(const PngDecImage& im, const unsigned char* row, int c, int k) {
    const long long s = (long long)c * im.channels + k;
    if (im.depth == 16) return row[2 * s];
    if (im.depth == 8) return row[s];
    const long long bit = s * im.depth;
    const unsigned v = (row[bit >> 3] >> (8 - im.depth - (int)(bit & 7))) & ((1u << im.depth) - 1);
    if (im.ctype == 3) return v;
    return im.depth == 1 ? v * 255u : im.depth == 2 ? v * 85u : v * 17u;
}

// Output pixel (y, x) of the oriented frame from the reconstructed rows `rows` (filter bytes in place).
B2P_PN_HD void png_px(const PngDecImage& im, const unsigned char* rows, int y, int x, unsigned char* bgr) {
    int sy, sx, p, r, c;
    fr_source_pixel(im.h, im.w, im.rot, y, im.mirror ? im.ow - 1 - x : x, &sy, &sx);
    pn_locate(im.interlace, sy, sx, &p, &r, &c);
    long long off = 0;
    for (int q = 0; q < p; ++q) off += pn_pass_bytes(im, q);
    int ph, pw;
    pn_pass(im.interlace, p, im.h, im.w, &ph, &pw);
    const unsigned char* row = rows + off + (long long)r * (pn_rowbytes(im, pw) + 1) + 1;
    if (im.ctype == 3) {
        const unsigned i = pn_sample(im, row, c, 0);
        bgr[0] = im.pal[3 * i + 2];
        bgr[1] = im.pal[3 * i + 1];
        bgr[2] = im.pal[3 * i + 0];
    } else if (im.ctype == 2 || im.ctype == 6) {
        bgr[0] = (unsigned char)pn_sample(im, row, c, 2);
        bgr[1] = (unsigned char)pn_sample(im, row, c, 1);
        bgr[2] = (unsigned char)pn_sample(im, row, c, 0);
    } else {
        bgr[0] = bgr[1] = bgr[2] = (unsigned char)pn_sample(im, row, c, 0);
    }
}

// ---------------------------------------------------------------------------------------------- inflate
// A Huffman code in decoding form: lut[next 9 bits, LSB first] = (length << 9) | symbol for codes of <= 9 bits (0:
// longer, or no such code); count[l] codes of length l, sym[] the symbols in canonical order (puff.c's decode).
struct PngHuff {
    unsigned short lut[1 << kPngLutBits];
    unsigned short count[16];
    unsigned short sym[288];
};

// What the decoding lane hands the warp: a literal (kind 0, byte src), a match (kind 1, from output position src) or
// a stored run (kind 2, from zlib byte src); len output bytes at output position pos.
struct PngToken {
    long long pos, src;
    int len, kind;
};

enum { kPnHeader = 0, kPnHuff = 1, kPnStored = 2, kPnDone = 3, kPnCheck = 4 };
constexpr long long kPngIdatRead = 8192;      // libpng's IDAT_read_size: a chunk's data reaches inflate in such pieces
constexpr long long kPnNever = 1LL << 62;     // a bit position past any stream

// The decoding lane's state between rounds.
struct PngInflate {
    long long bp;                // next bit of the zlib stream
    long long out;               // bytes produced
    long long stored_src, stored_left;
    int state, final, wsize;
    unsigned status;
    int ended;                   // the final block ended with out == flen: the stream's Adler-32 is checked
    unsigned adler;              // ... its stored value
    PngHuff lit, dist;
    unsigned char lens[320];
};

// 32 bits of the stream from bit p (LSB first); bytes past the end read as zeros.
B2P_PN_HD unsigned pn_peek(const unsigned char* z, long long n, long long p) {
    const long long i = p >> 3;
    unsigned long long v = 0;
    for (int j = 4; j >= 0; --j) v = (v << 8) | (i + j < n ? z[i + j] : 0u);
    return (unsigned)(v >> (p & 7));
}

// inflate_table's checks and the decoding form of a code of n lengths.  type 0: code lengths, 1: literal/length,
// 2: distance.  Returns false for a code zlib refuses.
B2P_PN_HD bool pn_build(const unsigned char* lens, int n, int type, PngHuff& t) {
    for (int l = 0; l < 16; ++l) t.count[l] = 0;
    for (int s = 0; s < n; ++s) t.count[lens[s]]++;
    int max = 15;
    while (max >= 1 && t.count[max] == 0) --max;
    int left = 1;
    for (int l = 1; l <= 15; ++l) {
        left = (left << 1) - t.count[l];
        if (left < 0) return false;                              // over-subscribed
    }
    if (max > 0 && left > 0 && (type == 0 || max != 1)) return false;   // incomplete
    unsigned short offs[16];
    offs[1] = 0;
    for (int l = 1; l < 15; ++l) offs[l + 1] = (unsigned short)(offs[l] + t.count[l]);
    for (int s = 0; s < n; ++s)
        if (lens[s]) t.sym[offs[lens[s]]++] = (unsigned short)s;
    for (int i = 0; i < (1 << kPngLutBits); ++i) t.lut[i] = 0;
    unsigned code = 0;
    int k = 0;
    for (int l = 1; l <= 15; ++l) {
        for (int i = 0; i < t.count[l]; ++i, ++k, ++code)
            if (l <= kPngLutBits) {
                const unsigned r = png_reverse(code, l);
                for (unsigned f = r; f < (1u << kPngLutBits); f += 1u << l) t.lut[f] = (unsigned short)((l << 9) | t.sym[k]);
            }
        code <<= 1;
    }
    t.count[0] = 0;
    return true;
}

// Decodes one symbol at bit *bp; -1 for a bit pattern that is no code.
B2P_PN_HD int pn_decode(const PngHuff& t, const unsigned char* z, long long n, long long* bp) {
    const unsigned bits = pn_peek(z, n, *bp);
    const unsigned e = t.lut[bits & ((1u << kPngLutBits) - 1)];
    if (e) {
        *bp += e >> 9;
        return (int)(e & 511);
    }
    int code = 0, first = 0, index = 0;
    for (int l = 1; l <= 15; ++l) {
        code |= (int)((bits >> (l - 1)) & 1u);
        const int count = t.count[l];
        if (code - count < first) {
            *bp += l;
            return t.sym[index + (code - first)];
        }
        index += count;
        first = (first + count) << 1;
        code <<= 1;
    }
    return -1;
}

B2P_PN_HD int pn_len_base(int i) {
    const unsigned short b[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115,
                                  131, 163, 195, 227, 258};
    return b[i];
}
B2P_PN_HD int pn_len_xbits(int i) { return i < 8 || i == 28 ? 0 : (i - 4) / 4; }
B2P_PN_HD int pn_dist_base(int i) {
    const unsigned short b[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025,
                                  1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
    return b[i];
}
B2P_PN_HD int pn_dist_xbits(int i) { return i < 4 ? 0 : i / 2 - 1; }

B2P_PN_HD unsigned pn_bits(const unsigned char* z, long long n, long long* bp, int k) {
    const unsigned v = k ? pn_peek(z, n, *bp) & ((1u << k) - 1) : 0u;
    *bp += k;
    return v;
}

// The zlib header: false when zlib refuses it.  Sets the window and the first block's bit.
B2P_PN_HD bool pn_zlib_header(PngInflate& s, const unsigned char* z, long long n) {
    s = PngInflate{};
    s.bp = 16;
    if (n < 2) {
        s.status = kPngShortData;
        s.state = kPnDone;
        return false;
    }
    const unsigned cmf = z[0], flg = z[1];
    if ((cmf * 256 + flg) % 31 || (cmf & 15) != 8 || (cmf >> 4) > 7 || (flg & 0x20)) {
        s.status = kPngBadDeflate;
        s.state = kPnDone;
        return false;
    }
    s.wsize = 1 << ((cmf >> 4) + 8);
    s.state = kPnHeader;
    return true;
}

B2P_PN_HD int pn_fail(PngInflate& s, unsigned bit) {
    s.status |= bit;
    s.state = kPnDone;
    return 0;
}

// A block header, with the dynamic block's code lengths: the tables in s.lit / s.dist.  Returns false on an error
// (s.status set).
B2P_PN_HD bool pn_block_header(PngInflate& s, const unsigned char* z, long long n) {
    s.final = (int)pn_bits(z, n, &s.bp, 1);
    const int type = (int)pn_bits(z, n, &s.bp, 2);
    if (type == 0) {
        s.bp = (s.bp + 7) & ~7LL;
        const unsigned len = pn_bits(z, n, &s.bp, 16), nlen = pn_bits(z, n, &s.bp, 16);
        if (s.bp > 8 * n) return pn_fail(s, kPngShortData);
        if (len != (~nlen & 0xFFFFu)) return pn_fail(s, kPngBadDeflate);
        s.stored_src = s.bp >> 3;
        s.stored_left = len;
        s.state = kPnStored;
        return true;
    }
    if (type == 3) return pn_fail(s, kPngBadDeflate);
    unsigned char* L = s.lens;
    int nlen = 288, ndist = 32;
    if (type == 1) {
        for (int i = 0; i < 288; ++i) L[i] = (unsigned char)(i < 144 ? 8 : i < 256 ? 9 : i < 280 ? 7 : 8);
        for (int i = 0; i < 32; ++i) L[288 + i] = 5;
    } else {
        nlen = (int)pn_bits(z, n, &s.bp, 5) + 257;
        ndist = (int)pn_bits(z, n, &s.bp, 5) + 1;
        const int ncode = (int)pn_bits(z, n, &s.bp, 4) + 4;
        if (nlen > 286 || ndist > 30) return pn_fail(s, kPngBadDeflate);
        unsigned char cl[19] = {0};
        for (int i = 0; i < ncode; ++i) cl[png_bl_order(i)] = (unsigned char)pn_bits(z, n, &s.bp, 3);
        if (s.bp > 8 * n) return pn_fail(s, kPngShortData);
        if (!pn_build(cl, 19, 0, s.dist)) return pn_fail(s, kPngBadDeflate);
        int have = 0;
        while (have < nlen + ndist) {
            const int sym = pn_decode(s.dist, z, n, &s.bp);
            if (s.bp > 8 * n) return pn_fail(s, kPngShortData);
            if (sym < 0) return pn_fail(s, kPngBadDeflate);
            if (sym < 16) {
                L[have++] = (unsigned char)sym;
                continue;
            }
            int len = 0, copy;
            if (sym == 16) {
                if (have == 0) return pn_fail(s, kPngBadDeflate);
                len = L[have - 1];
                copy = 3 + (int)pn_bits(z, n, &s.bp, 2);
            } else if (sym == 17) {
                copy = 3 + (int)pn_bits(z, n, &s.bp, 3);
            } else {
                copy = 11 + (int)pn_bits(z, n, &s.bp, 7);
            }
            if (s.bp > 8 * n) return pn_fail(s, kPngShortData);
            if (have + copy > nlen + ndist) return pn_fail(s, kPngBadDeflate);
            while (copy--) L[have++] = (unsigned char)len;
        }
        if (L[256] == 0) return pn_fail(s, kPngBadDeflate);
        // the distance lengths follow the literal/length ones
        for (int i = ndist - 1; i >= 0; --i) L[288 + i] = L[nlen + i];
        for (int i = nlen; i < 288; ++i) L[i] = 0;
    }
    if (!pn_build(L, type == 1 ? 288 : nlen, 1, s.lit) || !pn_build(L + 288, type == 1 ? 32 : ndist, 2, s.dist))
        return pn_fail(s, kPngBadDeflate);
    s.state = kPnHuff;
    return true;
}

// The end (byte) of the piece of zlib data that holds byte x: libpng hands inflate a chunk's data in pieces of at most
// kPngIdatRead bytes.  ch: the image's IDAT chunks (PngIdat::dst, len); kPnNever when x is past the data.
B2P_PN_HD long long pn_piece_end(const PngIdat* ch, int nch, long long x) {
    for (int i = 0; i < nch; ++i) {
        const long long e = ch[i].dst + ch[i].len;
        if (x < e) {
            const long long k = ch[i].dst + ((x - ch[i].dst) / kPngIdatRead + 1) * kPngIdatRead;
            return k < e ? k : e;
        }
    }
    return kPnNever;
}

// One step of inflate's state machine after the last row, decoded from s without output: the bit at which it is
// complete (or its error found; kPnNever when its bits run past the data), the output it makes (a stored run makes
// it from bit `start` on), whether it is invalid data, a distance past the output (found only when inflate has room
// to copy), or the stream's Adler-32.
struct PnStep {
    long long end, start, out;
    int err, far, check;
};

B2P_PN_HD PnStep pn_tail_step(PngInflate& s, const unsigned char* z, long long n, long long out) {
    PnStep t{0, 0, 0, 0, 0, 0};
    const long long lim = 8 * n;
    if (s.state == kPnCheck) {
        s.bp = (s.bp + 7) & ~7LL;
        t.check = 1;
        t.end = s.bp + 32 > lim ? kPnNever : s.bp + 32;
        s.state = kPnDone;
        return t;
    }
    if (s.state == kPnHeader) {
        const unsigned keep = s.status;
        s.status = 0;
        const bool ok = pn_block_header(s, z, n);
        const unsigned found = s.status;
        s.status = keep;
        t.end = s.bp > lim || (found & kPngShortData) ? kPnNever : s.bp;
        t.err = !ok && t.end != kPnNever;
        return t;
    }
    if (s.state == kPnStored) {
        if (s.stored_left == 0) {
            s.bp = s.stored_src * 8;
            s.state = s.final ? kPnCheck : kPnHeader;
            t.end = s.bp;
            return t;
        }
        t.start = s.stored_src * 8;
        t.out = s.stored_left;
        t.end = s.stored_src + s.stored_left > n ? kPnNever : (s.stored_src + s.stored_left) * 8;
        s.stored_src += s.stored_left;
        s.stored_left = 0;
        return t;
    }
    const long long b0 = s.bp;
    const int sym = pn_decode(s.lit, z, n, &s.bp);
    if (sym < 0 || sym > 285) {
        t.end = sym < 0 ? b0 + 1 : s.bp;     // an empty or one-code table's missing code is 1 bit long
        if (t.end > lim) t.end = kPnNever;
        t.err = t.end != kPnNever;
        s.state = kPnDone;
        return t;
    }
    if (sym < 256) {
        t.out = 1;
    } else if (sym == 256) {
        s.state = s.final ? kPnCheck : kPnHeader;
    } else {
        const int li = sym - 257;
        t.out = pn_len_base(li) + (int)pn_bits(z, n, &s.bp, pn_len_xbits(li));
        const long long b1 = s.bp;
        const int dsym = pn_decode(s.dist, z, n, &s.bp);
        if (dsym < 0 || dsym > 29) {
            t.end = dsym < 0 ? b1 + 1 : s.bp;
            if (t.end > lim) t.end = kPnNever;
            t.err = t.end != kPnNever;
            s.state = kPnDone;
            return t;
        }
        const long long d = pn_dist_base(dsym) + pn_bits(z, n, &s.bp, pn_dist_xbits(dsym));
        t.far = d > out || d > s.wsize;
    }
    t.end = s.bp > lim ? kPnNever : s.bp;
    return t;
}

// What libpng makes of the zlib data once the last row is complete (png_read_IDAT_data, png_read_finish_IDAT), from
// state s right after the step that completed it; rest: bytes of that step's match past the last row.
//  1. The inflate call that completed the last row goes on without room for output until it needs output or runs out
//     of its piece: an error found there is fatal, and the final block's end there checks the Adler-32.
//  2. Then inflate runs into a scratch buffer, one piece at a time: it stops at the stream's end, at any error (a
//     warning), or after a piece that made no output, and fails ("Not enough image data") when it needs another piece
//     and none is left.
B2P_PN_HD void pn_tail(PngInflate& s, const unsigned char* z, long long n, const PngIdat* ch, int nch, int rest) {
    long long pulled = s.state == kPnStored ? s.stored_src : (s.bp + 7) >> 3;     // bytes inflate has taken in
    const long long E = pn_piece_end(ch, nch, pulled - 1);
    long long out = s.out, extra = 0;
    PnStep t{s.bp, 0, rest, 0, 0, 0};
    if (!rest) {
        for (;;) {
            t = pn_tail_step(s, z, n, out);
            if (t.end > E * 8) {
                pulled = E;
                break;
            }
            if (t.out) {
                pulled = ((t.start ? t.start : t.end) + 7) >> 3;
                break;
            }
            if (t.err) {
                pn_fail(s, kPngBadDeflate);
                return;
            }
            if (t.check) {
                const long long i = t.end / 8 - 4;
                s.adler = (unsigned)z[i] << 24 | (unsigned)z[i + 1] << 16 | (unsigned)z[i + 2] << 8 | z[i + 3];
                s.ended = 1;
                s.state = kPnDone;
                return;
            }
        }
    }
    long long F = E;
    for (int it = 0;; ++it) {
        if (it > 0 && extra == 0) break;                // a piece that made no output ends the reading
        if (pulled >= F) {                              // the piece is used up: the next one, or none is left
            if (F >= n) {
                pn_fail(s, kPngShortData);
                return;
            }
            F = pn_piece_end(ch, nch, F);
        }
        while (t.end <= F * 8) {
            if (t.err || t.far || t.check) {             // the stream's end, or an error that is only a warning here
                s.state = kPnDone;
                return;
            }
            extra += t.out;
            out += t.out;
            t = pn_tail_step(s, z, n, out);
        }
        if (t.out && t.start < F * 8) extra += 1;       // a stored run copies what the piece holds
        pulled = F;
    }
    s.state = kPnDone;
}

// One round of the decoding lane: up to kPngTokens tokens of output below flen.  Once the last row is complete, the
// rest of the stream is judged as libpng judges it (pn_tail).  ch: the image's IDAT chunks.  Returns the tokens
// written to tok.
B2P_PN_HD int pn_inflate_round(PngInflate& s, const unsigned char* z, long long n, long long flen, const PngIdat* ch,
                               int nch, PngToken* tok) {
    int nt = 0;
    while (nt < kPngTokens && s.state != kPnDone) {
        if (s.state == kPnHeader) {
            if (!pn_block_header(s, z, n)) break;
            continue;
        }
        if (s.state == kPnStored) {
            if (s.stored_left == 0) {
                s.state = kPnHeader;
                s.bp = s.stored_src * 8;
                if (s.final) goto stream_end;
                continue;
            }
            long long len = s.stored_left < flen - s.out ? s.stored_left : flen - s.out;
            if (s.stored_src + len > n) {
                pn_fail(s, kPngShortData);
                break;
            }
            tok[nt++] = PngToken{s.out, s.stored_src, (int)len, 2};
            s.out += len;
            s.stored_src += len;
            s.stored_left -= len;
            if (s.out == flen) pn_tail(s, z, n, ch, nch, 0);
            continue;
        }
        {
            const int sym = pn_decode(s.lit, z, n, &s.bp);
            if (sym < 0 || sym > 285) {
                pn_fail(s, sym < 0 && s.bp + 15 > 8 * n ? kPngShortData : kPngBadDeflate);
                break;
            }
            if (sym == 256) {
                if (s.bp > 8 * n) {
                    pn_fail(s, kPngShortData);
                    break;
                }
                s.state = kPnHeader;
                if (s.final) goto stream_end;
                continue;
            }
            int len = 1;
            long long src = sym;
            int kind = 0;
            if (sym > 256) {
                const int li = sym - 257;
                len = pn_len_base(li) + (int)pn_bits(z, n, &s.bp, pn_len_xbits(li));
                const int dsym = pn_decode(s.dist, z, n, &s.bp);
                if (dsym < 0 || dsym > 29) {
                    pn_fail(s, s.bp > 8 * n ? kPngShortData : kPngBadDeflate);
                    break;
                }
                const long long d = pn_dist_base(dsym) + pn_bits(z, n, &s.bp, pn_dist_xbits(dsym));
                if (s.bp > 8 * n) {
                    pn_fail(s, kPngShortData);
                    break;
                }
                if (d > s.out || d > s.wsize) {
                    pn_fail(s, kPngBadDeflate);
                    break;
                }
                src = s.out - d;
                kind = 1;
            } else if (s.bp > 8 * n) {
                pn_fail(s, kPngShortData);
                break;
            }
            const int rest = len > flen - s.out ? len - (int)(flen - s.out) : 0;
            tok[nt++] = PngToken{s.out, src, len - rest, kind};
            s.out += len - rest;
            if (s.out == flen) pn_tail(s, z, n, ch, nch, rest);
        }
        continue;
    stream_end:
        pn_fail(s, kPngShortData);     // the stream ends before the last row
    }
    return nt;
}

// Writes output byte j of token t (j < t.len): literals and stored runs at once, a match as
// out[p + j] = out[p - d + (j mod d)], which reads only bytes before p.
B2P_PN_HD void pn_token_byte(const PngToken& t, int j, const unsigned char* z, unsigned char* out) {
    if (t.kind == 0) out[t.pos] = (unsigned char)t.src;
    else if (t.kind == 2) out[t.pos + j] = z[t.src + j];
    else {
        const long long d = t.pos - t.src;
        out[t.pos + j] = out[t.src + j % d];
    }
}

}  // namespace b2p

// ================================================================================================ host-side parse
namespace b2p {

struct PngParsed {
    bool supported = false;
    char reason[200] = {0};
    int h = 0, w = 0, orientation = 0;
    PngDecImage im{};
    std::vector<PngIdat> idat;   // src: offset of the chunk's type in the stream; dst: from the image's zlib start
    long long zlen = 0;
};

inline bool pn_fail_parse(PngParsed* P, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(P->reason, sizeof(P->reason), fmt, ap);
    va_end(ap);
    return false;
}

inline unsigned pn_be32(const unsigned char* p) { return (unsigned)p[0] << 24 | (unsigned)p[1] << 16 | (unsigned)p[2] << 8 | p[3]; }

inline unsigned pn_crc(const unsigned char* p, long long n) {
    unsigned c = 0xFFFFFFFFu;
    for (long long i = 0; i < n; ++i) c = png_crc_entry((c ^ p[i]) & 0xFFu) ^ (c >> 8);
    return c ^ 0xFFFFFFFFu;
}

// Walks a whole stream.  Returns false for a malformed stream (reason set); else P->supported tells whether the device
// decodes it (reason: why not).  max_pixels bounds h * w.
inline bool png_parse(const unsigned char* d, long long n, long long max_pixels, PngParsed* P) {
    *P = PngParsed{};
    const unsigned char sig[8] = {0x89, 'P', 'N', 'G', 0x0D, 0x0A, 0x1A, 0x0A};
    if (!d || n < 8 || memcmp(d, sig, 8)) return pn_fail_parse(P, "not a PNG stream (no signature)");
    PngDecImage& im = P->im;
    bool ihdr = false, plte = false, idat_open = false, idat_done = false, iend = false, exif = false, apng = false;
    long long i = 8;
    while (i < n) {
        if (i + 12 > n) return pn_fail_parse(P, "malformed: chunk header at byte %lld runs past the end", i);
        const long long len = pn_be32(d + i);
        const unsigned char* t = d + i + 4;
        char name[5] = {(char)t[0], (char)t[1], (char)t[2], (char)t[3], 0};
        if (len > 0x7FFFFFFFLL || i + 12 + len > n)
            return pn_fail_parse(P, "malformed: chunk %s of %lld bytes runs past the end", name, len);
        for (int k = 0; k < 4; ++k)
            if (!((t[k] >= 'A' && t[k] <= 'Z') || (t[k] >= 'a' && t[k] <= 'z')))
                return pn_fail_parse(P, "malformed: invalid chunk type at byte %lld", i + 4);
        const unsigned char* s = t + 4;
        const bool critical = !(t[0] & 0x20), crc_ok = pn_crc(t, len + 4) == pn_be32(s + len);
        const bool is_idat = !memcmp(t, "IDAT", 4);
        if (!ihdr && memcmp(t, "IHDR", 4)) return pn_fail_parse(P, "malformed: the first chunk is %s, not IHDR", name);
        if (critical && !is_idat && !crc_ok) return pn_fail_parse(P, "malformed: CRC error in chunk %s", name);
        if (idat_open && !is_idat) {
            idat_open = false;
            idat_done = true;
        }
        if (!memcmp(t, "IHDR", 4)) {
            if (ihdr) return pn_fail_parse(P, "malformed: a second IHDR");
            if (len != 13) return pn_fail_parse(P, "malformed: IHDR of %lld bytes", len);
            const unsigned w = pn_be32(s), h = pn_be32(s + 4);
            const int depth = s[8], ct = s[9];
            // libpng's default user limits refuse a side beyond 1 000 000 pixels
            if (w < 1 || h < 1 || w > 1000000u || h > 1000000u) return pn_fail_parse(P, "malformed: IHDR size %u x %u", w, h);
            const bool pair = (ct == 0 && (depth == 1 || depth == 2 || depth == 4 || depth == 8 || depth == 16)) ||
                              (ct == 3 && (depth == 1 || depth == 2 || depth == 4 || depth == 8)) ||
                              ((ct == 2 || ct == 4 || ct == 6) && (depth == 8 || depth == 16));
            if (!pair) return pn_fail_parse(P, "malformed: IHDR colour type %d with bit depth %d", ct, depth);
            if (s[10] || s[11] || s[12] > 1)
                return pn_fail_parse(P, "malformed: IHDR methods %d / %d / %d", s[10], s[11], s[12]);
            if ((long long)w * h > max_pixels)
                return pn_fail_parse(P, "%u x %u pixels: a frame has 1 .. %lld pixels", h, w, max_pixels);
            P->h = im.h = (int)h;
            P->w = im.w = (int)w;
            im.depth = depth;
            im.ctype = ct;
            im.interlace = s[12];
            im.channels = pn_channels(ct);
            im.bpp = im.channels * depth >= 8 ? im.channels * depth / 8 : 1;
            ihdr = true;
        } else if (!memcmp(t, "PLTE", 4)) {
            // only a palette image uses PLTE; libpng passes over it in the other colour types with a warning
            if (im.ctype == 3) {
                if (plte) return pn_fail_parse(P, "malformed: a second PLTE");
                if (idat_open || idat_done) return pn_fail_parse(P, "malformed: PLTE after IDAT");
                if (len % 3 || len < 3 || len > 768) return pn_fail_parse(P, "malformed: PLTE of %lld bytes", len);
                memcpy(im.pal, s, (size_t)len);
                plte = true;
            }
        } else if (is_idat) {
            if (idat_done) return pn_fail_parse(P, "malformed: IDAT chunks are not consecutive");
            if (im.ctype == 3 && !plte) return pn_fail_parse(P, "malformed: a palette image without PLTE");
            idat_open = true;
            P->idat.push_back(PngIdat{0, pn_be32(s + len), i + 4, len, P->zlen});
            P->zlen += len;
        } else if (!memcmp(t, "IEND", 4)) {
            iend = true;
            break;
        } else if (!memcmp(t, "acTL", 4)) {
            apng = true;
        } else if (!memcmp(t, "eXIf", 4)) {
            if (crc_ok && !exif) {
                exif = true;
                const int o = jpeg_exif_orientation(s, (size_t)len);
                if (o >= 0) P->orientation = o;
            }
        } else if (critical) {
            return pn_fail_parse(P, "malformed: unknown critical chunk %s", name);
        }
        i += 12 + len;
    }
    if (!ihdr) return pn_fail_parse(P, "malformed: no IHDR");
    if (P->idat.empty()) return pn_fail_parse(P, "malformed: no IDAT");
    if (!iend) return pn_fail_parse(P, "malformed: no IEND");
    jpeg_orientation(P->orientation, &im.rot, &im.mirror);
    fr_rotated_size(im.h, im.w, im.rot, &im.oh, &im.ow);
    im.flen = pn_filtered_bytes(im);
    if (apng) {
        snprintf(P->reason, sizeof(P->reason), "unsupported: APNG (acTL)");
        return true;
    }
    P->supported = true;
    return true;
}

}  // namespace b2p
