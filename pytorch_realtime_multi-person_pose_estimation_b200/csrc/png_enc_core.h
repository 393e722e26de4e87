// PNG encoding, host/device shared core: packed uint8 HWC BGR frames -> PNG files, byte for byte
//   cv2.imencode('.png', frame)
//   (OpenCV 4.13 with libpng 1.6 and zlib 1.3 at cv2's defaults: compression level 1, strategy Z_RLE, Sub filter).
// What libpng and zlib compute on that path, restated (DESIGN.md 2.15):
//  * the rows as R, G, B (png_set_bgr), each behind filter byte 1 (Sub): f[x] = raw[x] - raw[x - 3] mod 256 (filter
//    byte 0, None, when the frame is one pixel wide);
//  * deflate_rle's parse, in closed form over the maximal runs of equal filtered bytes (runs cross rows): a run of L
//    bytes is one literal, (L - 1) / 258 matches of 258 at distance 1, then one match of r = (L - 1) % 258 when r >= 3,
//    else r literals (png_symbol_at);
//  * a block after every 16 383 symbols (lit_bufsize - 1 at memLevel 8), and the final block always, even empty;
//  * trees.c per block: build_tree (heap with the depth tie-break, the forced second code), gen_bitlen (length limit
//    15, 7 for the code-length tree, and the overflow fix-up), gen_codes, scan_tree / send_tree (codes 16, 17, 18),
//    the bl_order trim, and _tr_flush_block's choice between stored, static and dynamic by its own size estimates;
//  * zlib's header with libpng's CINFO rewrite for images of at most 16 384 filtered bytes, Adler-32;
//  * IDAT chunks of 8 192 bytes (libpng's zbuf size) behind the signature and IHDR, CRC-32 on each chunk, IEND.
// zlib keeps a block stored only while its start is still in the window; that condition never decides here (a stored
// block covers at most about 21 100 bytes, the window slides a block start out only past 32 506: DESIGN.md 2.15).
// The work is split the way the kernels of png_enc.cu run it: per filtered byte the byte and whether a run starts
// there, per byte the symbol that starts there (from its run's start and end), per block the trees, per image the
// block offsets, per symbol group the codes, per chunk the framing.  tests/cuda/png_enc_core_host.cpp runs the same
// steps.
#pragma once

#if defined(__CUDACC__)
#define B2P_PN_HD __host__ __device__ __forceinline__
#else
#define B2P_PN_HD inline
#endif

namespace b2p {

constexpr int kPngBlockSymbols = 16383;   // symbols per deflate block: lit_bufsize - 1 at memLevel 8
constexpr int kPngChunk = 8192;           // IDAT data bytes per chunk: libpng's zbuf size
constexpr int kPngTile = 2048;            // filtered bytes per tile of the per-byte kernels
constexpr int kPngLCodes = 286, kPngDCodes = 30, kPngBlCodes = 19, kPngHeap = 2 * kPngLCodes + 1;
constexpr int kPngAdlerMod = 65521;
constexpr long long kPngFraming = 8 + 25 + 12;   // signature, IHDR and IEND; each IDAT chunk adds 12
enum { kPngStored = 0, kPngStatic = 1, kPngDynamic = 2 };   // deflate BTYPE

// One image of an encode batch (device-resident descriptor).
struct PngImage {
    int h, w;
    long long n;          // filtered bytes, h (3w + 1)
    long long src;        // byte offset of the BGR frame in the input
    long long f0;         // its filtered bytes and symbols in the batch buffers
    long long tile0;      // its first tile in the batch tile arrays
    long long blk0;       // its first block slot
    int tiles, max_blocks;
    unsigned char zhdr[2];
};

// What the kernels find out about an image (device-resident, zeroed before a call).
struct PngImageOut {
    unsigned long long adler[2];   // sum of bytes, sum of (n - p) * byte[p], each taken mod 65521 per thread
    long long symbols;             // deflate symbols
    long long bits;                // deflate bits before the final byte alignment
    long long size;                // the PNG file's bytes
    int blocks, chunks;
};

// One deflate block as _tr_flush_block sends it: its type and the codes it uses.
struct PngBlock {
    long long sym0, nsym;          // its symbols (image-relative)
    long long bytes;               // filtered bytes it covers (stored_len)
    long long byte0, off;          // its first byte and the bit its header starts at (set per image afterwards)
    long long bits;                // after the 3-bit header: trees and codes, or 32 + 8 bytes (stored; alignment apart)
    int type, last, tree_bits;
    int lmax, dmax, blindex;       // HLIT - 257 + 256 (the highest lit/len code sent), dist codes - 1, max_blindex
    unsigned short lcode[kPngLCodes], blcode[kPngBlCodes];
    unsigned char llen[kPngLCodes], bllen[kPngBlCodes], dlen[kPngDCodes];
    unsigned short dcode0;         // the code of distance 1
};

// ---------------------------------------------------------------------------------------------- filter and parse
// Filtered byte p of the image (h x w BGR frame): row p / (3w + 1), byte 0 of a row the filter type - Sub, or None
// for a frame one pixel wide (png_write_start_row drops Sub there, and Sub of one pixel is the pixel).
B2P_PN_HD unsigned png_raw(const unsigned char* frame, int w, long long row, long long x) {
    return frame[(row * w + x / 3) * 3 + 2 - x % 3];
}
B2P_PN_HD unsigned png_filtered(const unsigned char* frame, int w, long long p) {
    const long long rb = 3LL * w + 1, row = p / rb, col = p - row * rb;
    if (col == 0) return w == 1 ? 0u : 1u;
    const long long x = col - 1;
    const unsigned v = png_raw(frame, w, row, x);
    return x < 3 ? v : (v - png_raw(frame, w, row, x - 3)) & 255u;
}

// The symbol deflate_rle emits at byte p (value `byte`) of the run [s, e), or -1 when p is inside a symbol: a literal
// (0 .. 255), or 256 + (length - 3) for a match at distance 1.
B2P_PN_HD int png_symbol_at(long long p, long long s, long long e, unsigned byte) {
    const long long k = p - s;
    if (k == 0) return (int)byte;
    const long long j = k - 1, full = (e - s - 1) / 258;
    const int r = (int)((e - s - 1) % 258);
    if (j < full * 258) return j % 258 == 0 ? 256 + 255 : -1;
    if (r >= 3) return j == full * 258 ? 256 + r - 3 : -1;
    return (int)byte;
}

// Filtered bytes a symbol covers.
B2P_PN_HD int png_sym_bytes(int sym) { return sym < 256 ? 1 : sym - 256 + 3; }

// Length code (0 .. 28) of match length - 3 (zlib's _length_code), its extra bits and base.
B2P_PN_HD int png_len_code(int lc) {
    if (lc < 8) return lc;
    if (lc == 255) return 28;
    int e = 0;
    while ((lc >> (e + 3)) != 0) ++e;
    return 4 * (e + 1) + ((lc >> e) & 3);
}
B2P_PN_HD int png_len_extra(int code) { return code < 8 || code == 28 ? 0 : (code - 4) / 4; }
B2P_PN_HD int png_len_base(int code) { return code < 8 ? code : code == 28 ? 255 : (4 + (code & 3)) << png_len_extra(code); }

// Blocks of an image of `symbols` symbols: full blocks, then the final one (empty when the last full block ended the
// data: deflate_rle's FLUSH_BLOCK(s, 1) runs whatever is left).
B2P_PN_HD long long png_blocks(long long symbols) { return symbols / kPngBlockSymbols + 1; }

// ---------------------------------------------------------------------------------------------- trees.c
// Tree kinds: 0 literal/length, 1 distance, 2 code lengths.
B2P_PN_HD int png_tree_elems(int kind) { return kind == 0 ? kPngLCodes : kind == 1 ? kPngDCodes : kPngBlCodes; }
B2P_PN_HD int png_static_len(int kind, int n) {
    if (kind == 1) return 5;
    return n < 144 ? 8 : n < 256 ? 9 : n < 280 ? 7 : 8;
}
// Extra bits of code n (extra_lbits from code 257, extra_dbits, extra_blbits).
B2P_PN_HD int png_xbits(int kind, int n) {
    if (kind == 0) return n < 257 ? 0 : png_len_extra(n - 257);
    if (kind == 1) return n < 4 ? 0 : n / 2 - 1;
    return n == 16 ? 2 : n == 17 ? 3 : n == 18 ? 7 : 0;
}

// ct_data of one tree with Freq / Code and Dad / Len kept apart (zlib overlays them; each is read only while valid).
struct PngTree {
    unsigned freq[kPngHeap];
    unsigned short dad[kPngHeap], len[kPngHeap], code[kPngHeap];
    int max_code;
};
struct PngHeap {
    int heap[kPngHeap];
    unsigned char depth[kPngHeap];
    int heap_len, heap_max;
    unsigned short bl_count[16];
};
struct PngTrees {
    PngTree l, d, bl;
    PngHeap hp;
};

B2P_PN_HD bool png_smaller(const PngTree& t, const PngHeap& hp, int n, int m) {
    return t.freq[n] < t.freq[m] || (t.freq[n] == t.freq[m] && hp.depth[n] <= hp.depth[m]);
}

B2P_PN_HD void png_downheap(const PngTree& t, PngHeap& hp, int k) {
    const int v = hp.heap[k];
    int j = k << 1;
    while (j <= hp.heap_len) {
        if (j < hp.heap_len && png_smaller(t, hp, hp.heap[j + 1], hp.heap[j])) j++;
        if (png_smaller(t, hp, v, hp.heap[j])) break;
        hp.heap[k] = hp.heap[j];
        k = j;
        j <<= 1;
    }
    hp.heap[k] = v;
}

B2P_PN_HD unsigned png_reverse(unsigned code, int len) {
    unsigned r = 0;
    for (int i = 0; i < len; ++i, code >>= 1) r = (r << 1) | (code & 1u);
    return r;
}

// gen_codes: the (bit-reversed) codes of lengths len[0 .. max_code] with bl_count[1 .. 15] codes of each length.
B2P_PN_HD void png_gen_codes(const unsigned short* len, int max_code, const unsigned short* bl_count, unsigned short* code) {
    unsigned short next[16];
    unsigned c = 0;
    for (int b = 1; b <= 15; ++b) {
        c = (c + bl_count[b - 1]) << 1;
        next[b] = (unsigned short)c;
    }
    for (int n = 0; n <= max_code; ++n)
        if (len[n]) code[n] = (unsigned short)png_reverse(next[len[n]]++, len[n]);
}

// build_tree with gen_bitlen and gen_codes: t.freq[0 .. elems - 1] holds the counts; opt_len and static_len
// accumulate as in zlib (including its adjustments for the forced codes).
B2P_PN_HD void png_build_tree(PngTree& t, PngHeap& hp, int kind, long long* opt_len, long long* static_len) {
    const int elems = png_tree_elems(kind), max_length = kind == 2 ? 7 : 15, base = kind == 0 ? 257 : 0;
    int max_code = -1;
    hp.heap_len = 0;
    hp.heap_max = kPngHeap;
    for (int n = 0; n < elems; ++n) {
        if (t.freq[n] != 0) {
            hp.heap[++hp.heap_len] = max_code = n;
            hp.depth[n] = 0;
        } else {
            t.len[n] = 0;
        }
    }
    // a tree needs two codes: the missing ones are forced in with frequency 1
    while (hp.heap_len < 2) {
        const int node = hp.heap[++hp.heap_len] = (max_code < 2 ? ++max_code : 0);
        t.freq[node] = 1;
        hp.depth[node] = 0;
        --*opt_len;
        if (kind != 2) *static_len -= png_static_len(kind, node);
    }
    t.max_code = max_code;
    for (int n = hp.heap_len / 2; n >= 1; --n) png_downheap(t, hp, n);
    int node = elems;
    do {
        const int n = hp.heap[1];
        hp.heap[1] = hp.heap[hp.heap_len--];
        png_downheap(t, hp, 1);
        const int m = hp.heap[1];
        hp.heap[--hp.heap_max] = n;
        hp.heap[--hp.heap_max] = m;
        t.freq[node] = t.freq[n] + t.freq[m];
        hp.depth[node] = (unsigned char)((hp.depth[n] >= hp.depth[m] ? hp.depth[n] : hp.depth[m]) + 1);
        t.dad[n] = t.dad[m] = (unsigned short)node;
        hp.heap[1] = node++;
        png_downheap(t, hp, 1);
    } while (hp.heap_len >= 2);
    hp.heap[--hp.heap_max] = hp.heap[1];
    // gen_bitlen
    for (int b = 0; b <= 15; ++b) hp.bl_count[b] = 0;
    t.len[hp.heap[hp.heap_max]] = 0;
    int overflow = 0;
    for (int h = hp.heap_max + 1; h < kPngHeap; ++h) {
        const int n = hp.heap[h];
        int bits = t.len[t.dad[n]] + 1;
        if (bits > max_length) {
            bits = max_length;
            ++overflow;
        }
        t.len[n] = (unsigned short)bits;
        if (n > max_code) continue;
        hp.bl_count[bits]++;
        const int xb = n >= base ? png_xbits(kind, n) : 0;
        *opt_len += (long long)t.freq[n] * (bits + xb);
        if (kind != 2) *static_len += (long long)t.freq[n] * (png_static_len(kind, n) + xb);
    }
    if (overflow != 0) {
        do {
            int bits = max_length - 1;
            while (hp.bl_count[bits] == 0) bits--;
            hp.bl_count[bits]--;
            hp.bl_count[bits + 1] += 2;
            hp.bl_count[max_length]--;
            overflow -= 2;
        } while (overflow > 0);
        int h = kPngHeap;
        for (int bits = max_length; bits != 0; bits--) {
            int n = hp.bl_count[bits];
            while (n != 0) {
                const int m = hp.heap[--h];
                if (m > max_code) continue;
                if (t.len[m] != bits) {
                    *opt_len += ((long long)bits - t.len[m]) * t.freq[m];
                    t.len[m] = (unsigned short)bits;
                }
                n--;
            }
        }
    }
    png_gen_codes(t.len, max_code, hp.bl_count, t.code);
}

// scan_tree / send_tree: the code-length codes of len[0 .. max_code], each handed to emit(code, extra, extra_bits).
template <class Len, class Emit> B2P_PN_HD void png_walk_tree(const Len* len, int max_code, Emit emit) {
    int prevlen = -1, nextlen = len[0], count = 0, max_count = 7, min_count = 4;
    if (nextlen == 0) max_count = 138, min_count = 3;
    for (int n = 0; n <= max_code; n++) {
        const int curlen = nextlen;
        nextlen = n + 1 <= max_code ? len[n + 1] : 0xffff;     // the guard zlib stores behind max_code
        if (++count < max_count && curlen == nextlen) continue;
        if (count < min_count) {
            do emit(curlen, 0, 0);
            while (--count != 0);
        } else if (curlen != 0) {
            if (curlen != prevlen) {
                emit(curlen, 0, 0);
                count--;
            }
            emit(16, count - 3, 2);
        } else if (count <= 10) {
            emit(17, count - 3, 3);
        } else {
            emit(18, count - 11, 7);
        }
        count = 0;
        prevlen = curlen;
        if (nextlen == 0) max_count = 138, min_count = 3;
        else if (curlen == nextlen) max_count = 6, min_count = 3;
        else max_count = 7, min_count = 4;
    }
}

B2P_PN_HD int png_bl_order(int i) {
    const unsigned char o[kPngBlCodes] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
    return o[i];
}

// _tr_flush_block for one block: lfreq[0 .. 285] the literal/length counts (END_BLOCK's 1 included), nmatch the
// distance-1 matches, `bytes` the filtered bytes it covers.  Fills B's type, codes and sizes (not sym0, byte0, off).
B2P_PN_HD void png_block_trees(const unsigned* lfreq, unsigned nmatch, long long bytes, bool last, PngTrees& w,
                               PngBlock& B) {
    long long opt_len = 0, static_len = 0;
    for (int n = 0; n < kPngLCodes; ++n) w.l.freq[n] = lfreq[n];
    for (int n = 0; n < kPngDCodes; ++n) w.d.freq[n] = 0;
    w.d.freq[0] = nmatch;
    for (int n = 0; n < kPngBlCodes; ++n) w.bl.freq[n] = 0;
    png_build_tree(w.l, w.hp, 0, &opt_len, &static_len);
    png_build_tree(w.d, w.hp, 1, &opt_len, &static_len);
    // build_bl_tree
    PngTree& bl = w.bl;
    auto count = [&bl](int c, int, int) { bl.freq[c]++; };
    png_walk_tree(w.l.len, w.l.max_code, count);
    png_walk_tree(w.d.len, w.d.max_code, count);
    long long bl_opt = 0, bl_static = 0;
    png_build_tree(bl, w.hp, 2, &bl_opt, &bl_static);
    int max_blindex = kPngBlCodes - 1;
    for (; max_blindex >= 3; max_blindex--)
        if (bl.len[png_bl_order(max_blindex)] != 0) break;
    const long long tree_bits = bl_opt + 3 * ((long long)max_blindex + 1) + 5 + 5 + 4;
    opt_len += tree_bits;
    // the choice, by zlib's byte estimates
    long long opt_lenb = (opt_len + 3 + 7) >> 3;
    const long long static_lenb = (static_len + 3 + 7) >> 3;
    if (static_lenb <= opt_lenb) opt_lenb = static_lenb;
    B.bytes = bytes;
    B.last = last;
    B.lmax = w.l.max_code;
    B.dmax = w.d.max_code;
    B.blindex = max_blindex;
    if (bytes + 4 <= opt_lenb) {
        B.type = kPngStored;
        B.tree_bits = 0;
        B.bits = 32 + 8 * bytes;
        return;
    }
    if (static_lenb == opt_lenb) {
        B.type = kPngStatic;
        B.tree_bits = 0;
        B.bits = static_len;
        for (int n = 0; n < kPngLCodes; ++n) {     // static_ltree: what gen_codes makes of the static lengths
            const int l = png_static_len(0, n);
            const unsigned c = n < 144 ? 0x30 + n : n < 256 ? 0x190 + n - 144 : n < 280 ? n - 256 : 0xC0 + n - 280;
            B.llen[n] = (unsigned char)l;
            B.lcode[n] = (unsigned short)png_reverse(c, l);
        }
        B.dcode0 = 0;
        B.dlen[0] = 5;
        return;
    }
    B.type = kPngDynamic;
    B.tree_bits = (int)tree_bits;
    B.bits = opt_len;
    for (int n = 0; n < kPngLCodes; ++n) {
        B.llen[n] = (unsigned char)(n <= w.l.max_code ? w.l.len[n] : 0);
        B.lcode[n] = B.llen[n] ? w.l.code[n] : 0;
    }
    for (int n = 0; n < kPngDCodes; ++n) B.dlen[n] = (unsigned char)(n <= w.d.max_code ? w.d.len[n] : 0);
    B.dcode0 = w.d.code[0];
    for (int n = 0; n < kPngBlCodes; ++n) {
        B.bllen[n] = (unsigned char)bl.len[n];
        B.blcode[n] = bl.len[n] ? bl.code[n] : 0;
    }
}

// ---------------------------------------------------------------------------------------------- code emission
// Bits of one symbol's codes in block B (literal, or length code + extra + distance code).
B2P_PN_HD int png_sym_bits(const PngBlock& B, int sym) {
    if (sym < 256) return B.llen[sym];
    const int c = png_len_code(sym - 256);
    return B.llen[257 + c] + png_len_extra(c) + B.dlen[0];
}

// compress_block for one symbol: its codes handed to put(bits, length), least significant bit first.
template <class Put> B2P_PN_HD void png_put_sym(const PngBlock& B, int sym, Put& put) {
    if (sym < 256) {
        put(B.lcode[sym], B.llen[sym]);
        return;
    }
    const int lc = sym - 256, c = png_len_code(lc), xb = png_len_extra(c);
    put(B.lcode[257 + c], B.llen[257 + c]);
    if (xb) put((unsigned)(lc - png_len_base(c)), xb);
    put(B.dcode0, B.dlen[0]);
}

// The block's header bits: the 3-bit block header and, for a dynamic block, send_all_trees.  A stored block's
// header, padding to the byte and LEN / NLEN are written from its header bit `off` (the padding depends on it).
template <class Put> B2P_PN_HD void png_put_head(const PngBlock& B, long long off, Put& put) {
    put((unsigned)((B.type << 1) + B.last), 3);
    if (B.type == kPngStored) {
        const int pad = (int)((8 - ((off + 3) & 7)) & 7);
        if (pad) put(0u, pad);
        put((unsigned)(B.bytes & 0xFFFF), 16);
        put((unsigned)(~B.bytes & 0xFFFF), 16);
        return;
    }
    if (B.type != kPngDynamic) return;
    put((unsigned)(B.lmax + 1 - 257), 5);
    put((unsigned)(B.dmax + 1 - 1), 5);
    put((unsigned)(B.blindex + 1 - 4), 4);
    for (int rank = 0; rank <= B.blindex; rank++) put(B.bllen[png_bl_order(rank)], 3);
    auto send = [&B, &put](int c, int extra, int xb) {
        put(B.blcode[c], B.bllen[c]);
        if (xb) put((unsigned)extra, xb);
    };
    png_walk_tree(B.llen, B.lmax, send);
    png_walk_tree(B.dlen, B.dmax, send);
}

// The bit a block after one starting at `off` starts at.
B2P_PN_HD long long png_block_end(const PngBlock& B, long long off) {
    if (B.type == kPngStored) return ((off + 3 + 7) & ~7LL) + B.bits;
    return off + 3 + B.bits;
}

// Bit writer into 32-bit words, least significant bit first, from bit `off`: words the writer fills alone are
// stored; its first and last word may be shared with its neighbours and go to store_shared (an OR into a zeroed word).
template <class Store, class StoreShared> struct PngBitWriter {
    unsigned long long acc;
    int n;
    long long wi;
    bool first;
    Store store;
    StoreShared shared;
    B2P_PN_HD PngBitWriter(long long off, Store s, StoreShared ss)
        : acc(0), n((int)(off & 31)), wi(off >> 5), first(true), store(s), shared(ss) {}
    B2P_PN_HD void operator()(unsigned bits, int len) {
        acc |= (unsigned long long)bits << n;
        n += len;
        if (n >= 32) {
            if (first) shared(wi, (unsigned)acc);
            else store(wi, (unsigned)acc);
            first = false;
            acc >>= 32;
            n -= 32;
            ++wi;
        }
    }
    B2P_PN_HD void finish() {
        if (n > 0) shared(wi, (unsigned)acc);
    }
};

// ---------------------------------------------------------------------------------------------- zlib and PNG framing
// zlib's header (level 1: FLEVEL 0, no dictionary) with libpng's optimize_cmf: at most 16 384 filtered bytes lower
// CINFO to the smallest window (256 bytes at least) that covers them.
B2P_PN_HD void png_zlib_header(long long n, unsigned char* hdr) {
    int cinfo = 7;
    if (n <= 16384) {
        cinfo = 0;
        while ((1LL << (cinfo + 8)) < n) ++cinfo;
    }
    const unsigned cmf = 8u | (unsigned)cinfo << 4;
    hdr[0] = (unsigned char)cmf;
    hdr[1] = (unsigned char)(0x1f - (cmf << 8) % 0x1f);
}

// Adler-32 of n bytes from sum(b) and sum((n - p) b), both mod 65521.
B2P_PN_HD unsigned png_adler(long long n, unsigned long long a, unsigned long long b) {
    const unsigned s1 = (unsigned)((1 + a) % kPngAdlerMod), s2 = (unsigned)((n % kPngAdlerMod + b) % kPngAdlerMod);
    return s2 << 16 | s1;
}

// The bytes of the zlib stream, and its length, from the deflate bits.
B2P_PN_HD long long png_zlib_bytes(long long bits) { return 2 + (bits + 7) / 8 + 4; }
B2P_PN_HD long long png_chunks(long long zbytes) { return (zbytes + kPngChunk - 1) / kPngChunk; }
B2P_PN_HD long long png_file_bytes(long long zbytes) { return kPngFraming + zbytes + 12 * png_chunks(zbytes); }

// Byte k of the zlib stream: header, deflate bytes (words, little-endian), Adler-32 big-endian.
B2P_PN_HD unsigned png_zbyte(const unsigned char* hdr, const unsigned* words, long long dbytes, unsigned adler, long long k) {
    if (k < 2) return hdr[k];
    k -= 2;
    if (k < dbytes) return (words[k >> 2] >> (8 * (k & 3))) & 0xFFu;
    return (adler >> (8 * (3 - (k - dbytes)))) & 0xFFu;
}

// CRC-32 (reflected 0xEDB88320): the table entry, one byte's update, and zlib's crc32_combine (multmodp, x2nmodp).
B2P_PN_HD unsigned png_crc_entry(unsigned c) {
    for (int k = 0; k < 8; ++k) c = c & 1u ? 0xEDB88320u ^ (c >> 1) : c >> 1;
    return c;
}
B2P_PN_HD unsigned png_multmodp(unsigned a, unsigned b) {
    unsigned m = 1u << 31, p = 0;
    for (;;) {
        if (a & m) {
            p ^= b;
            if ((a & (m - 1)) == 0) break;
        }
        m >>= 1;
        b = b & 1 ? (b >> 1) ^ 0xEDB88320u : b >> 1;
    }
    return p;
}
// CRC of A followed by B from crc(A), crc(B) and B's length.
B2P_PN_HD unsigned png_crc_combine(unsigned crc_a, unsigned crc_b, long long len_b) {
    unsigned p = 1u << 31, t = 1u << 23;   // x^0, x^8
    for (long long n = len_b; n; n >>= 1) {
        if (n & 1) p = png_multmodp(t, p);
        t = png_multmodp(t, t);
    }
    return png_multmodp(p, crc_a) ^ crc_b;
}

// The signature and IHDR (33 bytes) of an h x w RGB image.
B2P_PN_HD void png_head(int h, int w, unsigned char* o) {
    const unsigned char sig[8] = {0x89, 'P', 'N', 'G', 0x0D, 0x0A, 0x1A, 0x0A};
    for (int i = 0; i < 8; ++i) o[i] = sig[i];
    const unsigned char ihdr[21] = {0, 0, 0, 13, 'I', 'H', 'D', 'R',
                                    (unsigned char)(w >> 24), (unsigned char)(w >> 16), (unsigned char)(w >> 8), (unsigned char)w,
                                    (unsigned char)(h >> 24), (unsigned char)(h >> 16), (unsigned char)(h >> 8), (unsigned char)h,
                                    8, 2, 0, 0, 0};
    unsigned crc = 0xFFFFFFFFu;
    for (int i = 0; i < 21; ++i) {
        o[8 + i] = ihdr[i];
        if (i >= 4) crc = png_crc_entry((crc ^ ihdr[i]) & 0xFFu) ^ (crc >> 8);
    }
    crc ^= 0xFFFFFFFFu;
    for (int i = 0; i < 4; ++i) o[29 + i] = (unsigned char)(crc >> (24 - 8 * i));
}

// The IEND chunk (12 bytes).
B2P_PN_HD void png_tail(unsigned char* o) {
    const unsigned char t[12] = {0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xAE, 0x42, 0x60, 0x82};
    for (int i = 0; i < 12; ++i) o[i] = t[i];
}

// Stream bytes that always suffice for n filtered bytes: zlib's worst case for these parameters is every block
// stored (deflateBound's tighter formula assumes stored blocks of up to 64 KB; deflate_rle's hold 16 383 symbols),
// each block at most its stored size + 5 bytes: 3 header bits, padding, LEN and NLEN.
B2P_PN_HD long long png_stream_bound(int h, int w) {
    const long long n = (long long)h * (3LL * w + 1), z = 2 + n + 5 * png_blocks(n) + 4;
    return png_file_bytes(z);
}

}  // namespace b2p
