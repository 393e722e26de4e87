// Host build of the PNG encoding core (csrc/png_enc_core.h), split the way the kernels of png_enc.cu run it: per
// filtered byte the byte and its run start flag, per byte the symbol that starts there from its run's start and end,
// per block the histograms and trees, per image the block offsets, per symbol the codes packed into 32-bit words (a
// writer per block part: first and last word ORed, the words between stored), per chunk the framing and CRC (a CRC
// per 256-byte part, combined).  PNG_ENC_CORE overrides the header's path, so that a test can compile a copy with a
// planted mistake.
#ifndef PNG_ENC_CORE
#define PNG_ENC_CORE "../../pytorch_realtime_multi-person_pose_estimation_b200/csrc/png_enc_core.h"
#endif
#include PNG_ENC_CORE

#include <cstring>
#include <memory>
#include <vector>

using namespace b2p;

extern "C" long long core_encode_bound(int h, int w) {
    if (h < 1 || w < 1) return -1;
    return png_stream_bound(h, w);
}

// Encodes the h x w BGR frame into out (cap bytes).  Returns the file's size, or -1 for bad arguments, -2 when cap is
// below the bound.
extern "C" long long core_encode(const unsigned char* frame, int h, int w, unsigned char* out, long long cap) {
    if (!frame || h < 1 || w < 1 || h > 65535 || w > 65535) return -1;
    if (cap < png_stream_bound(h, w)) return -2;
    const long long n = (long long)h * (3LL * w + 1);
    // filter, run starts, Adler-32 partial sums (png_enc_filter_kernel)
    std::vector<unsigned char> f(n);
    std::vector<long long> start;
    unsigned long long a = 0, b = 0;
    for (long long p = 0; p < n; ++p) {
        f[p] = (unsigned char)png_filtered(frame, w, p);
        if (p == 0 || f[p] != (unsigned char)png_filtered(frame, w, p - 1)) start.push_back(p);
        a = (a + f[p]) % kPngAdlerMod;
        b = (b + (unsigned long long)((n - p) % kPngAdlerMod) * f[p]) % kPngAdlerMod;
    }
    start.push_back(n);
    // symbols from each byte's run (png_enc_count_kernel, png_enc_symbols_kernel)
    std::vector<unsigned short> sym;
    for (size_t r = 0; r + 1 < start.size(); ++r)
        for (long long p = start[r]; p < start[r + 1]; ++p) {
            const int s = png_symbol_at(p, start[r], start[r + 1], f[p]);
            if (s >= 0) sym.push_back((unsigned short)s);
        }
    // per block: histograms and trees (png_enc_tree_kernel)
    const long long S = (long long)sym.size(), nb = png_blocks(S);
    std::vector<PngBlock> blk(nb);
    std::unique_ptr<PngTrees> work(new PngTrees);
    for (long long k = 0; k < nb; ++k) {
        PngBlock& B = blk[k];
        B.sym0 = k * kPngBlockSymbols;
        B.nsym = (k + 1 < nb ? (k + 1) * kPngBlockSymbols : S) - B.sym0;
        unsigned lfreq[kPngLCodes] = {0}, nmatch = 0;
        long long bytes = 0;
        for (long long i = B.sym0; i < B.sym0 + B.nsym; ++i) {
            const int s = sym[i];
            bytes += png_sym_bytes(s);
            if (s < 256) {
                lfreq[s]++;
            } else {
                lfreq[257 + png_len_code(s - 256)]++;
                nmatch++;
            }
        }
        lfreq[256] = 1;
        png_block_trees(lfreq, nmatch, bytes, k + 1 == nb, *work, B);
    }
    // per image: block offsets (png_enc_layout_kernel)
    long long off = 0, byte0 = 0;
    for (long long k = 0; k < nb; ++k) {
        blk[k].off = off;
        blk[k].byte0 = byte0;
        off = png_block_end(blk[k], off);
        byte0 += blk[k].bytes;
    }
    const long long dbytes = (off + 7) / 8, zbytes = png_zlib_bytes(off), size = png_file_bytes(zbytes);
    // codes into words (png_enc_pack_kernel): the head, then the symbols in parts of 97 with END in the last part
    std::vector<unsigned> words((size_t)(off / 32 + 2), 0u);
    unsigned* wd = words.data();
    auto store = [wd](long long i, unsigned v) { wd[i] = v; };
    auto shared = [wd](long long i, unsigned v) { wd[i] |= v; };
    using Writer = PngBitWriter<decltype(store), decltype(shared)>;
    for (long long k = 0; k < nb; ++k) {
        const PngBlock& B = blk[k];
        Writer head(B.off, store, shared);
        png_put_head(B, B.off, head);
        head.finish();
        if (B.type == kPngStored) {
            const long long at = ((B.off + 3 + 7) & ~7LL) + 32;
            for (long long i0 = 0; i0 < B.bytes; i0 += 97) {
                Writer wr(at + 8 * i0, store, shared);
                for (long long i = i0; i < B.bytes && i < i0 + 97; ++i) wr(f[B.byte0 + i], 8);
                wr.finish();
            }
            continue;
        }
        long long at = B.off + 3 + B.tree_bits;
        for (long long i0 = 0; i0 <= B.nsym; i0 += 97) {
            Writer wr(at, store, shared);
            for (long long i = i0; i <= B.nsym && i < i0 + 97; ++i) {
                if (i == B.nsym) {
                    wr(B.lcode[256], B.llen[256]);
                    at += B.llen[256];
                } else {
                    png_put_sym(B, sym[B.sym0 + i], wr);
                    at += png_sym_bits(B, sym[B.sym0 + i]);
                }
            }
            wr.finish();
        }
    }
    // framing (png_enc_write_kernel)
    unsigned char zh[2];
    png_zlib_header(n, zh);
    const unsigned adler = png_adler(n, a, b);
    png_head(h, w, out);
    long long at = 33;
    unsigned table[256];
    for (unsigned c = 0; c < 256; ++c) table[c] = png_crc_entry(c);
    for (long long c = 0; c < png_chunks(zbytes); ++c) {
        const long long k0 = c * kPngChunk, len = (zbytes - k0 < kPngChunk ? zbytes - k0 : kPngChunk);
        unsigned char* o = out + at;
        o[0] = (unsigned char)(len >> 24), o[1] = (unsigned char)(len >> 16), o[2] = (unsigned char)(len >> 8);
        o[3] = (unsigned char)len;
        memcpy(o + 4, "IDAT", 4);
        for (long long k = 0; k < len; ++k) o[8 + k] = (unsigned char)png_zbyte(zh, wd, dbytes, adler, k0 + k);
        unsigned crc = 0;
        for (long long q0 = 0; q0 < 4 + len; q0 += 256) {
            const long long q1 = q0 + 256 < 4 + len ? q0 + 256 : 4 + len;
            unsigned part = 0xFFFFFFFFu;
            for (long long q = q0; q < q1; ++q) part = table[(part ^ o[4 + q]) & 0xFFu] ^ (part >> 8);
            crc = png_crc_combine(crc, part ^ 0xFFFFFFFFu, q1 - q0);
        }
        for (int i = 0; i < 4; ++i) o[8 + len + i] = (unsigned char)(crc >> (24 - 8 * i));
        at += 12 + len;
    }
    png_tail(out + at);
    at += 12;
    return at == size ? at : -3;
}

