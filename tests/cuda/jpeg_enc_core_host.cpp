// Host build of the JPEG encoding core (csrc/jpeg_enc_core.h), split the way the kernels of jpeg_enc.cu run it: per
// block the quantised coefficients and their AC code length, per image an exclusive scan of the block lengths with
// the DC codes added, per block the packing of its codes into 32-bit words (first and last word ORed, the words
// between stored), and per image the padding and stuffing of the bytes with the header in front and EOI behind.
// JPEG_ENC_CORE overrides the header's path, so that a test can compile a copy with a planted mistake.
#ifndef JPEG_ENC_CORE
#define JPEG_ENC_CORE "../../pytorch_realtime_multi-person_pose_estimation_b200/csrc/jpeg_enc_core.h"
#endif
#include JPEG_ENC_CORE

#include <vector>

using namespace b2p;

// jcdctmgr.c's divisor of table value q as the core computes it: out = {reciprocal, correction, shift (r - 16)}.
extern "C" void core_reciprocal(int q, unsigned* out) {
    unsigned short recip, corr;
    unsigned char shift;
    jenc_reciprocal(q, &recip, &corr, &shift);
    out[0] = recip;
    out[1] = corr;
    out[2] = shift;
}

// The stream bound of an h x w frame at this sampling (jenc_stream_bound), or -1 for an unknown sampling.
extern "C" long long core_encode_bound(int h, int w, int sampling) {
    if (!jenc_sampling_ok(sampling) || h < 1 || w < 1) return -1;
    JencImage* im = new JencImage;
    jenc_image(h, w, 95, sampling, im);
    const long long b = jenc_stream_bound(*im);
    delete im;
    return b;
}

// Encodes the h x w BGR frame into out (cap bytes).  Returns the stream's size, or -1 for bad arguments, -2 when cap
// is below the bound.
extern "C" long long core_encode(const unsigned char* frame, int h, int w, int quality, int sampling, unsigned char* out,
                                 long long cap) {
    if (!frame || h < 1 || w < 1 || h > 65535 || w > 65535 || quality < 1 || quality > 100 || !jenc_sampling_ok(sampling))
        return -1;
    std::vector<JencImage> imv(1);
    JencImage& im = imv[0];
    jenc_image(h, w, quality, sampling, &im);
    if (cap < jenc_stream_bound(im)) return -2;
    JencHuff huff[4];
    for (int t = 0; t < 4; ++t) jenc_huff_table(t, &huff[t]);
    const long long nb = im.blocks;
    // coefficients and AC lengths (jpeg_enc_dct_kernel)
    std::vector<short> coef(nb * 64);
    std::vector<int> acbits(nb);
    for (long long g = 0; g < nb; ++g) {
        jenc_block_coefs(im, frame, g, coef.data() + g * 64);
        const int t = im.comp[im.mcu_comp[g % im.bpm]].t;
        acbits[g] = jenc_codes(coef.data() + g * 64, false, 0, huff[2 * t], huff[2 * t + 1], JencNoPut{});
    }
    // DC lengths and the exclusive scan (jpeg_enc_scan_kernel)
    std::vector<long long> off(nb);
    long long bits = 0;
    for (long long g = 0; g < nb; ++g) {
        const long long p = jenc_pred_block(im, g);
        const int t = im.comp[im.mcu_comp[g % im.bpm]].t;
        const int dc = jenc_codes(coef.data() + g * 64, true, p < 0 ? 0 : coef[p * 64], huff[2 * t], huff[2 * t + 1],
                                  JencNoPut{});
        off[g] = bits;
        bits += acbits[g] + dc;
    }
    std::vector<unsigned> words((size_t)jenc_words(bits), 0u);
    // packing (jpeg_enc_pack_kernel)
    unsigned* wd = words.data();
    auto store = [wd](long long i, unsigned v) { wd[i] = v; };
    auto shared = [wd](long long i, unsigned v) { wd[i] |= v; };
    for (long long g = 0; g < nb; ++g) {
        const long long p = jenc_pred_block(im, g);
        const int t = im.comp[im.mcu_comp[g % im.bpm]].t;
        JencBitWriter<decltype(store), decltype(shared)> wr(off[g], store, shared);
        const short* zz = coef.data() + g * 64;
        jenc_codes(zz, true, p < 0 ? 0 : coef[p * 64], huff[2 * t], huff[2 * t + 1], [&wr](unsigned b, int l) { wr(b, l); });
        jenc_codes(zz, false, 0, huff[2 * t], huff[2 * t + 1], [&wr](unsigned b, int l) { wr(b, l); });
        wr.finish();
    }
    // stuffing (jpeg_enc_count_kernel, jpeg_enc_write_kernel)
    const long long nbytes = jenc_data_bytes(bits);
    long long at = 0;
    memcpy(out, im.hdr, im.hdr_len);
    at += im.hdr_len;
    for (long long k = 0; k < nbytes; ++k) {
        at += jenc_put_stuffed(out + at, jenc_byte(wd, bits, k));
    }
    out[at++] = 0xFF;
    out[at++] = 0xD9;
    return at;
}
