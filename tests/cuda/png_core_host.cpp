// Host build of the PNG decoding core (csrc/png_core.h), walking an image the way the kernels of png.cu do: the chunk
// walk of the host runtime, the gather of the IDAT data with each chunk's CRC, the decoding lane's rounds of tokens
// written as the warp writes them (literals and stored runs, then the matches in order), the Adler-32 of the output,
// the rows of every pass reconstructed lane by lane, and the per-pixel colour rules and orientation.
// PNG_CORE overrides the header's path, so that a test can compile a copy with a planted mistake.
#ifndef PNG_CORE
#define PNG_CORE "../../pytorch_realtime_multi-person_pose_estimation_b200/csrc/png_core.h"
#endif
#include PNG_CORE

#include <cstdlib>
#include <memory>
#include <vector>

using namespace b2p;

namespace {
constexpr long long kMaxPixels = 1LL << 28;
}

// out: h, w, oriented h, oriented w, supported.  Returns 0, or 1 for a malformed stream; reason: the parse's message.
extern "C" int core_info(const unsigned char* d, long long n, int* out, char* reason, int cap) {
    std::unique_ptr<PngParsed> P(new PngParsed);
    const bool ok = png_parse(d, n, kMaxPixels, P.get());
    out[0] = P->h;
    out[1] = P->w;
    out[2] = P->im.oh;
    out[3] = P->im.ow;
    out[4] = ok && P->supported;
    snprintf(reason, cap, "%s", P->reason);
    return ok ? 0 : 1;
}

// Decodes a stream into out (oriented h x w x 3 BGR, cap bytes).  Returns 0 (status: the kPng* bits), 1 malformed,
// 2 unsupported, 3 output too small.
extern "C" int core_decode(const unsigned char* d, long long n, unsigned char* out, long long cap, unsigned* status) {
    std::unique_ptr<PngParsed> P(new PngParsed);
    if (!png_parse(d, n, kMaxPixels, P.get())) return 1;
    if (!P->supported) return 2;
    const PngDecImage& im = P->im;
    if ((long long)im.oh * im.ow * 3 > cap) return 3;
    unsigned st = 0;
    // gather (png_gather_kernel)
    std::vector<unsigned char> z((size_t)P->zlen + 1);
    for (const PngIdat& c : P->idat) {
        memcpy(z.data() + c.dst, d + c.src + 4, (size_t)c.len);
        if (pn_crc(d + c.src, c.len + 4) != c.crc) st |= kPngBadCrc;
    }
    // inflate (png_inflate_kernel)
    std::vector<unsigned char> rows((size_t)im.flen + 1, 0);
    std::unique_ptr<PngInflate> s(new PngInflate);
    std::vector<PngToken> tok(kPngTokens);
    if (pn_zlib_header(*s, z.data(), P->zlen))
        while (s->state != kPnDone) {
            const int m = pn_inflate_round(*s, z.data(), P->zlen, im.flen, P->idat.data(), (int)P->idat.size(), tok.data());
            for (int t = 0; t < m; ++t)
                if (tok[t].kind != 1)
                    for (int j = 0; j < tok[t].len; ++j) pn_token_byte(tok[t], j, z.data(), rows.data());
            for (int t = 0; t < m; ++t)
                if (tok[t].kind == 1)
                    for (int j = 0; j < tok[t].len; ++j) pn_token_byte(tok[t], j, z.data(), rows.data());
        }
    st |= s->status;
    if (s->ended && s->status == 0) {
        unsigned long long a = 0, b = 0;
        for (long long p = 0; p < im.flen; ++p) {
            a = (a + rows[p]) % kPngAdlerMod;
            b = (b + (unsigned long long)((im.flen - p) % kPngAdlerMod) * rows[p]) % kPngAdlerMod;
        }
        if (png_adler(im.flen, a, b) != s->adler) st |= kPngBadAdler;
    }
    // unfilter (png_unfilter_kernel): rows in order, the 32 lanes of a row one after another
    unsigned char* at = rows.data();
    for (int p = 0; p < (im.interlace ? 7 : 1); ++p) {
        int ph, pw;
        pn_pass(im.interlace, p, im.h, im.w, &ph, &pw);
        const long long rb = pn_rowbytes(im, pw);
        for (int r = 0; r < ph; ++r, at += rb + 1) {
            if (at[0] > 4) {
                st |= kPngBadFilter;
                continue;
            }
            if (at[0])
                for (int lane = 0; lane < 32; ++lane) pn_unfilter_lane(at + 1, r ? at - rb : nullptr, rb, im.bpp, at[0], lane, 32);
        }
    }
    // colour and orientation (png_color_kernel)
    for (int y = 0; y < im.oh; ++y)
        for (int x = 0; x < im.ow; ++x) png_px(im, rows.data(), y, x, out + 3 * ((long long)y * im.ow + x));
    *status = st;
    return 0;
}

#ifdef PNG_HOST_MAIN
// Standalone driver (built with -fsanitize=address by the tests): decodes each file named on the command line into an
// output buffer of exactly the oriented frame's size and prints "rc status" per file.
#include <cstdio>
int main(int argc, char** argv) {
    for (int a = 1; a < argc; ++a) {
        FILE* f = fopen(argv[a], "rb");
        if (!f) return 2;
        std::vector<unsigned char> buf;
        int ch;
        while ((ch = fgetc(f)) != EOF) buf.push_back((unsigned char)ch);
        fclose(f);
        // an exact-size copy, so that a read past the stream is a heap overflow
        unsigned char* d = (unsigned char*)malloc(buf.size() ? buf.size() : 1);
        if (!buf.empty()) memcpy(d, buf.data(), buf.size());
        int info[5];
        char reason[256];
        core_info(d, (long long)buf.size(), info, reason, sizeof(reason));
        const long long cap = 3LL * info[2] * info[3];
        unsigned char* out = (unsigned char*)malloc(cap > 0 ? cap : 1);
        unsigned st = 0;
        const int rc = core_decode(d, (long long)buf.size(), out, cap, &st);
        printf("%d %u\n", rc, st);
        free(out);
        free(d);
    }
    return 0;
}
#endif
