// Host build of the progressive JPEG path of csrc/jpeg_core.h, walking an image the way the kernels of jpeg.cu do:
// the parse with progressive streams on, per scan the unstuffing rule, every segment of a scan decoded by
// jp_prog_segment (scans in stream order), then the IDCT per block and the per-pixel upsampling, colour conversion and
// orientation.  Streams the parse finds to be baseline take jpeg_core_host.cpp's path (core_decode).
// JPEG_CORE overrides the header's path, so that a test can compile a copy with a planted mistake.
#include "jpeg_core_host.cpp"

// out: h, w, oriented h, oriented w, supported, progressive.  Returns 0, or 1 for a malformed stream; reason: the
// parse's message.
extern "C" int prog_info(const unsigned char* d, long long n, int progressive, int* out, char* reason, int cap) {
    JpegParsed* P = new JpegParsed;
    const bool ok = jpeg_parse(d, n, kMaxPixels, P, progressive != 0);
    out[0] = P->h;
    out[1] = P->w;
    out[2] = P->im.oh;
    out[3] = P->im.ow;
    out[4] = ok && P->supported;
    out[5] = P->progressive;
    snprintf(reason, cap, "%s", P->reason);
    delete P;
    return ok ? 0 : 1;
}

// Decodes a stream with progressive streams on into out (oriented h x w x 3 BGR, cap bytes).  Returns 0 (status: the
// kJpeg* bits), 1 malformed, 2 unsupported, 3 output too small.
extern "C" int prog_decode(const unsigned char* d, long long n, unsigned char* out, long long cap, unsigned* status) {
    JpegParsed* P = new JpegParsed;
    struct Free { JpegParsed* p; ~Free() { delete p; } } f{P};
    if (!jpeg_parse(d, n, kMaxPixels, P, true)) return 1;
    if (!P->supported) return 2;
    if (!P->progressive) return core_decode(d, n, out, cap, status);
    JpegImage& im = P->im;
    if ((long long)im.oh * im.ow * 3 > cap) return 3;
    // unstuffing per scan (jpeg_unstuff_kernel's rule over each scan's bytes)
    std::vector<unsigned char> data;
    std::vector<long long> base;
    for (size_t s = 0; s < P->scans.size(); ++s) {
        base.push_back((long long)data.size());
        const long long b = P->scan_raw[2 * s], e = P->scan_raw[2 * s + 1];
        for (long long i = b; i < e; ++i)
            if (keep(d, i, b, e)) data.push_back(d[i]);
    }
    data.push_back(0);
    std::vector<JpegScan> scans;
    std::vector<JpegSeg> segs;
    jpeg_prog_segments(*P, 0, base.data(), &scans, &segs);
    long long blocks = 0;
    for (int c = 0; c < im.ncomp; ++c) {
        im.comp[c].coef = blocks;
        blocks += (long long)im.comp[c].bw * im.comp[c].bh;
    }
    std::vector<short> coef(blocks * 64, 0);
    unsigned st = P->status;
    // jpeg_prog_kernel: the scans in stream order, each scan's segments independent of each other
    for (const JpegScan& sc : scans)
        for (int k = 0; k < sc.nseg; ++k) st |= jp_prog_segment(im, sc, segs[sc.seg0 + k], data.data(), coef.data());
    // IDCT (jpeg_idct_kernel)
    long long pbytes = 0;
    for (int c = 0; c < im.ncomp; ++c) {
        im.comp[c].plane = pbytes;
        pbytes += (long long)im.comp[c].bw * im.comp[c].bh * 64;
    }
    std::vector<unsigned char> planes(pbytes);
    for (int c = 0; c < im.ncomp; ++c) {
        const JpegComp& cp = im.comp[c];
        const long long pitch = (long long)cp.bw * 8;
        for (long long b = 0; b < (long long)cp.bw * cp.bh; ++b) {
            const long long by = b / cp.bw, bx = b % cp.bw;
            jp_idct_block(coef.data() + (cp.coef + b) * 64, im.qt[c], planes.data() + cp.plane + by * 8 * pitch + bx * 8, pitch);
        }
    }
    // upsampling, colour and orientation (jpeg_color_kernel)
    for (int y = 0; y < im.oh; ++y)
        for (int x = 0; x < im.ow; ++x) jpeg_px(im, planes.data(), y, x, out + 3 * ((long long)y * im.ow + x));
    *status = st;
    return 0;
}

#ifdef JPEG_PROG_HOST_MAIN
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
        memcpy(d, buf.data(), buf.size());
        int info[6];
        char reason[256];
        prog_info(d, (long long)buf.size(), 1, info, reason, sizeof(reason));
        const long long cap = 3LL * info[2] * info[3];
        unsigned char* out = (unsigned char*)malloc(cap > 0 ? cap : 1);
        unsigned st = 0;
        const int rc = prog_decode(d, (long long)buf.size(), out, cap, &st);
        printf("%d %u\n", rc, st);
        free(out);
        free(d);
    }
    return 0;
}
#endif
