// Host build of the JPEG decoding core (csrc/jpeg_core.h), walking an image the way the kernels of jpeg.cu do: the
// marker walk and segment table of the host runtime, the unstuffing rule, the Huffman kernel's work runs of whole
// segments (jpeg_work) in windows of kWindow chunks with rounds until no boundary state changes and the state carried
// between windows, the segmented block scan, the writing pass, the DC scan, the IDCT per block and the per-pixel
// upsampling, colour conversion and orientation.
// JPEG_CORE overrides the header's path, so that a test can compile a copy with a planted mistake.
#ifndef JPEG_CORE
#define JPEG_CORE "../../pytorch_realtime_multi-person_pose_estimation_b200/csrc/jpeg_core.h"
#endif
#include JPEG_CORE

#include <cstdlib>
#include <vector>

using namespace b2p;

namespace {

constexpr int kWindow = 256;               // jpeg.cu's kThreads
constexpr long long kMaxPixels = 1LL << 28;

bool keep(const unsigned char* raw, long long i, long long beg, long long end) {
    if (raw[i] != 0xFF) return !(i > beg && raw[i - 1] == 0xFF);
    return i + 1 < end && raw[i + 1] == 0x00;
}

}  // namespace

// out: h, w, oriented h, oriented w, supported.  Returns 0, or 1 for a malformed stream; reason: the parse's message.
extern "C" int core_info(const unsigned char* d, long long n, int* out, char* reason, int cap) {
    JpegParsed* P = new JpegParsed;
    const bool ok = jpeg_parse(d, n, kMaxPixels, P);
    out[0] = P->h;
    out[1] = P->w;
    out[2] = P->im.oh;
    out[3] = P->im.ow;
    out[4] = ok && P->supported;
    snprintf(reason, cap, "%s", P->reason);
    delete P;
    return ok ? 0 : 1;
}

// Decodes a stream into out (oriented h x w x 3 BGR, cap bytes).  Returns 0 (status: the kJpeg* bits), 1 malformed,
// 2 unsupported, 3 output too small.
extern "C" int core_decode(const unsigned char* d, long long n, unsigned char* out, long long cap, unsigned* status) {
    JpegParsed* P = new JpegParsed;
    struct Free { JpegParsed* p; ~Free() { delete p; } } f{P};
    if (!jpeg_parse(d, n, kMaxPixels, P)) return 1;
    if (!P->supported) return 2;
    JpegImage& im = P->im;
    if ((long long)im.oh * im.ow * 3 > cap) return 3;
    // unstuffing (jpeg_unstuff_kernel's rule over the whole scan)
    std::vector<unsigned char> data;
    data.reserve(P->scan_end - P->scan_beg);
    for (long long i = P->scan_beg; i < P->scan_end; ++i)
        if (keep(d, i, P->scan_beg, P->scan_end)) data.push_back(d[i]);
    data.push_back(0);
    std::vector<JpegSeg> segs;
    jpeg_segments(*P, 0, 0, 0, &segs);
    long long blocks = 0;
    for (int c = 0; c < im.ncomp; ++c) {
        im.comp[c].coef = blocks;
        blocks += (long long)im.comp[c].bw * im.comp[c].bh;
    }
    std::vector<short> coef(blocks * 64, 0);
    unsigned st = P->status;
    // Huffman (jpeg_huff_kernel): the same work runs of whole segments, each walked in windows of kWindow chunks that
    // may start inside a segment; thread t of a window holds chunk w0 + t
    long long chunks = 0;
    for (const JpegSeg& sg : segs) {
        const long long bits = (sg.end - sg.beg) * 8;
        chunks += bits > 0 ? (bits + kJpegChunkBits - 1) / kJpegChunkBits : 1;
    }
    std::vector<int> chunk_seg;
    std::vector<long long> work;
    jpeg_work(segs, chunks, &chunk_seg, &work);
    for (size_t w = 0; w + 1 < work.size(); ++w) {
        JpegState carry{0, 0, 0};
        long long carry_g = 0;
        for (long long w0 = work[w]; w0 < work[w + 1]; w0 += kWindow) {
            const int T = (int)(work[w + 1] - w0 < kWindow ? work[w + 1] - w0 : kWindow);
            std::vector<JpegState> entry(T), used(T, JpegState{-1, 0, 0}), exits(T);
            std::vector<long long> cb(T), ce(T), nblk(T, 0);
            std::vector<char> head(T), last(T);
            for (int t = 0; t < T; ++t) {
                const JpegSeg& sg = segs[chunk_seg[w0 + t]];
                const long long bits = (sg.end - sg.beg) * 8, q = w0 + t - sg.chunk0;
                const long long n = bits > 0 ? (bits + kJpegChunkBits - 1) / kJpegChunkBits : 1;
                cb[t] = q * kJpegChunkBits;
                ce[t] = cb[t] + kJpegChunkBits < bits ? cb[t] + kJpegChunkBits : bits;
                head[t] = q == 0;
                last[t] = q == n - 1;
                entry[t] = head[t] ? JpegState{0, 0, 0} : (t == 0 ? carry : JpegState{cb[t], 0, 0});
            }
            for (;;) {
                for (int t = 0; t < T; ++t)
                    if (!jp_same(entry[t], used[t])) {
                        const JpegSeg& sg = segs[chunk_seg[w0 + t]];
                        JpegState s = entry[t];
                        nblk[t] = jp_sync_chunk(im, s, data.data() + sg.beg, sg.end - sg.beg, ce[t]);
                        exits[t] = s;
                        used[t] = entry[t];
                    }
                bool changed = false;
                for (int t = T - 1; t > 0; --t)
                    if (!head[t] && !jp_same(entry[t], exits[t - 1])) {
                        entry[t] = exits[t - 1];
                        changed = true;
                    }
                if (!changed) break;
            }
            long long run = 0;
            for (int t = 0; t < T; ++t) {
                const JpegSeg& sg = segs[chunk_seg[w0 + t]];
                if (head[t]) run = 0;
                else if (t == 0) run = carry_g;
                const long long g = run - (entry[t].k > 0 ? 1 : 0);
                st |= jp_write_chunk(im, sg, entry[t], g, ce[t], last[t], data.data() + sg.beg, coef.data());
                run += nblk[t];
            }
            carry = exits[T - 1];
            carry_g = run;
        }
    }
    // DC: prefix sums per component in decode order, restarting at each restart interval (jpeg_dc_kernel)
    for (int c = 0; c < im.ncomp; ++c) {
        const long long total = (long long)im.comp[c].bw * im.comp[c].bh;
        unsigned acc = 0;
        for (long long i = 0; i < total; ++i) {
            bool head;
            short* b = jp_dc_block(im, coef.data(), c, i, &head);
            acc = (head ? 0u : acc) + (unsigned)(int)b[0];
            b[0] = (short)(int)acc;
        }
    }
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

#ifdef JPEG_HOST_MAIN
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
