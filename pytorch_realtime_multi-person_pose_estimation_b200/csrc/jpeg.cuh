// JPEG decoding on the device: baseline / extended sequential and, opt-in, progressive Huffman streams -> oriented
// uint8 HWC BGR frames packed back to back, what cv2.imdecode(buf, cv2.IMREAD_COLOR) gives (core in jpeg_core.h).
#pragma once
#include <cuda_runtime.h>

#include "jpeg_core.h"

namespace b2p {

constexpr int kJpegLaunches = 5;     // unstuff, Huffman, DC, IDCT, colour
// with progressive images: unstuff, [Huffman, DC when the call has baseline images], progressive, IDCT, colour
constexpr int kJpegProgLaunches = 6, kJpegProgOnlyLaunches = 4;

// The scan bytes [raw_beg, raw_end) of one image in the staging buffer; its unstuffed data starts at `out`.
struct JpegUnstuffJob {
    long long raw_beg, raw_end, out;
};

// One decode batch, every table in device memory.  work[w] .. work[w + 1]: the chunks (whole segments) CTA w of the
// Huffman kernel decodes; chunk_seg[c]: the segment of chunk c.  coef must be zeroed (blocks x 64 int16).
// Progressive images (nprog > 0) are JpegImage entries like the others; their scans are unstuffed by jobs of their own
// (njobs: one per baseline image plus one per progressive scan), and segs / chunk_seg / work cover the baseline images
// only (nwork 0: none).
struct JpegBatch {
    const JpegImage* ims;
    int n;
    const JpegUnstuffJob* jobs;
    const unsigned char* raw;
    unsigned char* data;
    const JpegSeg* segs;
    const int* chunk_seg;
    const long long* work;
    int nwork;
    short* coef;
    unsigned char* planes;
    unsigned char* out;
    unsigned* status;            // per image, ORed with kJpeg* bits
    long long max_blocks;        // the largest component's blocks (sizes the IDCT grid)
    long long max_px;            // the largest oriented frame's pixels
    int njobs;
    const JpegProgImage* prog;   // nprog progressive images, their scans and the scans' segments
    int nprog;
    const JpegScan* scans;
    const JpegSeg* pseg;
};

// The launches jpeg_decode_launch makes for b: kJpegLaunches without progressive images.
int jpeg_decode_launches(const JpegBatch& b);
cudaError_t jpeg_decode_launch(const JpegBatch& b, cudaStream_t s);

}  // namespace b2p
