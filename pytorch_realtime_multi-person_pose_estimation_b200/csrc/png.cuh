// PNG decoding on the device: PNG streams -> oriented uint8 HWC BGR frames packed back to back, what
// cv2.imdecode(buf, cv2.IMREAD_COLOR) gives (core in png_core.h).
#pragma once
#include <cuda_runtime.h>

#include "png_core.h"

namespace b2p {

constexpr int kPngLaunches = 4;     // gather, inflate, unfilter, colour

// One decode batch, every table in device memory.  raw: the uploaded IDAT chunks (type and data, PngIdat::src);
// zlib: their data gathered per image (PngDecImage::z0); rows: the inflated, then reconstructed, rows (::f0).
struct PngDecBatch {
    const PngDecImage* ims;
    int n;
    const PngIdat* idat;
    int nidat;
    const unsigned char* raw;
    unsigned char* zlib;
    unsigned char* rows;
    unsigned char* out;
    unsigned* status;            // per image, ORed with kPng* bits
    long long max_px;            // the largest oriented frame's pixels
};

cudaError_t png_decode_launch(const PngDecBatch& b, cudaStream_t s);

}  // namespace b2p
