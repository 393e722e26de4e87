// JPEG encoding on the device: packed uint8 HWC BGR frames -> baseline JPEG streams packed back to back, byte for byte
// what cv2.imencode('.jpg', frame, [quality, sampling]) gives (core in jpeg_enc_core.h).
#pragma once
#include <cuda_runtime.h>

#include "jpeg_enc_core.h"

namespace b2p {

// One encode batch, every table in device memory.  Image i's frame is at frames + ims[i].src, its blocks at
// ims[i].blk0 .. + blocks of coef / acbits / off, its bit buffer at words + wbase[i].  The streams are written to
// out back to back in image order; sizes[i] receives stream i's length.
struct JencBatch {
    const JencImage* ims;
    int n;
    const JencHuff* huff;        // DC luma, AC luma, DC chroma, AC chroma
    const unsigned char* frames;
    short* coef;                 // 64 per block, zig-zag order
    int* acbits;                 // per block
    long long* off;              // per block: first bit in its image's buffer
    const long long* wbase;      // per image: first word of its bit buffer (set before phase 1)
    unsigned* words;             // zeroed before phase 1
    long long* bits;             // per image: entropy-coded bits
    long long* sizes;            // per image: stream bytes
    unsigned char* out;
    long long max_blocks;        // the largest image's blocks (sizes the per-block grids)
};

// Phase 0: coefficients and scan (bits); phase 1: pack and count (sizes); phase 2: write.  The caller sizes words from
// bits between phases 0 and 1, and out from sizes between phases 1 and 2.
cudaError_t jpeg_encode_launch(const JencBatch& b, int phase, cudaStream_t s);

}  // namespace b2p
