// PNG encoding on the device: packed uint8 HWC BGR frames -> PNG files packed back to back, byte for byte what
// cv2.imencode('.png', frame) gives (core in png_enc_core.h).
#pragma once
#include <cuda_runtime.h>

#include "png_enc_core.h"

namespace b2p {

// One encode batch, every table in device memory.  Image i's frame is at frames + ims[i].src, its filtered bytes and
// symbols at ims[i].f0 of filt / sym, its tiles at ims[i].tile0 of the tile arrays, its blocks at ims[i].blk0 of
// blocks, its deflate words at words + wbase[i].  The files are written to out back to back in image order.
struct PngBatch {
    const PngImage* ims;
    int n;
    const unsigned char* frames;
    unsigned char* filt;
    long long *tfirst, *tlast;    // per tile: its first and last run start (none: LLONG_MAX, -1)
    long long *tstart, *tend;     // per tile: the last run start before it, the first after it (or n)
    long long *tcount, *tbase;    // per tile: its symbols, the symbols before it
    unsigned short* sym;
    PngBlock* blocks;
    PngImageOut* outs;            // zeroed before phase 0
    const long long* wbase;       // per image: first word of its deflate bits (set before phase 1)
    unsigned* words;              // zeroed before phase 1
    unsigned char* out;
    long long max_tiles;          // the largest image's tiles, blocks and chunks (size the grids)
    long long max_blocks, max_chunks;
};

// Phase 0: filter, runs, symbols, trees and layout (outs[i].size, .bits); phase 1: pack and write.  The caller sizes
// words and out from outs between the phases and sets max_chunks.
cudaError_t png_encode_launch(const PngBatch& b, int phase, cudaStream_t s);

}  // namespace b2p
