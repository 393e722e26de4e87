// Training-time augmentation of a ragged batch of uint8 BGR frames on the device: the reference loader's HFlip,
// RescaleRelative (Pillow BICUBIC), Crop, CenterPad, ColorJitter, RandomGrayscale, ToTensor + Normalize and
// mask_valid_area (core in aug_core.h, DESIGN.md 2.20).  The JPEG quality-50 round trip between the colour jitter and
// the grayscale runs on the existing encoder and decoder (api.cu).
#pragma once
#include <cuda_runtime.h>

#include "aug_core.h"

namespace b2p {

// One sample: its source, the draws of augment_params and the geometry derived from them.
struct AugImage {
    long long src;          // byte offset of the source frame (h x w x 3, BGR) in the packed sources
    long long tmp;          // byte offset of its horizontal pass (rows x cw x 3, RGB) in the intermediate
    int h, w, flip;
    int rw, rh;             // the resized size int(w f), int(h f)
    int x0, y0, cw, ch;     // Crop's offset in the resized image and the cropped size
    int left, top;          // CenterPad's offsets
    int r0, rows;           // first source row the vertical pass reads, and how many
    int order[4];           // ColorJitter's fn_idx
    double f[4];            // its brightness, contrast, saturation factors by fn id (f[3] unused)
    int dh;                 // the hue byte shift np.int32(hue * 255).astype(uint8)
    int gray;               // RandomGrayscale drew this sample
    int mx0, my0, mx1, my1; // mask_valid_area: columns < mx0 or >= mx1 and rows < my0 or >= my1 become 0
};

struct AugBatch {
    const AugImage* images;      // device
    const unsigned char* src;    // packed sources
    unsigned char* tmp;          // horizontal passes
    unsigned char* px;           // [n][E][E][3]: RGB after the operations before contrast, then BGR after the jitter
    unsigned long long* lsum;    // [n]: sum of L over the image before contrast (zeroed by the caller)
    float* out;                  // [n][3][E][E] normalised, RGB
    unsigned char* out_u8;       // [n][E][E][3] BGR before normalisation, or null
    int n, edge, max_tmp_px;     // images, edge, largest rows * cw
};

// Three launches before the JPEG round trip (horizontal pass; vertical pass, pad and the operations before contrast;
// contrast and the operations after it), one after it (grayscale, normalisation, mask).
constexpr int kAugLaunchesJitter = 3;
constexpr int kAugLaunchesFinish = 1;
cudaError_t aug_jitter_launch(const AugBatch& b, cudaStream_t s);
cudaError_t aug_finish_launch(const AugBatch& b, cudaStream_t s);

}  // namespace b2p
