// crop_with_factor on the device (SURVEY.md 8(f) rank 1):  /root/reference/lib/network/im_transform.py:113-134
// uint8 HWC BGR frames, each of its own source size -> bilinear resize (OpenCV INTER_LINEAR arithmetic, resize_core.h)
// so that the short side is dest_size -> zero padding bottom/right to a multiple of `factor`.  A batch of frames of one
// size is a frame table whose entries all have that size.
#pragma once
#include <cuda_runtime.h>

#include "resize_core.h"

namespace b2p {

// One frame of a batch (DESIGN.md §1): uint8 HWC source at byte offset `off`, and its crop_with_factor geometry
// (g.pad_h == 0: the source is an already cropped network input, copied unchanged).
struct RaggedFrame {
    long long off;
    int src_h, src_w;
    CropGeom g;
};

// frames [n] (device) -> out [n, Hc, Wc, 3]: frame i cropped (or copied) into the top-left corner of slot i, zeros elsewhere
cudaError_t crop_frames_launch(const unsigned char* in, const RaggedFrame* frames, int n, unsigned char* out, int Hc,
                               int Wc, cudaStream_t s);

// Bicubic resize (resize_core.h: rs_cubic_ragged_at) of n frames, fused with the running sum of the multi-scale
// average: src [n, channels, src_hc, src_wc] -> dst [n, channels, dst_hc, dst_wc] (canvas pitches); frames[i] (device)
// gives frame i's extent at both resolutions.  Inside frame i's destination extent dst = first ? r : dst + r, then
// dst /= divide_by when divide_by > 0; every other element of the destination canvas is written +0.
cudaError_t resize_cubic_accum_launch(const float* src, float* dst, const RaggedResize* frames, int n, int channels,
                                      int src_hc, int src_wc, int dst_hc, int dst_wc, int first, float divide_by,
                                      cudaStream_t s);

}  // namespace b2p
