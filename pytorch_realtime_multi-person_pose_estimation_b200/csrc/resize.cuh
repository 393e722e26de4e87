// crop_with_factor on the device (SURVEY.md 8(f) rank 1):  /root/reference/lib/network/im_transform.py:113-134
// uint8 HWC BGR frames of one source size -> bilinear resize (OpenCV INTER_LINEAR arithmetic, resize_core.h) so that
// the short side is dest_size -> zero padding bottom/right to a multiple of `factor`.
#pragma once
#include <cuda_runtime.h>

#include "resize_core.h"

namespace b2p {

// in [n, src_h, src_w, 3] -> out [n, g.pad_h, g.pad_w, 3], both on the device
cudaError_t crop_with_factor_launch(const unsigned char* in, unsigned char* out, int n, int src_h, int src_w,
                                    const CropGeom& g, cudaStream_t s);

// Bicubic resize of `planes` float32 planes [src_h, src_w] -> [dst_h, dst_w] (resize_core.h: rs_cubic_at), fused with
// the running sum of the multi-scale average: dst = first ? r : dst + r, then dst /= divide_by when divide_by > 0.
cudaError_t resize_cubic_accum_launch(const float* src, float* dst, long planes, int src_h, int src_w, int dst_h,
                                      int dst_w, int first, float divide_by, cudaStream_t s);

// Ragged batch of n frames: src [n, channels, src_hc, src_wc] -> dst [n, channels, dst_hc, dst_wc] (canvas pitches);
// frames[i] (device) gives frame i's extent at both resolutions.  Inside frame i's destination extent the running sum as
// above, every other element of the destination canvas is written +0.
cudaError_t resize_cubic_accum_ragged_launch(const float* src, float* dst, const RaggedResize* frames, int n, int channels,
                                             int src_hc, int src_wc, int dst_hc, int dst_wc, int first, float divide_by,
                                             cudaStream_t s);

// One frame of a ragged batch (DESIGN.md §1): uint8 HWC source at byte offset `off`, and its crop_with_factor geometry
// (g.pad_h == 0: the source is an already cropped network input, copied unchanged).
struct RaggedFrame {
    long long off;
    int src_h, src_w;
    CropGeom g;
};

// frames [n] (device) -> out [n, Hc, Wc, 3]: frame i cropped (or copied) into the top-left corner of slot i, zeros elsewhere
cudaError_t ragged_frames_launch(const unsigned char* in, const RaggedFrame* frames, int n, unsigned char* out, int Hc,
                                 int Wc, cudaStream_t s);

}  // namespace b2p
