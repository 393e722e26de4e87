// Flip test-time averaging on the device (SURVEY.md 8(a) row F1, 8(f) rank 2):
//   tta_mirror_*      : W-mirrored copies of a batch of frames (the second half of a 2n batch)
//   tta_flip_merge    : handle_paf_and_heat      /root/reference/evaluate/coco_eval.py:197-242
#pragma once
#include <cuda_runtime.h>

#include "resize.cuh"

namespace b2p {

// out[i, y, x, :] = in[i, y, W-1-x, :]   uint8 HWC frames (3 channels)
cudaError_t tta_mirror_u8hwc(const unsigned char* in, unsigned char* out, int n, int H, int W, cudaStream_t s);
// ragged batch: frame i (frames[i].src_h x frames[i].src_w, HWC at byte offset frames[i].off) mirrored from in + off into
// out + off; max_frame_bytes = the largest frame's size
cudaError_t tta_mirror_u8hwc_ragged(const unsigned char* in, unsigned char* out, const RaggedFrame* frames, int n,
                                    long max_frame_bytes, cudaStream_t s);
// out[i, c, y, x] = in[i, c, y, W-1-x]   fp32 planes; `planes` = n * channels
cudaError_t tta_mirror_f32(const float* in, float* out, long planes, int H, int W, cudaStream_t s);
// out(img, c, y, x) = (normal(img, c, y, x) +/- flipped(img, swap[c], y, w-1-x)) / 2 for `channels` = 19 (heat) or 38
// (PAF).  All three tensors share the layout: value = p[img*channels*h*w + c*sc + y*sy + x*sx].
// ext (ragged batch) or null: image i mirrors within its own width ext[2 i + 1] / 8 and is +0 outside its extent.
cudaError_t tta_flip_merge(const float* normal, const float* flipped, float* out, int n, int channels, int h, int w,
                           long sc, long sy, long sx, const int* ext, cudaStream_t s);

}  // namespace b2p
