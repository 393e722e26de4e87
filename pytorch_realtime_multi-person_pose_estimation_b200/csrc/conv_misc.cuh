// CUDA-core kernels around the wgmma conv (see conv_misc.cu).
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include "tc_format.h"

namespace b2p {

struct ConvF32Args {
    const float* in;      // NHWC fp32
    int in_cstride, in_ch_off;
    const float* w;       // OIHW fp32 (the state_dict tensor as is)
    const float* bias;
    float* out;           // NHWC fp32
    int out_cstride, out_ch_off;
    float* out_nchw;      // optional NCHW copy [n][cout][H][W]
    int n_img, H, W, cin, cout, ks, relu;
    const int* ext;       // ragged batch (DESIGN.md §1): padded H, W per image at the network input, or null
    int ext_shift;        // log2 of the network input size over H, W
    const float* slope;   // PReLU slope per output channel (OpenPose_Model): v = v > 0 ? v : slope * v after the bias,
                          // instead of `relu`; null: relu / none
};

// conv1_1 in format fmt.  in: fp32 NCHW [N,3,H,W] (in_is_u8_hwc = 0), or uint8 HWC BGR [N,H,W,3] with the
// normalisation `in_is_u8_hwc` (preprocess_core.h: 1 rtpose, 2 vgg, 3 inception, 4 ssd) fused into the load.
// out_lo: the residual plane (bf16x3).  aux: the format's per-image table (tc_aux): fp8 max |stored bf16| (fp32 bits,
// atomic max), fp16 overflow flags (1 = a value overflowed).  cudaErrorInvalidValue when the format's pointer is null.
// ext: ragged batch, padded H, W per image, or null.
cudaError_t conv_first_launch(const void* in, int in_is_u8_hwc, const float* w_oihw, const float* bias, TcFormat fmt,
                              __nv_bfloat16* out_nhwc, __nv_bfloat16* out_lo, unsigned* aux, int N, int H, int W,
                              const int* ext, cudaStream_t s);
// ext (ragged batch) or null: pixels outside image i's padded extent ext[2 i], ext[2 i + 1] become 0 (zero padding)
cudaError_t u8hwc_to_f32nchw_launch(const unsigned char* in, float* out, int N, int H, int W, int mode, const int* ext,
                                    cudaStream_t s);
cudaError_t conv_f32_launch(const ConvF32Args& a, cudaStream_t s);
cudaError_t maxpool_f32_launch(const float* in, float* out, int N, int H, int W, int C, cudaStream_t s);
cudaError_t nchw_to_nhwc_f32_launch(const float* in, float* out, int N, int C, int H, int W, int out_cstride,
                                    int out_ch_off, cudaStream_t s);

}  // namespace b2p
