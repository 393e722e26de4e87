// Video-frame ingestion, host/device shared core: NV12 / I420 / pitched BGR frames -> uint8 HWC BGR, rotated.
//   cv2.rotate(cv2.cvtColor(frame, COLOR_YUV2BGR_NV12 / COLOR_YUV2BGR_I420), code)   (OpenCV 4.13)
// OpenCV's 8-bit YUV 4:2:0 -> BGR conversion is BT.601 "video range" in 20-bit fixed point, restated here:
//   y = max(0, Y - 16) * CY + 2^19;  u = U - 128;  v = V - 128
//   B = sat((y + CUB u) >> 20),  G = sat((y + CVG v + CUG u) >> 20),  R = sat((y + CVR v) >> 20)
// with the chroma of pixel (r, c) taken from sample (r / 2, c / 2), no interpolation.  This equals cv2.cvtColor on all
// 2^24 (Y, U, V) triples for both layouts (tests/test_frames_host.py).  Every intermediate fits in int32.
// Rotation is in degrees clockwise: 90 = cv2.ROTATE_90_CLOCKWISE, 180 = cv2.ROTATE_180, 270 =
// cv2.ROTATE_90_COUNTERCLOCKWISE.  The same functions run in convert_frames_kernel (frames.cu) and in the host build of
// the tests, so the index logic is checked against cv2 on a machine without a GPU.
#pragma once

#if defined(__CUDACC__)
#define B2P_FR_HD __host__ __device__ __forceinline__
#else
#define B2P_FR_HD inline
#endif

namespace b2p {

// values of B200POSE_FRAME_* (include/b200pose.h)
constexpr int kFrameBGR = 0, kFrameNV12 = 1, kFrameI420 = 2;

// One source frame: planes (BGR: [0] HWC; NV12: Y, interleaved UV of h/2 rows; I420: Y, U, V with U and V h/2 x w/2),
// each with its own pitch in bytes; the stored size h x w; the byte offset of its rotated BGR output.
struct FrameSrc {
    const unsigned char* plane[3];
    int pitch[3];
    int h, w;
    long long off;
};

constexpr int kYuvShift = 20;
constexpr int kCY = 1220542, kCUB = 2116026, kCUG = -409993, kCVG = -852492, kCVR = 1673527;

B2P_FR_HD unsigned char fr_sat(int v) { return (unsigned char)(v < 0 ? 0 : (v > 255 ? 255 : v)); }

B2P_FR_HD void fr_yuv_to_bgr(int Y, int U, int V, unsigned char* bgr) {
    const int y = (Y > 16 ? Y - 16 : 0) * kCY + (1 << (kYuvShift - 1));
    const int u = U - 128, v = V - 128;
    bgr[0] = fr_sat((y + kCUB * u) >> kYuvShift);
    bgr[1] = fr_sat((y + kCVG * v + kCUG * u) >> kYuvShift);
    bgr[2] = fr_sat((y + kCVR * v) >> kYuvShift);
}

// Size of a stored h x w frame after rotating it by `rot` degrees clockwise.
B2P_FR_HD void fr_rotated_size(int h, int w, int rot, int* oh, int* ow) {
    const bool swap = rot == 90 || rot == 270;
    *oh = swap ? w : h;
    *ow = swap ? h : w;
}

// Stored pixel (sy, sx) that output pixel (y, x) of the rotated frame shows.
B2P_FR_HD void fr_source_pixel(int h, int w, int rot, int y, int x, int* sy, int* sx) {
    switch (rot) {
        case 90: *sy = h - 1 - x; *sx = y; break;
        case 180: *sy = h - 1 - y; *sx = w - 1 - x; break;
        case 270: *sy = x; *sx = w - 1 - y; break;
        default: *sy = y; *sx = x; break;
    }
}

// The BGR bytes of stored pixel (sy, sx).
B2P_FR_HD void fr_fetch(const FrameSrc& f, int fmt, int sy, int sx, unsigned char* bgr) {
    if (fmt == kFrameBGR) {
        const unsigned char* p = f.plane[0] + (long)sy * f.pitch[0] + 3L * sx;
        bgr[0] = p[0];
        bgr[1] = p[1];
        bgr[2] = p[2];
        return;
    }
    const int Y = f.plane[0][(long)sy * f.pitch[0] + sx];
    const int cy = sy >> 1, cx = sx >> 1;
    int U, V;
    if (fmt == kFrameNV12) {
        const unsigned char* uv = f.plane[1] + (long)cy * f.pitch[1] + 2L * cx;
        U = uv[0];
        V = uv[1];
    } else {
        U = f.plane[1][(long)cy * f.pitch[1] + cx];
        V = f.plane[2][(long)cy * f.pitch[2] + cx];
    }
    fr_yuv_to_bgr(Y, U, V, bgr);
}

// Output pixel (y, x) of frame f rotated by `rot`.
B2P_FR_HD void frame_px(const FrameSrc& f, int fmt, int rot, int y, int x, unsigned char* bgr) {
    int sy, sx;
    fr_source_pixel(f.h, f.w, rot, y, x, &sy, &sx);
    fr_fetch(f, fmt, sy, sx, bgr);
}

}  // namespace b2p
