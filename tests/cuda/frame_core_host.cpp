// Host build of the video-frame ingestion core (csrc/frame_core.h: frame_px), walked over a frame exactly as
// convert_frames_kernel walks it, optionally followed by the raw-frame mirror of flip test-time averaging and by
// crop_with_factor (csrc/resize_core.h: crop_px), the two stages that read the converted frame on the device.
// FRAME_CORE overrides the header's path, so that a test can compile a copy with a planted mistake.
#include <vector>

#ifndef FRAME_CORE
#define FRAME_CORE "../../pytorch_realtime_multi-person_pose_estimation_b200/csrc/frame_core.h"
#endif
#include FRAME_CORE
#include "../../pytorch_realtime_multi-person_pose_estimation_b200/csrc/resize_core.h"

using namespace b2p;

static FrameSrc frame_src(const unsigned char* const* planes, const int* pitch, int h, int w) {
    FrameSrc f{};
    for (int k = 0; k < 3; ++k) {
        f.plane[k] = planes[k];
        f.pitch[k] = pitch[k];
    }
    f.h = h;
    f.w = w;
    return f;
}

// planes[3] / pitch[3] of one stored h x w frame of format fmt -> out [oh, ow, 3] rotated by rot degrees clockwise;
// mirror: then out(y, x) = rotated(y, ow - 1 - x), what tta_mirror_u8hwc makes of it.
extern "C" int core_convert_frame(const unsigned char* const* planes, const int* pitch, int h, int w, int fmt, int rot,
                                  int mirror, unsigned char* out) {
    const FrameSrc f = frame_src(planes, pitch, h, w);
    int oh, ow;
    fr_rotated_size(h, w, rot, &oh, &ow);
    for (int y = 0; y < oh; ++y)
        for (int x = 0; x < ow; ++x) frame_px(f, fmt, rot, y, mirror ? ow - 1 - x : x, out + 3 * ((long)y * ow + x));
    return 0;
}

// The converted, rotated frame through crop_with_factor: out [pad_h, pad_w, 3].
extern "C" int core_convert_crop(const unsigned char* const* planes, const int* pitch, int h, int w, int fmt, int rot,
                                 int dest_size, int factor, unsigned char* out) {
    int oh, ow;
    fr_rotated_size(h, w, rot, &oh, &ow);
    std::vector<unsigned char> bgr((size_t)oh * ow * 3);
    core_convert_frame(planes, pitch, h, w, fmt, rot, 0, bgr.data());
    const CropGeom g = crop_geometry(oh, ow, dest_size, factor);
    for (int y = 0; y < g.pad_h; ++y)
        for (int x = 0; x < g.pad_w; ++x)
            for (int c = 0; c < 3; ++c)
                out[((long)y * g.pad_w + x) * 3 + c] = crop_px(bgr.data(), oh, ow, 3, g, y, x, c);
    return 0;
}
