// Video-frame ingestion on the device: NV12 / I420 / pitched BGR frames -> rotated uint8 HWC BGR frames packed back to
// back, what cv2.rotate(cv2.cvtColor(...)) gives (core in frame_core.h).
#pragma once
#include <cuda_runtime.h>

#include "frame_core.h"

namespace b2p {

// frames [n] (device table; planes in device memory) of format `fmt`, rotated by `rot` degrees clockwise -> out +
// frames[i].off, [oh_i, ow_i, 3] each.  max_px: the largest rotated frame's pixel count (sizes the grid).
cudaError_t convert_frames_launch(const FrameSrc* frames, int n, int fmt, int rot, long max_px, unsigned char* out,
                                  cudaStream_t s);

}  // namespace b2p
