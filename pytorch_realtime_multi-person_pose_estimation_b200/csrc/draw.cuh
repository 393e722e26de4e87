// Drawing of detected persons on the device: draw_humans' circles and limbs on packed uint8 HWC BGR frames, bit for bit
// what cv2 draws (core in draw_core.h).
#pragma once
#include <cuda_runtime.h>

#include "draw_core.h"

namespace b2p {

// One frame of a draw call: h x w pixels at byte offset `off` of the packed frames, coordinates in pixels of an
// net_h x net_w network input; its persons are rows person0 .. person0 + persons - 1 of the call.
struct DrawImage {
    int h, w, net_h, net_w;
    int person0, persons;
    long long off;
};

// images [n], rows [P][kDrawRowFloats] and person_img [P] (the frame of each row) in device memory; prims: room for
// P * kDrawPrimsPerPerson primitives.  Draws every frame in place; max_h / max_w: the largest frame (sizes the grid).
cudaError_t draw_launch(const DrawImage* images, int n, const float* rows, const int* person_img, int persons,
                        DrawPrim* prims, int max_h, int max_w, unsigned char* frames, cudaStream_t s);

}  // namespace b2p
