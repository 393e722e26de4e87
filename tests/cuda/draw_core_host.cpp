// Host build of the person-drawing core (csrc/draw_core.h): the same plans and cover tests draw.cu evaluates, applied
// primitive after primitive to an h x w BGR frame (the last covering primitive decides a pixel, as on the device).
// DRAW_CORE overrides the header's path, so that a test can compile a copy with a planted mistake;
// DRAW_REVERSE_PERSONS plants one in the composition (persons drawn last to first).
#ifndef DRAW_CORE
#define DRAW_CORE "../../pytorch_realtime_multi-person_pose_estimation_b200/csrc/draw_core.h"
#endif
#include DRAW_CORE

using namespace b2p;

static void paint(const DrawPrim& p, unsigned char* img, int w, const unsigned char* bgr) {
    if (p.kind == 0) return;
    for (int y = p.y0; y <= p.y1; ++y)
        for (int x = p.x0; x <= p.x1; ++x)
            if (draw_covers(p, x, y)) {
                unsigned char* q = img + 3 * ((long)y * w + x);
                q[0] = bgr[0];
                q[1] = bgr[1];
                q[2] = bgr[2];
            }
}

// cv2.circle(img, (cx, cy), 3, bgr, thickness=3, lineType=8, shift=0)
extern "C" int core_circle(unsigned char* img, int h, int w, int cx, int cy, const unsigned char* bgr) {
    DrawPrim p;
    draw_plan_circle(h, w, cx, cy, p);
    paint(p, img, w, bgr);
    return 0;
}

// cv2.line(img, (x0, y0), (x1, y1), bgr, 3)
extern "C" int core_line(unsigned char* img, int h, int w, int x0, int y0, int x1, int y1, const unsigned char* bgr) {
    DrawPrim p;
    draw_plan_limb(h, w, x0, y0, x1, y1, p);
    paint(p, img, w, bgr);
    return 0;
}

// draw_humans(img, humans_from_rows(rows, net_w, net_h)) for n person rows of B200POSE_HUMAN_FLOATS floats
extern "C" int core_draw(unsigned char* img, int h, int w, int net_h, int net_w, const float* rows, int n) {
    for (int j = 0; j < n; ++j)
        for (int k = 0; k < kDrawPrimsPerPerson; ++k) {
#ifdef DRAW_REVERSE_PERSONS
            const int i = n - 1 - j;
#else
            const int i = j;
#endif
            DrawPrim p;
            draw_plan(rows + (long)i * kDrawRowFloats, h, w, net_h, net_w, k, p);
            paint(p, img, w, p.bgr);
        }
    return 0;
}
