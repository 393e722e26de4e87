// Drawing of detected persons, host/device shared core: lib/utils/common.py draw_humans on an h x w BGR frame, i.e.
//   cv2.circle(img, c, 3, color, thickness=3, lineType=8, shift=0)  and  cv2.line(img, p0, p1, color, 3)
// restated from OpenCV 4.13's drawing code (imgproc/src/drawing.cpp), clipping included.  Colours are written, not
// blended, so a primitive is fully described by its pixel set and its colour.
//
// Both calls reduce to ThickLine segments in 16.16 fixed point.  A segment of thickness 3 covers the union of
//   - FillConvexPoly of the quadrilateral p0 +- dp, p1 -+ dp (dp = the normal of half-length 2, rounded to 1/65536):
//     the four outline edges drawn by Line2 (a fixed-point DDA after clipLine) and the scan-line fill between the two
//     edge chains, whose x advance by a rounded per-row step;
//   - a filled Bresenham circle of radius 2 at each end the segment's flags ask for (the round caps).
// cv2.line is one segment with both caps.  cv2.circle of radius 3 is the 13-point polygon ellipse2Poly makes with a
// 30 degree step (SinTable values), drawn as an open PolyLine: 12 segments, the first with both caps, the others with
// their end cap.
//
// Instead of replaying the rasteriser, the core answers "does primitive k cover pixel (x, y)" in O(1): draw_plan()
// solves a primitive's fill chains, DDA parameters and caps once, and the cover tests evaluate them at any pixel, so a
// pixel's colour is that of the last primitive in draw order that covers it.  A circle is small: its plan is a 16 x 16
// bit mask around its centre.  The same functions run in draw.cu and in the host build of the tests, which compare
// them to cv2 (tests/test_draw_host.py).
#pragma once

#include <stdint.h>

#if defined(__CUDACC__)
#define B2P_DR_HD __host__ __device__ __forceinline__
#else
#define B2P_DR_HD inline
#endif

namespace b2p {

constexpr int kDrawParts = 18;               // CocoPart 0 .. 17 (Background is never drawn)
constexpr int kDrawLimbs = 17;               // CocoPairsRender
constexpr int kDrawPrimsPerPerson = kDrawParts + kDrawLimbs;
constexpr int kDrawRowFloats = 1 + 4 * kDrawParts;     // B200POSE_HUMAN_FLOATS
constexpr int kDrawMask = 16;                // circle mask: rows / columns cy - 7 .. cy + 8
constexpr int kDrawMaskOrg = 7;

constexpr int kXYShift = 16;
constexpr long long kXYOne = 1LL << kXYShift;

// CocoColors (B, G, R) and CocoPairsRender (lib/utils/common.py)
B2P_DR_HD void draw_color(int k, unsigned char* bgr) {
    const unsigned char c[kDrawParts][3] = {
        {255, 0, 0}, {255, 85, 0}, {255, 170, 0}, {255, 255, 0}, {170, 255, 0}, {85, 255, 0}, {0, 255, 0},
        {0, 255, 85}, {0, 255, 170}, {0, 255, 255}, {0, 170, 255}, {0, 85, 255}, {0, 0, 255}, {85, 0, 255},
        {170, 0, 255}, {255, 0, 255}, {255, 0, 170}, {255, 0, 85}};
    bgr[0] = c[k][0];
    bgr[1] = c[k][1];
    bgr[2] = c[k][2];
}
B2P_DR_HD void draw_pair(int k, int* a, int* b) {
    const unsigned char p[kDrawLimbs][2] = {{1, 2}, {1, 5}, {2, 3}, {3, 4}, {5, 6}, {6, 7}, {1, 8}, {8, 9}, {9, 10},
                                            {1, 11}, {11, 12}, {12, 13}, {1, 0}, {0, 14}, {14, 16}, {0, 15}, {15, 17}};
    *a = p[k][0];
    *b = p[k][1];
}

// double arithmetic exactly as written (no FMA contraction on the device; the host build uses -ffp-contract=off)
B2P_DR_HD double dr_mul(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
B2P_DR_HD double dr_div(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}
B2P_DR_HD double dr_add(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
B2P_DR_HD double dr_sqrt(double a) {
#if defined(__CUDA_ARCH__)
    return __dsqrt_rn(a);
#else
    return __builtin_sqrt(a);
#endif
}
// cvRound(double): round half to even
B2P_DR_HD long long dr_round(double v) {
#if defined(__CUDA_ARCH__)
    return __double2ll_rn(v);
#else
    return __builtin_llrint(v);
#endif
}

// Centre of a part: int(float(x) / net_w * w + 0.5) (humans_from_rows, then draw_humans), truncated toward zero.
B2P_DR_HD int draw_centre(float v, int net, int size) {
    return (int)dr_add(dr_mul(dr_div((double)v, (double)net), (double)size), 0.5);
}

struct DrawPt {
    long long x, y;
};

// Line2 after clipLine: pixels (m0 + k, (a + k * step) >> 16) for k = 0 .. count (x-major; y-major swaps x and y), plus
// the rounded end point (ex, ey).
struct DrawDDA {
    long long a, step;
    int m0, count, xmaj, valid, ex, ey;
};

// One edge chain of the scan-line fill: from row y[i] on, x = x[i] + dx[i] * (row - y[i]).
struct DrawChain {
    int n, y[4];
    long long x[4], dx[4];
};

struct DrawSeg {
    DrawDDA e[4];
    DrawChain side[2];
    int fy0, fy1;            // rows the fill covers (fy0 > fy1: none)
    int cx[2], cy[2], caps;  // cap centres, cap i drawn iff caps & (1 << i)
    int x0, y0, x1, y1;      // a bounding box of everything above
};

// clipLine(Size2l, pt1, pt2) on the image scaled to 16.16
B2P_DR_HD bool dr_clip(long long W, long long H, DrawPt& p1, DrawPt& p2) {
    const long long right = W - 1, bottom = H - 1;
    if (W <= 0 || H <= 0) return false;
    long long &x1 = p1.x, &y1 = p1.y, &x2 = p2.x, &y2 = p2.y;
    int c1 = (x1 < 0) + (x1 > right) * 2 + (y1 < 0) * 4 + (y1 > bottom) * 8;
    int c2 = (x2 < 0) + (x2 > right) * 2 + (y2 < 0) * 4 + (y2 > bottom) * 8;
    if ((c1 & c2) == 0 && (c1 | c2) != 0) {
        long long a;
        if (c1 & 12) {
            a = c1 < 8 ? 0 : bottom;
            x1 += (long long)dr_div(dr_mul((double)(a - y1), (double)(x2 - x1)), (double)(y2 - y1));
            y1 = a;
            c1 = (x1 < 0) + (x1 > right) * 2;
        }
        if (c2 & 12) {
            a = c2 < 8 ? 0 : bottom;
            x2 += (long long)dr_div(dr_mul((double)(a - y2), (double)(x2 - x1)), (double)(y2 - y1));
            y2 = a;
            c2 = (x2 < 0) + (x2 > right) * 2;
        }
        if ((c1 & c2) == 0 && (c1 | c2) != 0) {
            if (c1) {
                a = c1 == 1 ? 0 : right;
                y1 += (long long)dr_div(dr_mul((double)(a - x1), (double)(y2 - y1)), (double)(x2 - x1));
                x1 = a;
                c1 = 0;
            }
            if (c2) {
                a = c2 == 1 ? 0 : right;
                y2 += (long long)dr_div(dr_mul((double)(a - x2), (double)(y2 - y1)), (double)(x2 - x1));
                x2 = a;
                c2 = 0;
            }
        }
    }
    return (c1 | c2) == 0;
}

// Line2(img, p1, p2): an 8-connected fixed-point line
B2P_DR_HD DrawDDA dr_line2(int h, int w, DrawPt p1, DrawPt p2) {
    DrawDDA d{};
    if (!dr_clip((long long)w << kXYShift, (long long)h << kXYShift, p1, p2)) return d;
    long long dx = p2.x - p1.x, dy = p2.y - p1.y;
    const long long j = dx < 0 ? -1 : 0, ax = (dx ^ j) - j;
    const long long i = dy < 0 ? -1 : 0, ay = (dy ^ i) - i;
    d.valid = 1;
    d.xmaj = ax > ay;
    const long long s = d.xmaj ? j : i;      // swap the end points when the major coordinate decreases
    if (s) {
        const DrawPt t = p1;
        p1 = p2;
        p2 = t;
    }
    if (d.xmaj) {
        dy = (dy ^ j) - j;
        d.step = (dy * kXYOne) / (ax | 1);
        d.count = (int)((p2.x - p1.x) >> kXYShift);
    } else {
        dx = (dx ^ i) - i;
        d.step = (dx * kXYOne) / (ay | 1);
        d.count = (int)((p2.y - p1.y) >> kXYShift);
    }
    d.ex = (int)((p2.x + (kXYOne >> 1)) >> kXYShift);
    d.ey = (int)((p2.y + (kXYOne >> 1)) >> kXYShift);
    p1.x += kXYOne >> 1;
    p1.y += kXYOne >> 1;
    d.m0 = (int)((d.xmaj ? p1.x : p1.y) >> kXYShift);
    d.a = d.xmaj ? p1.y : p1.x;
    return d;
}

B2P_DR_HD bool dr_dda_covers(const DrawDDA& d, int x, int y) {
    if (!d.valid) return false;
    if (x == d.ex && y == d.ey) return true;
    const int k = (d.xmaj ? x : y) - d.m0;
    if (k < 0 || k > d.count) return false;
    return (int)((d.a + (long long)k * d.step) >> kXYShift) == (d.xmaj ? y : x);
}

// FillConvexPoly(img, v, 4, color, 8, XY_SHIFT): outline edges and the edge chains of the scan-line fill
B2P_DR_HD void dr_fill_plan(int h, int w, const DrawPt* v, DrawSeg& s) {
    constexpr int npts = 4;
    constexpr long long delta = kXYOne >> 1;
    long long xmin = v[0].x, xmax = v[0].x, ymin = v[0].y, ymax = v[0].y;
    int imin = 0;
    DrawPt p0 = v[npts - 1];
    for (int i = 0; i < npts; ++i) {
        if (v[i].y < ymin) {
            ymin = v[i].y;
            imin = i;
        }
        ymax = v[i].y > ymax ? v[i].y : ymax;
        xmax = v[i].x > xmax ? v[i].x : xmax;
        xmin = v[i].x < xmin ? v[i].x : xmin;
        s.e[i] = dr_line2(h, w, p0, v[i]);
        p0 = v[i];
    }
    xmin = (xmin + delta) >> kXYShift;
    xmax = (xmax + delta) >> kXYShift;
    ymin = (ymin + delta) >> kXYShift;
    ymax = (ymax + delta) >> kXYShift;
    s.fy0 = 1;
    s.fy1 = 0;
    s.side[0].n = s.side[1].n = 0;
    if ((int)xmax < 0 || (int)ymax < 0 || (int)xmin >= w || (int)ymin >= h) return;
    if (ymax > h - 1) ymax = h - 1;
    // the scan loop, visiting only the rows where an edge chain moves on to its next vertex
    int eidx[2] = {imin, imin}, eye[2], edi[2] = {1, npts - 1};
    int edges = npts;
    int y = (int)ymin;
    eye[0] = eye[1] = y;
    s.fy0 = y;
    for (;;) {
        for (int i = 0; i < 2; ++i) {
            if (y < eye[i]) continue;
            int idx0 = eidx[i], di = edi[i];
            int idx = idx0 + di;
            if (idx >= npts) idx -= npts;
            for (; edges-- > 0;) {
                const int ty = (int)((v[idx].y + delta) >> kXYShift);
                if (ty > y) {
                    DrawChain& c = s.side[i];
                    c.y[c.n] = y;
                    c.x[c.n] = v[idx0].x;
                    c.dx[c.n] = ((v[idx].x - v[idx0].x) * 2 + ((long long)ty - y)) / (2 * ((long long)ty - y));
                    c.n += 1;
                    eye[i] = ty;
                    eidx[i] = idx;
                    break;
                }
                idx0 = idx;
                idx += di;
                if (idx >= npts) idx -= npts;
            }
        }
        if (edges < 0) {
            s.fy1 = y - 1;
            return;
        }
        const int next = eye[0] < eye[1] ? eye[0] : eye[1];
        if (next > (int)ymax) {
            s.fy1 = (int)ymax;
            return;
        }
        y = next;
    }
}

B2P_DR_HD long long dr_chain_x(const DrawChain& c, int y) {
    if (c.n == 0) return -kXYOne;      // the scan loop's initial edge: x = -XY_ONE, dx = 0
    int k = c.n - 1;
    while (k > 0 && c.y[k] > y) --k;
    return c.x[k] + c.dx[k] * (long long)(y - c.y[k]);
}

// Row half-widths of Circle(img, c, r, color, fill = 1), OpenCV's Bresenham filled circle: |y - cy| = ady covers
// |x - cx| <= the value returned, -1 if the row is not covered.
B2P_DR_HD int dr_disc_halfwidth(int r, int ady) {
    int hw = -1;
    int err = 0, dx = r, dy = 0, plus = 1, minus = (r << 1) - 1;
    while (dx >= dy) {
        if (ady == dy && dx > hw) hw = dx;
        if (ady == dx && dy > hw) hw = dy;
        dy++;
        err += plus;
        plus += 2;
        const int mask = (err <= 0) - 1;
        err -= minus & mask;
        dx += mask;
        minus -= mask & 2;
    }
    return hw;
}

// ThickLine(img, p0, p1, color, thickness = 3, LINE_8, flags, XY_SHIFT)
constexpr int kDrawThick = 3;
constexpr long long kDrawThickFx = (long long)kDrawThick << (kXYShift - 1);      // thickness <<= XY_SHIFT - 1
constexpr int kDrawCapR = (int)((kDrawThickFx + (kXYOne >> 1)) >> kXYShift);   // 2

B2P_DR_HD void dr_seg_plan(int h, int w, DrawPt p0, DrawPt p1, int flags, DrawSeg& s) {
    const double inv = 1. / kXYOne;
    const double dx = dr_mul((double)(p0.x - p1.x), inv), dy = dr_mul((double)(p1.y - p0.y), inv);
    double r = dr_add(dr_mul(dx, dx), dr_mul(dy, dy));
    const int odd = kDrawThick & 1;
    long long bx0 = p0.x < p1.x ? p0.x : p1.x, bx1 = p0.x < p1.x ? p1.x : p0.x;
    long long by0 = p0.y < p1.y ? p0.y : p1.y, by1 = p0.y < p1.y ? p1.y : p0.y;
    if ((r < 0 ? -r : r) > 2.220446049250313e-16) {
        r = dr_div((double)kDrawThickFx + odd * kXYOne * 0.5, dr_sqrt(r));
        const long long dpx = dr_round(dr_mul(dy, r)), dpy = dr_round(dr_mul(dx, r));
        const DrawPt v[4] = {{p0.x + dpx, p0.y + dpy}, {p0.x - dpx, p0.y - dpy}, {p1.x - dpx, p1.y - dpy},
                             {p1.x + dpx, p1.y + dpy}};
        dr_fill_plan(h, w, v, s);
        const long long ax = dpx < 0 ? -dpx : dpx, ay = dpy < 0 ? -dpy : dpy;
        bx0 -= ax; bx1 += ax; by0 -= ay; by1 += ay;
    } else {
        for (int i = 0; i < 4; ++i) s.e[i].valid = 0;
        s.fy0 = 1;
        s.fy1 = 0;
        s.side[0].n = s.side[1].n = 0;
    }
    s.caps = flags;
    s.cx[0] = (int)((p0.x + (kXYOne >> 1)) >> kXYShift);
    s.cy[0] = (int)((p0.y + (kXYOne >> 1)) >> kXYShift);
    s.cx[1] = (int)((p1.x + (kXYOne >> 1)) >> kXYShift);
    s.cy[1] = (int)((p1.y + (kXYOne >> 1)) >> kXYShift);
    // every pixel lies within a pixel of the fixed-point hull, caps included
    const int m = kDrawCapR + 2;
    s.x0 = (int)(bx0 >> kXYShift) - m;
    s.x1 = (int)(bx1 >> kXYShift) + m;
    s.y0 = (int)(by0 >> kXYShift) - m;
    s.y1 = (int)(by1 >> kXYShift) + m;
}

B2P_DR_HD bool dr_seg_covers(const DrawSeg& s, int x, int y) {
    if (x < s.x0 || x > s.x1 || y < s.y0 || y > s.y1) return false;
    if (y >= s.fy0 && y <= s.fy1) {
        long long a = dr_chain_x(s.side[0], y), b = dr_chain_x(s.side[1], y);
        if (a > b) {
            const long long t = a;
            a = b;
            b = t;
        }
        if ((int)((a + (kXYOne >> 1)) >> kXYShift) <= x && x <= (int)((b + (kXYOne >> 1)) >> kXYShift)) return true;
    }
    for (int i = 0; i < 4; ++i)
        if (dr_dda_covers(s.e[i], x, y)) return true;
    for (int i = 0; i < 2; ++i) {
        if (!(s.caps & (1 << i))) continue;
        const int ady = y > s.cy[i] ? y - s.cy[i] : s.cy[i] - y, adx = x > s.cx[i] ? x - s.cx[i] : s.cx[i] - x;
        if (ady <= kDrawCapR && adx <= dr_disc_halfwidth(kDrawCapR, ady)) return true;
    }
    return false;
}

// cv2.circle(radius 3, thickness 3): EllipseEx's polygon (ellipse2Poly, delta 30 degrees, 16.16 vertices)
constexpr int kDrawCircleR = 3;
constexpr int kDrawCirclePts = 13;

B2P_DR_HD int dr_circle_poly(int cx, int cy, DrawPt* v) {
    // SinTable at 0, 30, ..., 450 degrees (float values); cos(angle) = SinTable[450 - angle]
    const float sn[16] = {0.0000000f, 0.5000000f, 0.8660254f, 1.0000000f, 0.8660254f, 0.5000000f, 0.0000000f, -0.5000000f,
                          -0.8660254f, -1.0000000f, -0.8660254f, -0.5000000f, -0.0000000f, 0.5000000f, 0.8660254f,
                          1.0000000f};
    const double ax = (double)((long long)kDrawCircleR << kXYShift);
    const double ccx = (double)((long long)cx << kXYShift), ccy = (double)((long long)cy << kXYShift);
    int n = 0;
    for (int k = 0; k < kDrawCirclePts; ++k) {
        const float c = sn[15 - k], s = sn[k];
        // pt = center + x * alpha - y * beta, center + x * beta + y * alpha with alpha = 1, beta = 0
        const double x = dr_mul(ax, (double)c), y = dr_mul(ax, (double)s);
        const double px = dr_add(dr_add(ccx, dr_mul(x, 1.0)), -dr_mul(y, 0.0));
        const double py = dr_add(dr_add(ccy, dr_mul(x, 0.0)), dr_mul(y, 1.0));
        DrawPt p;
        p.x = dr_round(dr_div(px, (double)kXYOne)) << kXYShift;
        p.y = dr_round(dr_div(py, (double)kXYOne)) << kXYShift;
        p.x += dr_round(dr_add(px, -(double)p.x));
        p.y += dr_round(dr_add(py, -(double)p.y));
        if (n == 0 || p.x != v[n - 1].x || p.y != v[n - 1].y) v[n++] = p;
    }
    return n;
}

// A planned primitive: a limb (one segment) or a circle (a bit mask of kDrawMask rows around its centre).
struct DrawPrim {
    int kind;                       // 0: nothing, 1: circle, 2: limb
    int x0, y0, x1, y1;             // bounding box, clipped to the image (inclusive)
    unsigned char bgr[4];
    int cx, cy;                     // circle centre
    unsigned short mask[kDrawMask]; // circle: bit c of row r = pixel (cx - 7 + c, cy - 7 + r)
    DrawSeg seg;                    // limb
};

B2P_DR_HD bool dr_clip_box(int h, int w, DrawPrim& p) {
    p.x0 = p.x0 < 0 ? 0 : p.x0;
    p.y0 = p.y0 < 0 ? 0 : p.y0;
    p.x1 = p.x1 > w - 1 ? w - 1 : p.x1;
    p.y1 = p.y1 > h - 1 ? h - 1 : p.y1;
    return p.x0 <= p.x1 && p.y0 <= p.y1;
}

B2P_DR_HD void draw_plan_circle(int h, int w, int cx, int cy, DrawPrim& p) {
    p.kind = 1;
    p.cx = cx;
    p.cy = cy;
    p.x0 = cx - kDrawMaskOrg;
    p.y0 = cy - kDrawMaskOrg;
    p.x1 = p.x0 + kDrawMask - 1;
    p.y1 = p.y0 + kDrawMask - 1;
    for (int r = 0; r < kDrawMask; ++r) p.mask[r] = 0;
    if (!dr_clip_box(h, w, p)) {
        p.kind = 0;
        return;
    }
    DrawPt v[kDrawCirclePts];
    const int n = dr_circle_poly(cx, cy, v);
    for (int k = 0; k + 1 < n; ++k) {       // PolyLine(v, n, open): flags 3 on the first segment, 2 after it
        DrawSeg s;
        dr_seg_plan(h, w, v[k], v[k + 1], k == 0 ? 3 : 2, s);
        for (int y = p.y0; y <= p.y1; ++y)
            for (int x = p.x0; x <= p.x1; ++x)
                if (dr_seg_covers(s, x, y))
                    p.mask[y - cy + kDrawMaskOrg] |= (unsigned short)(1u << (x - cx + kDrawMaskOrg));
    }
}

// cv2.line(img, a, b, color, 3): with shift 0 the end points are first clipped (clipLine, integer coordinates) to the
// image grown by the thickness on every side; then one segment with both caps.
constexpr int kDrawLineMargin = kDrawThick;

B2P_DR_HD void draw_plan_limb(int h, int w, int ax, int ay, int bx, int by, DrawPrim& p) {
    p.kind = 0;
    const int m = kDrawLineMargin;
    DrawPt a{(long long)ax + m, (long long)ay + m}, b{(long long)bx + m, (long long)by + m};
    if (!dr_clip((long long)w + 2 * m, (long long)h + 2 * m, a, b)) return;
    p.kind = 2;
    dr_seg_plan(h, w, DrawPt{(a.x - m) << kXYShift, (a.y - m) << kXYShift}, DrawPt{(b.x - m) << kXYShift, (b.y - m) << kXYShift},
                3, p.seg);
    p.x0 = p.seg.x0;
    p.y0 = p.seg.y0;
    p.x1 = p.seg.x1;
    p.y1 = p.seg.y1;
    if (!dr_clip_box(h, w, p)) p.kind = 0;
}

B2P_DR_HD bool draw_covers(const DrawPrim& p, int x, int y) {
    if (x < p.x0 || x > p.x1 || y < p.y0 || y > p.y1) return false;
    if (p.kind == 1) return (p.mask[y - p.cy + kDrawMaskOrg] >> (x - p.cx + kDrawMaskOrg)) & 1u;
    return p.kind == 2 && dr_seg_covers(p.seg, x, y);
}

// Primitive `slot` (0 .. kDrawPrimsPerPerson - 1) of one person row on an h x w frame whose coordinates are in pixels
// of an net_h x net_w network input, in draw_humans' order: the circles of parts 0 .. 17, then the limbs of
// CocoPairsRender.  A part is present iff its peak id is >= 0.
B2P_DR_HD void draw_plan(const float* row, int h, int w, int net_h, int net_w, int slot, DrawPrim& p) {
    p.kind = 0;
    auto has = [&](int part) { return row[1 + 4 * part + 3] >= 0.f; };
    auto cx = [&](int part) { return draw_centre(row[1 + 4 * part], net_w, w); };
    auto cy = [&](int part) { return draw_centre(row[1 + 4 * part + 1], net_h, h); };
    if (slot < kDrawParts) {
        if (!has(slot)) return;
        draw_color(slot, p.bgr);
        draw_plan_circle(h, w, cx(slot), cy(slot), p);
        return;
    }
    const int k = slot - kDrawParts;
    int a, b;
    draw_pair(k, &a, &b);
    if (!has(a) || !has(b)) return;
    draw_color(k, p.bgr);
    draw_plan_limb(h, w, cx(a), cy(a), cx(b), cy(b), p);
}

}  // namespace b2p
