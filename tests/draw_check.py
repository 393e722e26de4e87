"""Shared by tests/test_draw_host.py and tests/test_gpu_draw.py: the host build of csrc/draw_core.h
(tests/cuda/draw_core_host.cpp) and seeded person rows (B200POSE_HUMAN_FLOATS layout) for the composition cases."""
import ctypes
import os
import subprocess

import numpy as np

from conftest import ROOT

FLOATS = 73


def compile_core(so, core=None, reverse_persons=False):
    """The host drawing core as a ctypes library; `core` replaces draw_core.h (a copy with a planted mistake);
    reverse_persons draws the persons of a frame last to first (a planted mistake of the composition)."""
    cmd = ["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-o", so,
           os.path.join(ROOT, "tests", "cuda", "draw_core_host.cpp")]
    if core:
        cmd.insert(1, '-DDRAW_CORE="%s"' % core)
    if reverse_persons:
        cmd.insert(1, "-DDRAW_REVERSE_PERSONS")
    subprocess.run(cmd, check=True)
    lib = ctypes.CDLL(so)
    V, I = ctypes.c_void_p, ctypes.c_int
    lib.core_circle.argtypes = [V, I, I, I, I, V]
    lib.core_line.argtypes = [V, I, I, I, I, I, I, V]
    lib.core_draw.argtypes = [V, I, I, I, I, V, I]
    return lib


def core_draw(lib, frame, rows, net_h, net_w):
    """draw_humans(frame, humans_from_rows(rows, net_w, net_h)) in place, by the host core."""
    rows = np.ascontiguousarray(rows, np.float32).reshape(-1, FLOATS)
    h, w = frame.shape[:2]
    assert frame.flags.c_contiguous
    lib.core_draw(frame.ctypes.data, h, w, int(net_h), int(net_w), rows.ctypes.data, len(rows))
    return frame


def person_rows(n, seed, net_h, net_w, box=(140, 70), spread=None, drop=0.15, edge=True):
    """n person rows in pixels of a net_h x net_w input: each person's parts in a box (h, w) of network pixels placed
    anywhere in the input (or in `spread`, a wider range, for long limbs), some parts missing (peak id -1), some at
    x = net_w (the centre falls on the frame's right edge) and some on half-pixel positions."""
    rs = np.random.RandomState(seed)
    rows = np.zeros((n, FLOATS), np.float32)
    for i in range(n):
        rows[i, 0] = rs.uniform(0.3, 2.0)
        if spread is None:
            y0, x0 = rs.uniform(-10, net_h - box[0] + 10), rs.uniform(-10, net_w - box[1] + 10)
            ys, xs = y0 + rs.uniform(0, box[0], 18), x0 + rs.uniform(0, box[1], 18)
        else:
            ys, xs = rs.uniform(-spread, net_h + spread, 18), rs.uniform(-spread, net_w + spread, 18)
        ys, xs = np.clip(ys, 0, net_h), np.clip(xs, 0, net_w)
        half = rs.rand(18) < 0.2
        xs[half] = np.floor(xs[half]) + 0.5
        ys[half] = np.floor(ys[half]) + 0.5
        if edge:
            xs[rs.rand(18) < 0.06] = net_w
        cid = np.arange(18, dtype=np.float32) + 100 * i
        cid[rs.rand(18) < drop] = -1
        rows[i, 1::4], rows[i, 2::4], rows[i, 3::4], rows[i, 4::4] = xs, ys, rs.uniform(0.1, 1, 18), cid
    return rows


def overlap_pixels(frame_shape, rows, net_h, net_w, lib):
    """Pixels covered by two or more primitives of different colours (each primitive drawn alone on a blank frame)."""
    from lib.utils.common import CocoColors, CocoPairsRender
    h, w = frame_shape[:2]
    seen = np.full((h, w), -1, np.int64)
    clash = np.zeros((h, w), bool)

    def add(img, k):
        m = img.any(-1)
        clash[m & (seen >= 0) & (seen != k)] = True
        seen[m] = k

    for r in np.asarray(rows, np.float32).reshape(-1, FLOATS):
        c = {p: (int(float(r[1 + 4 * p]) / net_w * w + 0.5), int(float(r[2 + 4 * p]) / net_h * h + 0.5))
             for p in range(18) if r[4 + 4 * p] >= 0}
        for p, (x, y) in c.items():
            img = np.zeros((h, w, 3), np.uint8)
            lib.core_circle(img.ctypes.data, h, w, x, y, np.array(CocoColors[p], np.uint8).ctypes.data)
            add(img, p)
        for k, (a, b) in enumerate(CocoPairsRender):
            if a in c and b in c:
                img = np.zeros((h, w, 3), np.uint8)
                lib.core_line(img.ctypes.data, h, w, *c[a], *c[b], np.array(CocoColors[k], np.uint8).ctypes.data)
                add(img, k)
    return int(clash.sum())
