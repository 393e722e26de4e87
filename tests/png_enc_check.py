"""Shared by tests/test_png_encode_host.py and tests/test_gpu_png_encode.py: the host build of csrc/png_enc_core.h
(tests/cuda/png_enc_core_host.cpp), cv2.imencode('.png') at its defaults, and seeded frames."""
import ctypes
import os
import subprocess

import numpy as np

from conftest import ROOT

HOST_SRC = os.path.join(ROOT, "tests", "cuda", "png_enc_core_host.cpp")
CSRC = os.path.join(ROOT, "pytorch_realtime_multi-person_pose_estimation_b200", "csrc")


def compile_core(so, core=None):
    """The host encoding core as a ctypes library; `core` replaces png_enc_core.h (a copy with a planted mistake)."""
    cmd = ["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-I", CSRC, "-o", so, HOST_SRC]
    if core:
        cmd.insert(1, '-DPNG_ENC_CORE="%s"' % core)
    subprocess.run(cmd, check=True)
    lib = ctypes.CDLL(so)
    lib.core_encode.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_longlong]
    lib.core_encode.restype = ctypes.c_longlong
    lib.core_encode_bound.argtypes = [ctypes.c_int, ctypes.c_int]
    lib.core_encode_bound.restype = ctypes.c_longlong
    return lib


def core_encode(lib, img):
    """The host core's PNG file of a uint8 [h, w, 3] BGR frame, as bytes."""
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape[:2]
    cap = lib.core_encode_bound(h, w)
    out = np.empty(cap, np.uint8)
    n = lib.core_encode(img.ctypes.data, h, w, out.ctypes.data, cap)
    assert n > 0, n
    return out[:n].tobytes()


def cv2_encode(img):
    import cv2
    ok, buf = cv2.imencode(".png", img)
    assert ok
    return buf.tobytes()


def unfilter(filtered, h, w):
    """The BGR frame whose Sub-filtered rows (filter bytes left out) are `filtered` ([h, 3w] uint8): lets a test choose
    the deflate input byte for byte."""
    f = np.asarray(filtered, np.uint8).reshape(h, 3 * w).astype(np.int64)
    raw = np.zeros_like(f)
    for x in range(3 * w):
        raw[:, x] = (f[:, x] + (raw[:, x - 3] if x >= 3 else 0)) % 256
    return np.ascontiguousarray(raw.reshape(h, w, 3)[:, :, ::-1].astype(np.uint8))


def frame(h, w, seed, kind="photo"):
    """Seeded BGR frames: 'photo' (jpeg_check.content: smooth shapes, dynamic blocks), 'noise' (uniform bytes: stored
    blocks), 'flat' (one colour: 258-byte matches), 'stripes' (vertical bands: runs within and across rows), 'norun'
    (no two equal filtered bytes in a row: literals only), 'drawn' (photo with filled rectangles and lines)."""
    import jpeg_check
    rs = np.random.RandomState(seed)
    if kind == "photo":
        return jpeg_check.content(h, w, seed, "photo")
    if kind == "noise":
        return rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
    if kind == "flat":
        return np.broadcast_to(rs.randint(0, 256, 3).astype(np.uint8), (h, w, 3)).copy()
    if kind == "stripes":
        band = rs.randint(1, 9)
        cols = rs.randint(0, 256, ((w + band - 1) // band + 1, 3)).astype(np.uint8)
        return np.ascontiguousarray(np.broadcast_to(np.repeat(cols, band, axis=0)[:w], (h, w, 3)))
    if kind == "norun":
        f = np.zeros((h, 3 * w), np.int64)
        f[:, 0] = 2 + (np.arange(h) % 7)          # never the filter byte 1, never equal to its neighbours
        for x in range(1, 3 * w):
            f[:, x] = (f[:, x - 1] + 1 + rs.randint(0, 200, h)) % 256
            f[:, x] = np.where(f[:, x] == 1, 3, f[:, x])
            f[:, x] = np.where(f[:, x] == f[:, x - 1], (f[:, x] + 2) % 256, f[:, x])
        return unfilter(f, h, w)
    if kind == "drawn":
        img = jpeg_check.content(h, w, seed, "photo")
        for _ in range(4):
            y0, x0 = rs.randint(0, h), rs.randint(0, w)
            img[y0:y0 + rs.randint(1, 40), x0:x0 + rs.randint(1, 60)] = rs.randint(0, 256, 3)
            img[rs.randint(0, h), :] = rs.randint(0, 256, 3)
        return img
    raise ValueError(kind)
