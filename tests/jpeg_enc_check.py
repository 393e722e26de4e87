"""Shared by tests/test_jpeg_encode_host.py and tests/test_gpu_jpeg_encode.py: the host build of csrc/jpeg_enc_core.h
(tests/cuda/jpeg_enc_core_host.cpp), cv2.imencode at the encoder's settings, and seeded frames."""
import ctypes
import os
import subprocess

import numpy as np

from conftest import ROOT

HOST_SRC = os.path.join(ROOT, "tests", "cuda", "jpeg_enc_core_host.cpp")
CSRC = os.path.join(ROOT, "pytorch_realtime_multi-person_pose_estimation_b200", "csrc")
SAMPLING = {"420": 0x221111, "422": 0x211111, "440": 0x121111, "411": 0x411111, "444": 0x111111}


def compile_core(so, core=None):
    """The host encoding core as a ctypes library; `core` replaces jpeg_enc_core.h (a copy with a planted mistake)."""
    cmd = ["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-I", CSRC, "-o", so, HOST_SRC]
    if core:
        cmd.insert(1, '-DJPEG_ENC_CORE="%s"' % core)
    subprocess.run(cmd, check=True)
    lib = ctypes.CDLL(so)
    lib.core_encode.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int,
                                ctypes.c_void_p, ctypes.c_longlong]
    lib.core_encode.restype = ctypes.c_longlong
    lib.core_encode_bound.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int]
    lib.core_encode_bound.restype = ctypes.c_longlong
    lib.core_reciprocal.argtypes = [ctypes.c_int, ctypes.c_void_p]
    return lib


def core_encode(lib, img, quality=95, sampling="420"):
    """The host core's stream of a uint8 [h, w, 3] BGR frame, as bytes."""
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape[:2]
    cap = lib.core_encode_bound(h, w, SAMPLING[sampling])
    out = np.empty(cap, np.uint8)
    n = lib.core_encode(img.ctypes.data, h, w, int(quality), SAMPLING[sampling], out.ctypes.data, cap)
    assert n > 0, n
    return out[:n].tobytes()


def cv2_encode(img, quality=95, sampling="420"):
    import cv2
    ok, buf = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, int(quality),
                                         cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMPLING[sampling]])
    assert ok
    return buf.tobytes()


def frame(h, w, seed, kind="photo"):
    """Seeded BGR frames: 'photo' (jpeg_check.content), 'checker' (0 / 255 squares: long codes, ZRL runs), 'noise'
    (uniform bytes: many stuffed 0xFF bytes), 'flat' (one colour: EOB-only blocks), 'saturated' (0 / 255 channels)."""
    import jpeg_check
    rs = np.random.RandomState(seed)
    if kind in ("photo", "checker"):
        return jpeg_check.content(h, w, seed, kind)
    if kind == "noise":
        return rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
    if kind == "flat":
        return np.broadcast_to(rs.randint(0, 256, 3).astype(np.uint8), (h, w, 3)).copy()
    if kind == "saturated":
        return (rs.randint(0, 2, (h, w, 3)) * 255).astype(np.uint8)
    raise ValueError(kind)
