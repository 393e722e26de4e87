"""Shared by the training-batch tests (DESIGN.md 2.20): the fixtures of tests/golden/make_aug_golden.py, the host build of
csrc/aug_core.h (tests/cuda/aug_core_host.cpp) and a host restatement of the whole per-sample path on top of it, with
cv2 for the JPEG round trip."""
import ctypes
import glob
import json
import os
import subprocess

import numpy as np

from conftest import ROOT, pkg_module

GOLDEN = os.path.join(ROOT, "tests", "golden")
HOST_SRC = os.path.join(ROOT, "tests", "cuda", "aug_core_host.cpp")
CORE_H = os.path.join(ROOT, "pytorch_realtime_multi-person_pose_estimation_b200", "csrc", "aug_core.h")
MEAN = np.array([0.485, 0.456, 0.406], np.float32)
STD = np.array([0.229, 0.224, 0.225], np.float32)

# (name, original text of aug_core.h, replacement): each plants one mistake the goldens must catch.  Rounding the
# fixed-point weights half up instead of away from zero moves negative weights by one unit in 2^22 and changed no
# golden pixel, so it is not among them.
PLANTED = [
    ("fixed_point_truncated", "k[x] = v < 0 ? (int32_t)AUG_DADD(-0.5, f) : (int32_t)AUG_DADD(0.5, f);",
     "k[x] = (int32_t)f;"),
    ("weights_normalised_in_float", "const double v = ww != 0.0 ? AUG_DDIV(w[x], ww) : w[x];",
     "const double v = ww != 0.0 ? (double)((float)w[x] / (float)ww) : w[x];"),
    ("fma_in_blend", "AUG_FADD((float)in1, AUG_FMUL(a, (float)(in2 - in1)))", "fmaf(a, (float)(in2 - in1), (float)in1)"),
]


def goldens():
    return {os.path.basename(p)[4:-4]: dict(np.load(p)) for p in sorted(glob.glob(os.path.join(GOLDEN, "aug_*.npz")))}


def cube():
    with open(os.path.join(GOLDEN, "aug_cube.json")) as f:
        return json.load(f)


def compile_core(out, header=None):
    cmd = ["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-o", out, HOST_SRC]
    if header:
        cmd.insert(1, '-DAUG_CORE="%s"' % header)
    subprocess.run(cmd, check=True)
    lib = ctypes.CDLL(out)
    vp, ci = ctypes.c_void_p, ctypes.c_int
    lib.core_resize.argtypes = [vp, ci, ci, ci, ci, vp]
    lib.core_pixels.argtypes = [ci, vp, ctypes.c_longlong, ctypes.c_double, ci]
    lib.core_jitter.argtypes = [vp, ctypes.c_longlong, vp, vp]
    lib.core_ground_truth_f64.argtypes = [vp, ci, ci, ci, vp, vp]
    return lib


def planted_header(tmpdir, name):
    src = open(CORE_H).read()
    old, new = next((o, n) for k, o, n in PLANTED if k == name)
    assert src.count(old) == 1, name
    path = os.path.join(str(tmpdir), "aug_core_%s.h" % name)
    open(path, "w").write(src.replace(old, new))
    return path


def engine():
    return pkg_module("engine")


def params_of(g):
    import torch
    return engine().augment_params([g["src"].shape[:2]], torch.Generator().manual_seed(int(g["seed"])), int(g["edge"]))


def colour_stages(core, g, p, jpeg=True):
    """The host core's image ToTensor receives (RGB [E, E, 3]) for fixture g under params record p."""
    import cv2
    E = int(g["edge"])
    src = np.ascontiguousarray(g["src"][:, ::-1] if p["hflip"] else g["src"])
    (rw, rh), (x0, y0), (cw, ch), (left, top) = p["resized"], p["crop"], p["cropped"], p["pad"]
    h, w = src.shape[:2]
    res = np.empty((rh, rw, 3), np.uint8)
    core.core_resize(src.ctypes.data, h, w, rh, rw, res.ctypes.data)
    img = np.empty((E, E, 3), np.uint8)
    img[:] = engine().AUG_PAD
    img[top:top + ch, left:left + cw] = res[y0:y0 + ch, x0:x0 + cw]
    order = np.array(p["order"], np.int32)
    f = np.array(p["factors"], np.float64)
    core.core_jitter(img.ctypes.data, E * E, order.ctypes.data, f.ctypes.data)
    if jpeg and p["jpeg"]:
        ok, blob = cv2.imencode(".jpg", img[:, :, ::-1], [cv2.IMWRITE_JPEG_QUALITY, 50])
        img = np.ascontiguousarray(cv2.imdecode(blob, cv2.IMREAD_COLOR)[:, :, ::-1])
    if p["gray"]:
        lum = img.copy()
        core.core_pixels(4, lum.ctypes.data, E * E, 0.0, 0)
        img = np.repeat(lum[:, :, :1], 3, 2)
    return img


def to_tensor(u8, p):
    """ToTensor + Normalize + mask_valid_area of an RGB [E, E, 3] image, in float32 as torch computes them."""
    x = (u8.astype(np.float32).transpose(2, 0, 1) / np.float32(255) - MEAN[:, None, None]) / STD[:, None, None]
    x0, y0, x1, y1 = p["mask"]
    x[:, :y0] = 0
    x[:, :, :x0] = 0
    x[:, y1:] = 0
    x[:, :, x1:] = 0
    return x


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32 if a.dtype == np.float32 else np.uint64)
