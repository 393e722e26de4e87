"""Shared by the training-target tests (DESIGN.md 2.19): the golden fixtures, the host build of csrc/gt_core.h
(tests/cuda/gt_core_host.cpp), copies of the core with planted mistakes, and seeded random scenarios."""
import ctypes
import glob
import os
import subprocess

import numpy as np

from conftest import GOLDEN, ROOT

CSRC = os.path.join(ROOT, "pytorch_realtime_multi-person_pose_estimation_b200", "csrc")
HOST_SRC = os.path.join(ROOT, "tests", "cuda", "gt_core_host.cpp")
CORE = os.path.join(CSRC, "gt_core.h")

# (name, original text of gt_core.h, replacement): each plants one mistake the golden comparison must catch
PLANTED = [
    ("no_clamp", "            if (acc > 1.0) acc = 1.0;\n", ""),
    ("fma_limb_width", "fabs(GT_SUB(GT_MUL(bax, L.uy), GT_MUL(bay, L.ux)))", "fabs(GT_FMA(bax, L.uy, -GT_MUL(bay, L.ux)))"),
    ("round_half_up", "#define GT_RINT(a) std::nearbyint(a)", "#define GT_RINT(a) std::floor((a) + 0.5)"),
    ("neck_visibility_max", "rs[2] * ls[2];", "(rs[2] > ls[2] ? rs[2] : ls[2]);"),
    ("x_equal_input_x_legal", "if (x >= fx ||", "if (x > fx ||"),
]
# Variants that give the reference's results on every golden, so that no comparison can fail on them.  Clamping once
# after all persons equals clamping after each: provably, since the heat terms are non-negative.  A PAF value is always
# the quotient of the last division by the cell's count c, and (q * c) / c returned such a quotient unchanged in every
# one of 10^6 samples for each c tried (an observation, not a proof), so skipping that step where a person does not cover
# the cell changed nothing on the goldens.
EQUIVALENT = [
    ("clamp_after_all_persons", "            if (acc > 1.0) acc = 1.0;\n        }\n    }\n    return acc;",
     "        }\n    }\n    return acc > 1.0 ? 1.0 : acc;"),
    ("skip_rescale_when_uncovered", "    const double c = (double)count;",
     "    if (!(fabs(nx) > 0.0 || fabs(ny) > 0.0)) return;\n    const double c = (double)count;"),
]


def goldens():
    return {os.path.basename(p)[3:-4]: dict(np.load(p)) for p in sorted(glob.glob(os.path.join(GOLDEN, "gt_*.npz")))}


def compile_core(out, header=None):
    cmd = ["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-o", out, HOST_SRC]
    if header:
        cmd.insert(1, '-DGT_CORE="%s"' % header)
    subprocess.run(cmd, check=True)
    lib = ctypes.CDLL(out)
    lib.core_exp.argtypes = [ctypes.c_double]
    lib.core_exp.restype = ctypes.c_double
    lib.core_limb_norm.argtypes = [ctypes.c_double, ctypes.c_double]
    lib.core_limb_norm.restype = ctypes.c_double
    lib.core_ground_truth.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_int] * 3 + [ctypes.c_void_p] * 3
    lib.core_ground_truth.restype = None
    return lib


def planted_header(tmpdir, name):
    src = open(CORE).read()
    old, new = next((o, n) for k, o, n in PLANTED + EQUIVALENT if k == name)
    assert src.count(old) == 1, name
    path = os.path.join(str(tmpdir), "gt_core_%s.h" % name)
    open(path, "w").write(src.replace(old, new))
    return path


def pack(kps):
    """list of [P_i, 17, 3] keypoint arrays -> (table [sum P_i, 17, 3] float32, counts int32)"""
    kps = [np.asarray(k, np.float32).reshape(-1, 17, 3) for k in kps]
    table = np.ascontiguousarray(np.concatenate(kps) if kps else np.zeros((0, 17, 3), np.float32), np.float32)
    return table, np.array([len(k) for k in kps], np.int32)


def core_gt(lib, kps, sizes, canvas=None, want64=False):
    """Host core: heat [n, 19, gh, gw], paf [n, 38, gh, gw] (and the float64 PAFs) at the canvas of the largest grid."""
    table, counts = pack(kps)
    hw = np.ascontiguousarray(np.asarray(sizes, np.int32).reshape(-1, 2))
    gh, gw = canvas or (max(h // 8 for h, _ in hw), max(w // 8 for _, w in hw))
    n = len(hw)
    heat = np.empty((n, 19, gh, gw), np.float32)
    paf = np.empty((n, 38, gh, gw), np.float32)
    paf64 = np.empty((n, 38, gh, gw), np.float64) if want64 else None
    lib.core_ground_truth(table.ctypes.data, counts.ctypes.data, hw.ctypes.data, n, gh, gw, heat.ctypes.data,
                          paf.ctypes.data, paf64.ctypes.data if want64 else None)
    return (heat, paf, paf64) if want64 else (heat, paf)


def random_person(rs, h, w):
    x = rs.uniform(-0.05 * w, 1.05 * w, 17)
    y = rs.uniform(-0.05 * h, 1.05 * h, 17)
    c = rs.randint(0, 3)
    if c == 1:       # a compact person
        cx, cy, s = rs.uniform(0, w), rs.uniform(0, h), rs.uniform(8, 80)
        x, y = cx + s * rs.uniform(-1, 1, 17), cy + s * rs.uniform(-1, 1, 17)
    elif c == 2:     # integer and tie coordinates
        x, y = 8 * rs.randint(-1, w // 8 + 1, 17) + 12.0, 8 * rs.randint(-1, h // 8 + 1, 17) + rs.choice([4.0, 12.0, 0.0], 17)
    v = rs.choice([0, 1, 2], 17, p=[0.2, 0.3, 0.5])
    return np.stack([x, y, v], 1).astype(np.float32)


def random_scenario(seed, n, sizes=((368, 368),), max_persons=8):
    """n images: (keypoints per image, (input_y, input_x) per image)"""
    rs = np.random.RandomState(seed)
    kps, hw = [], []
    for i in range(n):
        h, w = sizes[rs.randint(len(sizes))]
        people = [random_person(rs, h, w) for _ in range(rs.randint(0, max_persons + 1))]
        kps.append(np.stack(people) if people else np.zeros((0, 17, 3), np.float32))
        hw.append((h, w))
    return kps, hw


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint32 if a.dtype == np.float32 else np.uint64)
