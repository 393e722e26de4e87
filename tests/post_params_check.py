"""Shared by tests/test_post_params_host.py and tests/test_gpu_post_params.py: the scenarios the post-processing
settings are checked on, and person rows of the pafprocess oracles in the product's [k, 73] layout."""
import numpy as np

from conftest import POST_CASES
from oracle import nms_port, synth

STICK_CASES = ("p1", "p3", "p8", "p30", "noise0")
FUZZ_SEEDS = range(1000, 1300)


def stick_case(name):
    """(heat, paf) low-resolution HWC maps of one of conftest.POST_CASES."""
    return POST_CASES[name](synth)


def joint_list(heat, thresh=0.1):
    return nms_port.joint_list_from_nms(nms_port.nms(heat, thresh, 18))


def fuzz_case(seed):
    """(joint list, paf, h, w) of the fuzz scenario tests/test_host.py draws from `seed`."""
    rs = np.random.RandomState(seed)
    t = seed - 1000
    h, w = int(rs.choice([12, 23, 46])), int(rs.choice([23, 46, 53]))
    if t % 2:
        h = max(h, 23)
        jl, paf = synth.fuzz_persons(rs, h, w)
    else:
        jl, paf = synth.fuzz_field(rs, h, w, ("uniform", "cluster", "ties")[(t // 2) % 3])
    return np.ascontiguousarray(jl, np.float32), np.ascontiguousarray(paf, np.float32), h, w


def scenarios():
    """name -> (joint list, paf, h, w): the stick figures with 1/3/8/30 persons, the noise maps, 300 fuzz scenarios."""
    out = {}
    for name in STICK_CASES:
        heat, paf = stick_case(name)
        out[name] = (joint_list(heat), np.ascontiguousarray(paf), heat.shape[0], heat.shape[1])
    for s in FUZZ_SEEDS:
        jl, paf, h, w = fuzz_case(s)
        if len(jl):
            out["fuzz%d" % s] = (jl, paf, h, w)
    return out


def oracle_rows(pafprocess, jl, paf, h, w):
    """pafprocess.process_paf on the x8 nearest-upsampled maps (paf_to_pose.py:382-385), its persons as float32 rows
    [k, 73]: score, 18 x (x, y, peak score, cid | -1), the layout of b200pose_post_get_humans."""
    paf_up = np.ascontiguousarray(np.repeat(np.repeat(paf, 8, axis=0), 8, axis=1))
    heat_up = np.zeros((h * 8, 1, 19), np.float32)       # only its height is read (h1, pafprocess.cpp:83)
    pafprocess.process_paf(np.ascontiguousarray(jl[None]), heat_up, paf_up)
    rows = []
    for k in range(pafprocess.get_num_humans()):
        r = [pafprocess.get_score(k)]
        for p in range(18):
            c = int(pafprocess.get_part_cid(k, p))
            r += [0.0, 0.0, 0.0, -1.0] if c < 0 else [pafprocess.get_part_x(c), pafprocess.get_part_y(c),
                                                      pafprocess.get_part_score(c), c]
        rows.append(r)
    return np.array(rows, np.float32).reshape(-1, 73)


def same_bits(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))
