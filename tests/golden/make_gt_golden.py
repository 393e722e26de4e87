"""Generates the training-target fixtures tests/golden/gt_*.npz by running the UNMODIFIED reference method
CocoKeypoints.get_ground_truth (lib/datasets/datasets.py) on hand-made annotations.  Usage:

    python tests/golden/make_gt_golden.py <reference checkout>

Shims needed to import the reference (none of them touches its arithmetic): stub modules for matplotlib and
matplotlib.pyplot, which lib/datasets/heatmap.py and paf.py import at load time, and, where scipy is not installed, for
scipy, scipy.misc and scipy.ndimage, which they import without using.  get_ground_truth runs on an object
made with CocoKeypoints.__new__ carrying the attributes it reads (HEATMAP_COUNT, LIMB_IDS, input_y, input_x, stride); no
COCO file or pycocotools is needed.

Each fixture holds `kp` (persons x 17 x 3 float32, as transforms.Normalize leaves them), `size` (input_y, input_x),
`heat` [19, gh, gw] and `paf` [38, gh, gw] (get_ground_truth's maps, transpose((2, 0, 1)).astype(float32)), `paf64`
(the PAFs before that cast: float64, which no exp touches, so that steps the cast hides are still pinned), and
`norm_d` / `norm`: every visible limb's B - A in grid units and np.linalg.norm of it, so that the tests pin the norm's
formula to these recorded numbers rather than to the BLAS of the machine that runs them.
"""
import os
import sys
import types

import numpy as np

OUT = os.path.dirname(os.path.abspath(__file__))


def import_reference(ref):
    mpl = types.ModuleType("matplotlib")
    plt = types.ModuleType("matplotlib.pyplot")
    mpl.pyplot = plt
    sys.modules.setdefault("matplotlib", mpl)
    sys.modules.setdefault("matplotlib.pyplot", plt)
    try:
        import scipy.misc  # noqa: F401
        import scipy.ndimage  # noqa: F401
    except ImportError:
        sp = types.ModuleType("scipy")
        for sub in ("misc", "ndimage"):
            m = types.ModuleType("scipy." + sub)
            setattr(sp, sub, m)
            sys.modules["scipy." + sub] = m
        sys.modules["scipy"] = sp
    sys.path.insert(0, ref)
    from lib.datasets import datasets
    return datasets


def ground_truth(ds, kp, size):
    obj = ds.CocoKeypoints.__new__(ds.CocoKeypoints)
    obj.HEATMAP_COUNT = 18
    obj.LIMB_IDS = ds.kp_connections(ds.get_keypoints())
    obj.input_y, obj.input_x = int(size[0]), int(size[1])
    obj.stride = 8
    anns = [{"keypoints": k.copy()} for k in kp]
    heat, paf = obj.get_ground_truth(anns)
    return heat.transpose((2, 0, 1)), paf.transpose((2, 0, 1)), obj


def limb_norms(ds, obj, kp):
    """B - A in grid units of every limb putVecMaps draws, and np.linalg.norm of it."""
    d, nrm = [], []
    for single in kp:
        j = obj.remove_illegal_joint(obj.add_neck(single.copy())[None])[0]
        for a, b in obj.LIMB_IDS:
            if j[a, 2] > 0.5 and j[b, 2] > 0.5:
                v = j[b, :2].astype(float) / 8 - j[a, :2].astype(float) / 8
                d.append(v)
                nrm.append(np.linalg.norm(v))
    return np.array(d, np.float64).reshape(-1, 2), np.array(nrm, np.float64)


def person(rs, h, w, vis=None, frac=True):
    """17 COCO keypoints spread over an h x w image: x, y float32 with fractional parts, v in {0, 1, 2}."""
    cx, cy = rs.uniform(0.15 * w, 0.85 * w), rs.uniform(0.15 * h, 0.85 * h)
    s = rs.uniform(0.05, 0.3) * min(h, w)
    x = cx + s * rs.uniform(-1, 1, 17)
    y = cy + s * rs.uniform(-1.2, 1.2, 17)
    if not frac:
        x, y = np.round(x), np.round(y)
    v = rs.choice([0, 1, 2], 17, p=[0.15, 0.25, 0.6]) if vis is None else vis
    return np.stack([x, y, v], 1).astype(np.float32)


def scenarios():
    rs = np.random.RandomState(2026)
    sc = {}
    for n in (1, 5, 30):
        sc["p%d" % n] = (np.stack([person(rs, 368, 368) for _ in range(n)]), (368, 368))
    # a crowd: limbs crossing near the centre, so 2 to 4 of them cover some cells
    crowd = []
    for i in range(6):
        k = np.zeros((17, 3), np.float32)
        ang = np.pi * i / 6
        for p in range(17):
            t = (p - 8) * 10.0
            k[p] = (184 + t * np.cos(ang) + rs.uniform(-3, 3), 184 + t * np.sin(ang) + rs.uniform(-3, 3), 2)
        crowd.append(k)
    sc["crowd"] = (np.stack(crowd), (368, 368))
    # joints on and beyond every border (x == input_x and y == input_y are illegal; 367.5 and 0 are not)
    edge = [0.0, -0.25, 367.5, 368.0, 369.0, -8.0, 367.99, 0.5]
    border = []
    for i in range(len(edge)):
        k = person(rs, 368, 368, vis=np.full(17, 2))
        k[rs.choice(17, 4, replace=False), 0] = edge[i]
        k[rs.choice(17, 4, replace=False), 1] = edge[(i + 3) % len(edge)]
        border.append(k)
    sc["borders"] = (np.stack(border), (368, 368))
    # zero-length limbs: both joints of several limbs on one point
    z = person(rs, 368, 368, vis=np.full(17, 2))
    z[12] = z[11]                      # hips: neck-hip limbs differ, hip-knee etc. as drawn
    z[13] = z[11]                      # left hip -> knee zero length
    z[8] = z[6]                        # right shoulder -> elbow zero length
    z[1] = z[0]                        # nose -> left eye
    sc["zero_length"] = (np.stack([z, person(rs, 368, 368)]), (368, 368))
    # ties for round(): coordinates 8k + 12 put min - 1 and max + 1 at k + 0.5 and k + 2.5 in grid units
    ties = []
    for i in range(4):
        k = person(rs, 368, 368, vis=np.full(17, 2))
        k[:, :2] = (8 * rs.randint(2, 40, (17, 2)) + 12).astype(np.float32)
        ties.append(k)
    sc["round_ties"] = (np.stack(ties), (368, 368))
    # vertical and horizontal limbs: one unit component is 0
    ax = []
    for i in range(3):
        k = person(rs, 368, 368, vis=np.full(17, 2))
        k[[6, 8, 10], 0] = k[6, 0]     # right arm vertical
        k[[5, 7, 9], 1] = k[5, 1]      # left arm horizontal
        k[[12, 14, 16], 0] = k[12, 0] + np.float32(0.5)
        k[[11, 13, 15], 1] = k[11, 1]
        ax.append(k)
    sc["axis_limbs"] = (np.stack(ax), (368, 368))
    # all nine (r_shoulder, l_shoulder) visibility pairs
    nv = []
    for a in range(3):
        for b in range(3):
            k = person(rs, 368, 368, vis=np.full(17, 2))
            k[6, 2], k[5, 2] = a, b
            nv.append(k)
    sc["neck_visibility"] = (np.stack(nv), (368, 368))
    sc["size_656x368"] = (np.stack([person(rs, 656, 368) for _ in range(4)]), (656, 368))
    sc["size_64x128"] = (np.stack([person(rs, 64, 128) for _ in range(3)]), (64, 128))
    # integer coordinates (the neck's rounding then lands on .5 ties of the shoulders' mean)
    sc["integer_coords"] = (np.stack([person(rs, 368, 368, frac=False) for _ in range(5)]), (368, 368))
    # three nearly identical persons, then six elsewhere: heat sums above 1 are clamped, and cells covered three times
    # keep being multiplied and divided by 3 while the later persons' limbs pass elsewhere (only the float64 PAFs show it)
    same = person(rs, 368, 368, vis=np.full(17, 2))
    same[:, :2] = np.clip(same[:, :2], 20, 180)
    near = [same + np.concatenate([rs.uniform(-5, 5, (17, 2)), np.zeros((17, 1))], 1).astype(np.float32) for _ in range(3)]
    others = [person(rs, 368, 368, vis=np.full(17, 2)) for _ in range(6)]
    for k in others:
        k[:, :2] = np.clip(k[:, :2], 200, 360)
    sc["overlap"] = (np.stack(near + others), (368, 368))
    # limbs with a cell whose width |ba_x u_y - ba_y u_x| is 1 with two roundings and below 1 if fused into an fma
    width = []
    for a, b in [((216, 228), (156, 183)), ((288, 292), (48, 192)), ((115, 164), (73, 108)), ((260, 137), (152, 182))]:
        k = np.zeros((17, 3), np.float32)
        k[6] = (a[0], a[1], 2)         # right shoulder -> right elbow
        k[8] = (b[0], b[1], 2)
        width.append(k)
    sc["width_edges"] = (np.stack(width), (368, 368))
    return sc


def main():
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    ds = import_reference(sys.argv[1])
    for name, (kp, size) in scenarios().items():
        heat, paf, obj = ground_truth(ds, kp, size)
        d, nrm = limb_norms(ds, obj, kp)
        np.savez_compressed(os.path.join(OUT, "gt_%s.npz" % name), kp=kp, size=np.array(size, np.int32),
                            heat=heat.astype(np.float32), paf=paf.astype(np.float32), paf64=paf, norm_d=d, norm=nrm)
        print("gt_%s: %d persons, %s, heat %s, %d limbs" % (name, len(kp), size, heat.shape, len(nrm)))


if __name__ == "__main__":
    main()
