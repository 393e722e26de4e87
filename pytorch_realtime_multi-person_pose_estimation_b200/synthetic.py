"""Seeded synthetic weights / inputs for benchmarks and smoke runs (no checkpoints exist offline):
He-normal weights N(0, 2/fan_in), biases U(-0.1, 0.1), in the reference state_dict order.  The reference's own
init (std=0.01, rtpose_vgg.py:200-206) would make every output ~1e-10 and any accuracy statement vacuous."""
import numpy as np
import torch

from .distributed import tensor_shapes


def he_state_arrays(seed=1234):
    g = torch.Generator().manual_seed(seed)
    out = []
    for shape in tensor_shapes():
        if len(shape) == 4:
            fan_in = shape[1] * shape[2] * shape[3]
            out.append((torch.randn(shape, generator=g) * float(np.sqrt(2.0 / fan_in))).numpy())
        else:
            out.append((torch.rand(shape, generator=g) * 0.2 - 0.1).numpy())
    return out


def openpose_state_dict(l2_stages=4, l1_stages=2, seed=2024):
    """Seeded weights for OpenPose_Model(l2_stages, l1_stages, 38, 19), an OrderedDict in its state_dict order (keys:
    engine.openpose_state_dict_keys, shapes: the library's table).  PReLU slopes ~ U(-0.5, 1.5) - negative and steeper
    than 1, so that a PReLU mistake shows - biases U(-0.1, 0.1), weights N(0, g / fan_in) with the gain that keeps the
    activations' variance through the conv's activation: 2 for ReLU and for none, 2 / (1 + 7/12) for PReLU (He's rule;
    7/12 is the slopes' mean square), so that 90 layers neither explode nor vanish."""
    from collections import OrderedDict
    from . import _native as nat
    from .engine import openpose_state_dict_keys
    keys = openpose_state_dict_keys(l2_stages, l1_stages)
    shapes = nat.openpose_shapes(l2_stages, l1_stages)
    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict()
    for i, (key, shape) in enumerate(zip(keys, shapes)):
        if len(shape) == 4:
            # a conv's tensors are weight, bias and, with a PReLU after it, the slope
            prelu = i + 2 < len(keys) and len(shapes[i + 2]) == 1 and not keys[i + 2].endswith("bias")
            gain = 2.0 / (1.0 + 7.0 / 12.0) if prelu else 2.0
            sd[key] = torch.randn(shape, generator=g) * float(np.sqrt(gain / (shape[1] * shape[2] * shape[3])))
        elif key.endswith("bias"):
            sd[key] = torch.rand(shape, generator=g) * 0.2 - 0.1
        else:
            sd[key] = torch.rand(shape, generator=g) * 2.0 - 0.5
    return sd


# 18 COCO parts of a schematic standing person in a unit box, and the 19 limbs / their PAF channel pairs in the order of
# pafprocess.h:16-24 (the layout SURVEY.md appendix B pins).
_BODY = ((.50, .08), (.50, .22), (.36, .22), (.30, .40), (.27, .56), (.64, .22), (.70, .40), (.73, .56), (.42, .55),
         (.41, .75), (.40, .95), (.58, .55), (.59, .75), (.60, .95), (.46, .05), (.54, .05), (.41, .07), (.59, .07))
_LIMBS = ((1, 2), (1, 5), (2, 3), (3, 4), (5, 6), (6, 7), (1, 8), (8, 9), (9, 10), (1, 11), (11, 12), (12, 13), (1, 0),
          (0, 14), (14, 16), (0, 15), (15, 17), (2, 16), (5, 17))
_PAF_CH = ((12, 13), (20, 21), (14, 15), (16, 17), (22, 23), (24, 25), (0, 1), (2, 3), (4, 5), (6, 7), (8, 9), (10, 11),
           (28, 29), (30, 31), (34, 35), (32, 33), (36, 37), (18, 19), (26, 27))


def person_maps(n, persons, seed=7, h=46, w=46, stride=8):
    """Person-like network outputs for the benchmark's alternative workload: `n` images with `persons` schematic people
    each, as fp32 NCHW heat [n,19,h,w] / PAF [n,38,h,w] maps (Gaussian joint blobs, unit vectors along the limbs).
    A trained model emits maps of this kind (tens of peaks per frame); the random-weight network the benchmark has to
    use emits noise with ~4000 peaks per frame, which makes the post-processing cost unrepresentative."""
    rs = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w]
    px = xx * stride + (stride - 1) / 2.0
    py = yy * stride + (stride - 1) / 2.0
    heat = np.zeros((n, 19, h, w), np.float32)
    paf = np.zeros((n, 38, h, w), np.float32)
    body = np.asarray(_BODY)
    for i in range(n):
        hits = np.zeros((19, h, w), np.float32)
        for _ in range(persons):
            size = rs.uniform(0.3, 0.6) * min(h, w) * stride
            org = np.array([rs.uniform(0, w * stride - 0.5 * size), rs.uniform(0, h * stride - size)])
            pts = org + body * size + rs.normal(0, 0.01 * size, body.shape)
            for j, (x, y) in enumerate(pts):
                blob = np.exp(-((px - x) ** 2 + (py - y) ** 2) / 98.0) * rs.uniform(0.8, 1.0)
                heat[i, j] = np.maximum(heat[i, j], blob)
            for l, (a, b) in enumerate(_LIMBS):
                d = pts[b] - pts[a]
                length = float(np.hypot(*d))
                if length < 1e-3:
                    continue
                u = d / length
                rx, ry = px - pts[a][0], py - pts[a][1]
                t = rx * u[0] + ry * u[1]
                on = (t >= 0) & (t <= length) & (np.abs(rx * u[1] - ry * u[0]) <= 6.0)
                paf[i, _PAF_CH[l][0]][on] += u[0]
                paf[i, _PAF_CH[l][1]][on] += u[1]
                hits[l][on] += 1
        for l in range(19):
            m = hits[l] > 1
            for ch in _PAF_CH[l]:
                paf[i, ch][m] /= hits[l][m]
        heat[i, 18] = 1.0 - heat[i, :18].max(axis=0)
    heat += rs.normal(0, 0.004, heat.shape).astype(np.float32)
    paf += rs.normal(0, 0.004, paf.shape).astype(np.float32)
    return heat, paf
