"""numpy restatement of CocoKeypoints.get_ground_truth (lib/datasets/datasets.py) + transpose((2, 0, 1)).astype(float32),
pinned to the reference's own outputs in tests/golden/gt_*.npz (tests/test_gt_host.py).  It gives the GPU tests
expectations on scenarios the reference never saw, without the reference.  The limb length is
sqrt(fma(dy, dy, dx * dx)) computed exactly in rationals (what np.linalg.norm gives with OpenBLAS's ddot), so the
port does not depend on the BLAS of the machine it runs on; only np.exp is the platform's."""
from fractions import Fraction

import numpy as np

STRIDE, SIGMA, PARTS = 8, 7.0, 18
OUR_ORDER = [0, 17, 6, 8, 10, 5, 7, 9, 12, 14, 16, 11, 13, 15, 2, 1, 4, 3]
LIMBS = [(1, 8), (8, 9), (9, 10), (1, 11), (11, 12), (12, 13), (1, 2), (2, 3), (3, 4), (2, 14), (1, 5), (5, 6), (6, 7),
         (5, 15), (1, 0), (0, 14), (0, 15), (14, 16), (15, 17)]


def fma(a, b, c):
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def limb_norm(dx, dy):
    return float(np.sqrt(fma(dy, dy, dx * dx)))


def joints(kp, input_x, input_y):
    """add_neck, the 18-part order and remove_illegal_joint of one person: [17, 3] float32 -> [18, 3] float32"""
    kp = np.asarray(kp, np.float32)
    rs, ls = kp[6], kp[5]
    neck = (rs + ls) / np.float32(2)
    neck[2] = 2 if (rs[2] == 2 and ls[2] == 2) else rs[2] * ls[2]
    j = np.vstack([kp, np.rint(neck)[None]])[OUR_ORDER].astype(np.float32)
    bad = (j[:, 0] >= input_x) | (j[:, 0] < 0) | (j[:, 1] >= input_y) | (j[:, 1] < 0)
    j[bad] = (-1, -1, 0)
    return j


def ground_truth(kp, size, exp=np.exp, float64=False):
    """kp [P, 17, 3], size (input_y, input_x) -> heat [19, gh, gw], paf [38, gh, gw] float32 (float64=True: before
    the cast).  P = 0 gives zero maps and a background of 1."""
    iy, ix = int(size[0]), int(size[1])
    gh, gw = int(iy / STRIDE), int(ix / STRIDE)
    js = [joints(k, ix, iy) for k in np.asarray(kp, np.float32).reshape(-1, 17, 3)]
    heat = np.zeros((PARTS + 1, gh, gw))
    start = STRIDE / 2.0 - 0.5
    xs = (np.arange(gw) * STRIDE + start)[None, :]
    ys = (np.arange(gh) * STRIDE + start)[:, None]
    for p in range(PARTS):
        for j in js:
            if j[p, 2] > 0.5:
                ex = ((xs - np.float64(j[p, 0])) ** 2 + (ys - np.float64(j[p, 1])) ** 2) / 2.0 / SIGMA / SIGMA
                heat[p] = np.minimum(heat[p] + np.where(ex <= 4.6052, exp(-ex), 0.0), 1.0)
    heat[PARTS] = np.maximum(1 - heat[:PARTS].max(0), 0.0)
    paf = np.zeros((2 * len(LIMBS), gh, gw))
    gx = np.arange(gw, dtype=np.float64)[None, :]
    gy = np.arange(gh, dtype=np.float64)[:, None]
    for l, (a, b) in enumerate(LIMBS):
        acc = paf[2 * l:2 * l + 2]
        count = np.zeros((gh, gw))
        for j in js:
            if not (j[a, 2] > 0.5 and j[b, 2] > 0.5):
                continue
            A = j[a, :2].astype(np.float64) / STRIDE
            B = j[b, :2].astype(np.float64) / STRIDE
            d = B - A
            norm = limb_norm(d[0], d[1])
            if norm == 0.0:
                continue
            u = d / norm
            x0, x1 = max(int(round(min(A[0], B[0]) - 1)), 0), min(int(round(max(A[0], B[0]) + 1)), gw)
            y0, y1 = max(int(round(min(A[1], B[1]) - 1)), 0), min(int(round(max(A[1], B[1]) + 1)), gh)
            inbox = (gx >= x0) & (gx < x1) & (gy >= y0) & (gy < y1)
            width = np.abs((gx - A[0]) * u[1] - (gy - A[1]) * u[0])
            m = (width < 1).astype(np.float64)
            vec = np.where(inbox[None], m[None] * u[:, None, None], acc * 0.0)
            acc = acc * count + vec
            count = count + ((np.abs(vec[0]) > 0) | (np.abs(vec[1]) > 0))
            acc = acc / np.maximum(count, 1)
        paf[2 * l:2 * l + 2] = acc
    if float64:
        return heat, paf
    return heat.astype(np.float32), paf.astype(np.float32)


def ground_truth_batch(kps, sizes, canvas=None):
    """engine.ground_truth's layout: [n, 19, gh, gw] / [n, 38, gh, gw] at the largest grid, +0 outside each image's."""
    gh, gw = canvas or (max(int(h) // STRIDE for h, _ in sizes), max(int(w) // STRIDE for _, w in sizes))
    heat = np.zeros((len(sizes), PARTS + 1, gh, gw), np.float32)
    paf = np.zeros((len(sizes), 2 * len(LIMBS), gh, gw), np.float32)
    for i, (k, s) in enumerate(zip(kps, sizes)):
        h, p = ground_truth(k, s)
        heat[i, :, :h.shape[1], :h.shape[2]] = h
        paf[i, :, :p.shape[1], :p.shape[2]] = p
    return heat, paf
