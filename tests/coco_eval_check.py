"""Shared by tests/test_coco_eval_host.py and tests/test_gpu_coco_eval.py: the host build of csrc/coco_eval_core.h
(tests/cuda/coco_eval_core_host.cpp), COCO keypoint datasets built by hand and at val2017 scale from a seed, and the
margin check that keeps exp's last bit out of the comparison."""
import ctypes
import os
import subprocess

import numpy as np

from conftest import ROOT, pkg_module

HOST_SRC = os.path.join(ROOT, "tests", "cuda", "coco_eval_core_host.cpp")
CSRC = os.path.join(ROOT, "pytorch_realtime_multi-person_pose_estimation_b200", "csrc")
MARGIN = 1e-12


def compile_core(so, core=None):
    """The host evaluation core as a ctypes library; `core` replaces coco_eval_core.h (a copy with a planted mistake)."""
    cmd = ["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-I", CSRC, "-o", so, HOST_SRC]
    if core:
        cmd.insert(1, '-DCOCO_EVAL_CORE="%s"' % core)
    subprocess.run(cmd, check=True)
    lib = ctypes.CDLL(so)
    vp = ctypes.c_void_p
    lib.core_oks.argtypes = [vp, vp, vp]
    lib.core_oks.restype = ctypes.c_double
    lib.core_dt_area.argtypes = [vp]
    lib.core_dt_area.restype = ctypes.c_double
    lib.core_sum.argtypes = [vp, ctypes.c_int]
    lib.core_sum.restype = ctypes.c_double
    lib.core_eval.argtypes = [ctypes.c_int] * 2 + [vp] * 14
    lib.core_eval.restype = ctypes.c_int
    return lib


def core_eval(lib, gt, results, img_ids):
    """The host core on engine.coco_pack's arrays: (precision [10,101,K,3,1], recall [10,K,3,1], OKS blocks)."""
    eng = pkg_module("engine")
    pk = eng.coco_pack(gt, results, img_ids)
    K = len(pk["cat_ids"])
    prec, rec = np.empty((10, 101, K, 3)), np.empty((10, K, 3))
    n_oks = sum(min(nd, 20) * ng for _, _, ng, nd in pk["units"])
    oks = np.empty(max(n_oks, 1))
    p = lambda a: a.ctypes.data if a.size else None
    lib.core_eval(len(pk["units"]), K, p(pk["unit_cat"]), p(pk["unit_gt0"]), p(pk["unit_dt0"]), p(pk["gt_kpt"]),
                  p(pk["gt_box"]), p(pk["gt_crowd"]), p(pk["gt_ignore"]), p(pk["dt_kpt"]), p(pk["dt_score"]),
                  p(pk["thr"]), prec.ctypes.data, rec.ctypes.data, oks.ctypes.data, None)
    return prec[..., None], rec[..., None], eng.coco_oks_blocks(pk, oks)


def oracle(gt, results, img_ids):
    from oracle import coco_kpt_eval
    return coco_kpt_eval.Eval(gt, results, img_ids)


def ulps(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a.view(np.int64) - b.view(np.int64)).max() if a.size else 0


def assert_margins(ev):
    """No oracle OKS within MARGIN of a threshold (min(t, 1 - 1e-10)) or of another OKS of the same detection, other
    than exactly equal: then the evaluation decides every comparison the same way however exp rounds its last bit."""
    from oracle import coco_kpt_eval
    thr = np.minimum(coco_kpt_eval.IOU_THRS, 1 - 1e-10)
    for key, m in ev.ious.items():
        if len(m) == 0:
            continue
        near = np.abs(m[..., None] - thr).min()
        assert near >= MARGIN, (key, near)
        for row in m:
            row = row[row >= thr[0] - MARGIN]      # below every threshold no OKS competes
            d = np.abs(row[:, None] - row[None, :])
            d = d[d > 0]
            assert not d.size or d.min() >= MARGIN, (key, d.min())


# ---------------------------------------------------------------------------------------------------- datasets
def gt_file(images, anns, cats=(1,)):
    return {"images": [{"id": i, "file_name": "%012d.jpg" % i, "height": 480, "width": 640} for i in images],
            "annotations": anns, "categories": [{"id": c, "name": "person" if c == 1 else "c%d" % c} for c in cats]}


def ann(aid, image_id, kpt, bbox, area, iscrowd=0, num_keypoints=None, cat=1):
    kpt = [float(v) for v in np.asarray(kpt, np.float64).reshape(51)]
    n = int(np.count_nonzero(np.asarray(kpt[2::3]) > 0)) if num_keypoints is None else num_keypoints
    return {"id": aid, "image_id": image_id, "category_id": cat, "keypoints": kpt, "bbox": [float(v) for v in bbox],
            "area": float(area), "iscrowd": iscrowd, "num_keypoints": n}


def res(image_id, kpt, score=1.0, cat=1):
    return {"image_id": image_id, "category_id": cat, "keypoints": [float(v) for v in np.asarray(kpt).reshape(51)],
            "score": float(score)}


def skeleton(cx, cy, s, v=2):
    """17 keypoints of a standing person of height ~4s around (cx, cy), visibility v."""
    off = np.array([[0, -2], [-.2, -2.1], [.2, -2.1], [-.4, -2], [.4, -2], [-.6, -1.4], [.6, -1.4], [-.8, -.8],
                    [.8, -.8], [-.9, -.2], [.9, -.2], [-.4, 0], [.4, 0], [-.4, 1], [.4, 1], [-.4, 2], [.4, 2]])
    k = np.zeros((17, 3))
    k[:, 0], k[:, 1], k[:, 2] = cx + s * off[:, 0], cy + s * off[:, 1], v
    return k


def with_xy(k, dx=0.0, dy=0.0):
    k = np.array(k, np.float64)
    k[:, 0] += dx
    k[:, 1] += dy
    return k


def _box(k, s):
    return [k[:, 0].min() - s / 4, k[:, 1].min() - s / 4, np.ptp(k[:, 0]) + s / 2, np.ptp(k[:, 1]) + s / 2]


def hand_cases():
    """name -> (gt file, results, img_ids)."""
    cases = {}
    g1, g2, g3 = skeleton(200, 200, 40), skeleton(400, 300, 15), skeleton(150, 300, 30)
    # perfect detections, gts in the medium and the large range
    gts = [ann(1, 1, g1, _box(g1, 40), 20000), ann(2, 1, g2, _box(g2, 15), 3000), ann(3, 2, g3, _box(g3, 30), 9000)]
    cases["perfect"] = (gt_file([1, 2, 3], gts), [res(a["image_id"], a["keypoints"]) for a in gts], [1, 2, 3])
    # one detection at a known OKS (shifted by 6 px in x)
    gts = [ann(1, 1, g1, _box(g1, 40), 20000)]
    cases["known_oks"] = (gt_file([1], gts), [res(1, with_xy(g1, 6.0))], [1])
    # a crowd gt absorbs several detections; a normal gt gets a perfect one
    crowd = ann(2, 1, g2, _box(g2, 15), 3000, iscrowd=1)
    cases["crowd"] = (gt_file([1], [ann(1, 1, g1, _box(g1, 40), 20000), crowd]),
                      [res(1, g1, .5)] + [res(1, with_xy(g2, d), .9) for d in (0.0, .02, .04)], [1])
    # num_keypoints == 0: OKS from the distance outside the enlarged box (one detection inside it, one outside)
    g0 = skeleton(300, 200, 20, v=0)
    z = ann(2, 1, g0, [280, 150, 40, 100], 2500)
    cases["no_keypoints"] = (gt_file([1], [ann(1, 1, g1, _box(g1, 40), 20000), z]),
                             [res(1, g1, .3), res(1, with_xy(g0, 5.0), .9), res(1, with_xy(g0, 90.0, 40.0), .8)], [1])
    # gt areas exactly 32^2 and 96^2: in both neighbouring ranges
    gts = [ann(1, 1, g2, _box(g2, 15), 32 ** 2), ann(2, 2, g3, _box(g3, 30), 96 ** 2)]
    cases["area_bounds"] = (gt_file([1, 2], gts), [res(1, g2, .7), res(2, g3, .6)], [1, 2])
    # 25 detections in one image: the 5 perfect ones score lowest and fall off the cut to 20
    gts = [ann(i + 1, 1, skeleton(60 + 120 * i, 200, 25), _box(skeleton(60 + 120 * i, 200, 25), 25), 12000) for i in range(5)]
    rs = [res(1, a["keypoints"], .1) for a in gts] + [res(1, with_xy(skeleton(60 + 25 * i, 420, 10), 0), .5 + i / 100)
                                                      for i in range(20)]
    cases["truncation"] = (gt_file([1], gts), rs, [1])
    # no non-ignored gt in the medium range
    cases["empty_range"] = (gt_file([1], [ann(1, 1, g1, _box(g1, 40), 20000)]), [res(1, g1)], [1])
    # detection A is equally close to gts 1 and 2 and takes the later one; B then matches gt 1
    base = skeleton(300, 250, 30)
    ga, gb = with_xy(base, 8.0), with_xy(base, -8.0)
    gts = [ann(1, 1, ga, _box(ga, 30), 10000), ann(2, 1, gb, _box(gb, 30), 10000)]
    cases["tie_last"] = (gt_file([1], gts), [res(1, base, .9), res(1, ga, .8)], [1])
    # every score 1.0: images in ascending id, each image's detections in list order
    gts = [ann(1, 3, g1, _box(g1, 40), 20000), ann(2, 5, g3, _box(g3, 30), 9000), ann(3, 5, g2, _box(g2, 15), 3000)]
    cases["equal_scores"] = (gt_file([3, 5], gts), [res(5, g3), res(5, with_xy(g2, 200.0)), res(5, g2), res(3, with_xy(g1, 300.0)),
                                                    res(3, g1)], [5, 3])
    # an unmatched detection whose undetected (0, 0) parts make its box large: ignored in the medium range
    far = skeleton(500, 400, 8)
    far[3:6] = 0
    cases["zero_parts"] = (gt_file([1], [ann(1, 1, g2, _box(g2, 15), 3000)]), [res(1, g2, .5), res(1, far, .9)], [1])
    # a result for an image of the gt file outside img_ids is left out
    cases["outside_img_ids"] = (gt_file([1, 2], [ann(1, 1, g1, _box(g1, 40), 20000), ann(2, 2, g3, _box(g3, 30), 9000)]),
                                [res(1, g1), res(2, with_xy(g3, 100.0))], [1])
    return cases


def scenario(seed, n_images=5000, n_person=2700, n_gts=11000, n_dets=25000, scores="const", cats=(1,)):
    """A val2017-sized evaluation from a seed: person images with 1 .. 30 gts (crowd and num_keypoints == 0 among
    them), detections near the gts plus false ones, a few images with hundreds of detections.  scores: 'const' (1.0,
    as run_eval writes them) or 'ties' (random, rounded to 2 decimals)."""
    rs = np.random.RandomState(seed)
    images = list(rs.permutation(np.arange(1, 3 * n_images, 3))[:n_images])
    person = images[:n_person]
    per = rs.multinomial(n_gts - n_person, np.ones(n_person) / n_person) + 1
    anns, results, aid = [], [], 1
    for n, img in enumerate(person):
        cat = cats[n % len(cats)]
        for _ in range(per[n]):
            s = rs.uniform(4, 60)
            k = skeleton(rs.uniform(0, 640), rs.uniform(0, 480), s)
            k[:, :2] += rs.normal(0, s / 10, (17, 2))
            k[:, 2] = rs.choice([0, 1, 2], 17, p=[.3, .2, .5])
            kind = rs.rand()
            if kind < .04:
                k[:, 2] = 0
            area = float(s * s * rs.uniform(1.5, 5))
            anns.append(ann(aid, int(img), k, _box(k, s), area, iscrowd=int(kind > .98), cat=cat))
            aid += 1
            for _ in range(rs.poisson(1.6)):
                d = k.copy()
                d[:, :2] += rs.normal(0, s * rs.uniform(.02, .3), (17, 2))
                d[:, 2] = 1
                d[rs.rand(17) < .15, :2] = 0
                results.append(res(int(img), d, cat=cat))
    for img in person[:12]:                         # crowded images: hundreds of detections
        for _ in range(rs.randint(100, 400)):
            d = skeleton(rs.uniform(0, 640), rs.uniform(0, 480), rs.uniform(4, 60))
            d[:, 2] = 1
            results.append(res(int(img), d, cat=cats[0]))
    while len(results) < n_dets:                    # false detections spread over the person images
        img = person[rs.randint(len(person))]
        d = skeleton(rs.uniform(0, 640), rs.uniform(0, 480), rs.uniform(4, 60))
        d[:, 2] = 1
        results.append(res(int(img), d, cat=cats[rs.randint(len(cats))]))
    order = rs.permutation(len(results))
    results = [results[i] for i in order]
    if scores == "ties":
        for r in results:
            r["score"] = float(np.round(rs.uniform(0, 1), 2))
    return gt_file([int(i) for i in images], anns, cats), results, [int(i) for i in person]
