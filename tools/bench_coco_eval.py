#!/usr/bin/env python
"""COCO keypoint evaluation on the device (DESIGN.md 2.16) at val2017 scale: tests/coco_eval_check.py's seeded
evaluation of 5 000 images, 2 700 with 11 000 person gts, 25 000 detections (scores 1.0, as run_eval writes them):
  call   : engine.coco_keypoint_eval, host clock around the call (it ends in a stream synchronise): loadRes, _prepare and
           packing on the host, upload, four kernels, copies back, the ten means
  device : b200pose_coco_kpt_eval alone on the packed arrays, host clock (validation, upload, kernels, copies)
  kernels: the four kernels' time from torch.profiler (own pass)
  oracle : oracle/coco_kpt_eval.py (float64 numpy in pycocotools' loop structure), one run on the host CPU
pycocotools itself is not timed: it is not installed where this runs.  Every call's precision and recall are checked
against the oracle's.  The card's name and power limit are read in the same call.  One JSON line.

  python tools/bench_coco_eval.py [--runs R] [--seed S]"""
import argparse
import importlib
import json
import os
import re
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _b200_alias  # noqa: E402


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--seed", type=int, default=11)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    import coco_eval_check as ce
    _b200_alias.load_package()
    eng = importlib.import_module(_b200_alias.PKG + ".engine")
    nat = importlib.import_module(_b200_alias.PKG + "._native")
    assert torch.cuda.is_available(), "bench_coco_eval needs a GPU"
    gt, rs, ids = ce.scenario(a.seed)
    t = time.perf_counter()
    ev = ce.oracle(gt, rs, ids)
    oracle_s = time.perf_counter() - t
    pk = eng.coco_pack(gt, rs, ids)
    K = len(pk["cat_ids"])
    prec, rec = np.empty((10, 101, K, 3)), np.empty((10, K, 3))
    p = lambda x: x.ctypes.data if x.size else None

    def device_call():
        nat.check(nat.lib().b200pose_coco_kpt_eval(
            0, len(pk["units"]), K, p(pk["unit_cat"]), p(pk["unit_gt0"]), p(pk["unit_dt0"]), p(pk["gt_id"]),
            p(pk["gt_kpt"]), 51, p(pk["gt_box"]), p(pk["gt_crowd"]), p(pk["gt_ignore"]), p(pk["dt_kpt"]), 51,
            p(pk["dt_score"]), p(pk["thr"]), prec.ctypes.data, rec.ctypes.data, None, 0, None), "coco_kpt_eval")

    for _ in range(3):                                   # warm-up: module load, first allocations
        got = eng.coco_keypoint_eval(gt, rs, ids)
        device_call()
    calls, devs = [], []
    for _ in range(a.runs):
        t = time.perf_counter()
        got = eng.coco_keypoint_eval(gt, rs, ids)
        calls.append(time.perf_counter() - t)
        assert np.array_equal(got.precision, ev.precision) and np.array_equal(got.recall, ev.recall)
        t = time.perf_counter()
        device_call()
        devs.append(time.perf_counter() - t)
        assert np.array_equal(prec[..., None], ev.precision)
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        for _ in range(a.runs):
            device_call()
    kern = {}
    for e in prof.key_averages():
        name = re.search(r"coco_\w+_kernel", e.key)
        if name:
            us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
            kern[name.group(0)] = kern.get(name.group(0), 0.0) + us / a.runs / 1e3
    print(json.dumps({
        "bench": "coco_kpt_eval", "card": card(), "images": len(gt["images"]), "img_ids": len(ids),
        "gts": len(gt["annotations"]), "detections": len(rs), "runs": a.runs,
        "call_ms_median": 1e3 * float(np.median(calls)), "call_ms_min": 1e3 * float(np.min(calls)),
        "device_call_ms_median": 1e3 * float(np.median(devs)), "kernels_ms": kern,
        "kernels_ms_total": float(sum(kern.values())), "oracle_s": oracle_s, "stats": got.stats.tolist(),
        "pycocotools": "not timed (not installed)"}))


if __name__ == "__main__":
    main()
