#!/usr/bin/env python
"""COCO training targets and validation loss on the device (DESIGN.md 2.19):
  targets   : engine.ground_truth at batch B (default 32) of 368 x 368 images with P persons each (default 5), CUDA
              events around the call on the current stream (host packing, upload, 2 kernels); targets per second
  kernels   : the two target kernels' time from torch.profiler (own pass)
  cpu       : the numpy restatement tests/gt_port.py, one image at a time on the host CPU (it runs the reference's
              loops and numpy operations); with --reference DIR also the reference's own
              CocoKeypoints.get_ground_truth from that checkout, per image
  validation: PoseEngine.validation_loss (device crop, bf16 forward, targets, stage losses) over F frames of mixed
              sizes (default 64), host clock; frames per second
Every device batch is checked against the host port first.  The card's name and power limit are read in the same
call.  One JSON line.

  python tools/bench_gt.py [--batch B] [--persons P] [--runs R] [--frames F] [--reference DIR]"""
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


def scenario(seed, batch, persons):
    rs = np.random.RandomState(seed)
    kps = []
    for _ in range(batch):
        k = np.zeros((persons, 17, 3), np.float32)
        for p in range(persons):
            cx, cy, s = rs.uniform(60, 308), rs.uniform(60, 308), rs.uniform(20, 60)
            k[p, :, 0] = cx + s * rs.uniform(-1, 1, 17)
            k[p, :, 1] = cy + s * rs.uniform(-1.5, 1.5, 17)
            k[p, :, 2] = rs.choice([0, 1, 2], 17, p=[0.2, 0.2, 0.6])
        kps.append(k)
    return kps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--persons", type=int, default=5)
    ap.add_argument("--runs", type=int, default=50)
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--reference", default=None)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    import gt_port
    _b200_alias.load_package()
    eng = importlib.import_module(_b200_alias.PKG + ".engine")
    assert torch.cuda.is_available(), "bench_gt needs a GPU"
    kps = scenario(1, a.batch, a.persons)
    sizes = [(368, 368)] * a.batch
    heat, paf = eng.ground_truth(kps, sizes)
    want = gt_port.ground_truth_batch(kps, sizes)
    assert np.array_equal(heat.cpu().numpy(), want[0]) and np.array_equal(paf.cpu().numpy(), want[1])
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(a.runs):
        ev0.record()
        eng.ground_truth(kps, sizes)
        ev1.record()
        ev1.synchronize()
        ms.append(ev0.elapsed_time(ev1))
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        for _ in range(a.runs):
            eng.ground_truth(kps, sizes)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        name = re.search(r"gt_\w+_kernel", e.key)
        if name:
            us = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
            kern[name.group(0)] = kern.get(name.group(0), 0.0) + us / a.runs / 1e3
    t = time.perf_counter()
    for k in kps:
        gt_port.ground_truth(k, (368, 368))
    port_ms = 1e3 * (time.perf_counter() - t) / len(kps)
    ref_ms = None
    if a.reference:
        sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
        import make_gt_golden as mg
        ds = mg.import_reference(a.reference)
        t = time.perf_counter()
        for k in kps:
            mg.ground_truth(ds, k, (368, 368))
        ref_ms = 1e3 * (time.perf_counter() - t) / len(kps)
    # validation_loss over frames of mixed sizes
    from oracle import net_port
    sd = net_port.he_state_dict(1234)
    pe = eng.PoseEngine([v.numpy() for v in sd.values()], mode="bf16", batch_cap=32)
    rs = np.random.RandomState(2)
    srcs = [((480, 640), (640, 480), (427, 640), (360, 640))[i % 4] for i in range(a.frames)]
    images = [rs.randint(0, 256, s + (3,), dtype=np.uint8) for s in srcs]
    vk = [scenario(10 + i, 1, a.persons)[0] * np.array([s[1] / 368, s[0] / 368, 1], np.float32) for i, s in enumerate(srcs)]
    pe.validation_loss(images[:4], vk[:4])
    t = time.perf_counter()
    loss = pe.validation_loss(images, vk)
    val_s = time.perf_counter() - t
    print(json.dumps({
        "bench": "ground_truth", "card": card(), "batch": a.batch, "persons": a.persons, "size": [368, 368],
        "runs": a.runs, "call_ms_median": float(np.median(ms)), "call_ms_min": float(np.min(ms)),
        "targets_per_s": a.batch / (float(np.median(ms)) / 1e3), "kernels_ms": kern,
        "cpu_port_ms_per_image": port_ms, "cpu_reference_ms_per_image": ref_ms,
        "validation_frames": a.frames, "validation_s": val_s, "validation_frames_per_s": a.frames / val_s,
        "validation_total_loss": loss["total_loss"]}))


if __name__ == "__main__":
    main()
