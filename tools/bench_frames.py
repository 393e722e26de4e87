#!/usr/bin/env python
"""Video-frame ingestion (DESIGN.md 2.10): 1920x1080 frames at dest_size 368 in three forms, alternating in one process:
  nv12_device : NV12 frames resident on the device (a hardware decoder's output), PoseEngine.infer_frames_async
  nv12_pinned : NV12 frames in pinned host memory, PoseEngine.infer_frames_async (planes cross PCIe, then convert)
  bgr_pinned  : the same frames as BGR in pinned host memory through the existing b200pose_infer_raw_u8 path
Two submissions are kept in flight (submit batch i + 1, then fetch batch i), as PoseStream does.  Prints per batch size
and form frames/s (wall clock, median over the runs) and launches per frame, then the conversion kernel's time per
frame and its GB/s (NV12 read + BGR written, over CUDA-event time of b200pose_net_convert_frames into device memory),
with the card's name, SM clocks and power limit read in the same call.  One JSON line per measurement.

  python tools/bench_frames.py [--batches 8 32] [--runs R] [--steps K] [--warmup W] [--mode bf16]"""
import argparse
import ctypes
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import _b200_alias  # noqa: E402

H, W, DEST = 1080, 1920, 368


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[8, 32])
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--mode", default="bf16")
    args = ap.parse_args()
    import cv2
    import torch
    _b200_alias.load_package()
    engine = importlib.import_module(_b200_alias.PKG + ".engine")
    nat = importlib.import_module(_b200_alias.PKG + "._native")
    syn = importlib.import_module(_b200_alias.PKG + ".synthetic")
    print(json.dumps({"card_before": card(), "gpu": torch.cuda.get_device_properties(0).name}))
    rng = np.random.default_rng(7)
    cap = max(args.batches)
    # seeded photo-like frames: smooth gradients plus noise, so that the network sees structure
    yy, xx = np.mgrid[0:H, 0:W]
    frames_nv12 = []
    for i in range(cap):
        bgr = np.stack([(xx * (i + 1) // 8 + yy // 4) % 256, (yy * 3 // 5 + i * 17) % 256, (xx + yy) // 12 % 256], -1)
        bgr = (bgr + rng.integers(0, 32, bgr.shape)).clip(0, 255).astype(np.uint8)
        i420 = cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420)
        flat, q = i420.reshape(-1), (H // 2) * (W // 2)
        uv = np.stack([flat[H * W:H * W + q], flat[H * W + q:]], -1).reshape(H // 2, W)
        frames_nv12.append(np.concatenate([i420[:H], uv]))
    nv12_pinned = torch.from_numpy(np.stack(frames_nv12)).pin_memory()
    nv12_dev = nv12_pinned.cuda()
    bgr_pinned = torch.from_numpy(np.stack([cv2.cvtColor(f, cv2.COLOR_YUV2BGR_NV12) for f in frames_nv12])).pin_memory()
    eng = engine.PoseEngine(syn.he_state_arrays(1234), 0, mode=args.mode, batch_cap=cap, peak_cap=1024, human_cap=4096)

    def submit(form, n):
        if form == "nv12_device":
            return eng.infer_frames_async(list(nv12_dev[:n]), "nv12", 0, DEST)
        if form == "nv12_pinned":
            return eng.infer_frames_async(list(nv12_pinned[:n].numpy()), "nv12", 0, DEST)
        return eng.infer_raw_async_u8(bgr_pinned.data_ptr(), False, n, H, W, DEST)

    def run(form, n, steps):
        prev = submit(form, n)
        for _ in range(steps - 1):
            t = submit(form, n)
            eng.fetch_arrays(check=False, ticket=prev)
            prev = t
        eng.fetch_arrays(check=False, ticket=prev)

    forms = ("nv12_device", "nv12_pinned", "bgr_pinned")
    for n in args.batches:
        for form in forms:
            run(form, n, args.warmup + 1)
        rates = {f: [] for f in forms}
        launches = {}
        for _ in range(args.runs):
            for form in forms:
                torch.cuda.synchronize()
                l0 = nat.launch_count()
                t0 = time.perf_counter()
                run(form, n, args.steps)
                torch.cuda.synchronize()
                rates[form].append(n * args.steps / (time.perf_counter() - t0))
                launches[form] = (nat.launch_count() - l0) / (n * args.steps)
        for form in forms:
            print(json.dumps({"metric": "frames/s", "form": form, "batch": n, "value": round(float(np.median(rates[form])), 1),
                              "runs": [round(r, 1) for r in rates[form]], "launches_per_frame": round(launches[form], 3),
                              "frame": "%dx%d" % (W, H), "dest_size": DEST, "mode": args.mode}))
    # the conversion kernel alone: device NV12 -> device BGR, CUDA events around R calls
    for n in args.batches:
        table, keep, on_dev, _ = engine.frame_table(list(nv12_dev[:n]), "nv12")
        out = torch.empty(n * H * W * 3, dtype=torch.uint8, device="cuda")
        s = torch.cuda.current_stream()

        def convert():
            nat.check(nat.lib().b200pose_net_convert_frames(eng.net._h, table, n, 1, 1, 0, ctypes.c_void_p(out.data_ptr()),
                                                            1, ctypes.c_void_p(s.cuda_stream)), "convert_frames")
        for _ in range(5):
            convert()
        reps = 50
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(s)
        for _ in range(reps):
            convert()
        e1.record(s)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / reps
        moved = n * H * W * (1.5 + 3)
        print(json.dumps({"metric": "convert_frames_kernel", "batch": n, "ms_per_call": round(ms, 4),
                          "us_per_frame": round(ms * 1e3 / n, 2), "GB_per_s": round(moved / (ms * 1e-3) / 1e9, 1),
                          "bytes_per_frame": int(H * W * 4.5), "note": "includes the 1-entry table upload per call"}))
    print(json.dumps({"card_after": card()}))


if __name__ == "__main__":
    main()
