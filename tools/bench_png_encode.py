#!/usr/bin/env python
"""PNG encoding on the device (DESIGN.md 2.15), three batches of drawn frames (bench_jpeg_encode.py's: photo-like
content with lines and circles drawn on it): 32 x 640x480, 32 x 1920x1080 and bench_mixed.py's 96 mixed shapes, in
calls of up to 32:
  device : b200pose_net_encode_pngs from device frames to host bytes - the call's time from CUDA events around it
           (descriptor upload, nine kernels, size copy and synchronisation, file copy), images/s, and the nine
           kernels' time from torch.profiler (own pass)
  host   : cv2.imencode('.png') on one thread and on os.cpu_count() threads
Every repetition checks that the device's bytes equal cv2's.  The card's name and power limit are read in the same
call.  One JSON line.

  python tools/bench_png_encode.py [--runs R]"""
import argparse
import concurrent.futures
import importlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import _b200_alias  # noqa: E402
from bench_jpeg_encode import BATCH, batches, card  # noqa: E402


def main():
    import cv2
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    _b200_alias.load_package()
    engine = importlib.import_module(_b200_alias.PKG + ".engine")
    net = engine.NativeNet(0)
    res = {"card": card(), "runs": a.runs, "batches": {}}
    pool = concurrent.futures.ThreadPoolExecutor(os.cpu_count())
    for name, frames in batches().items():
        want = [cv2.imencode(".png", f)[1].tobytes() for f in frames]
        chunks = [[torch.from_numpy(f).cuda() for f in frames[i:i + BATCH]] for i in range(0, len(frames), BATCH)]
        out_mb = sum(len(w) for w in want) / 1e6
        for c in chunks:                                    # warm-up: every shape and buffer size
            net.encode_pngs(c)
        torch.cuda.synchronize()
        times = []
        for _ in range(a.runs):
            got = []
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            for c in chunks:
                got += net.encode_pngs(c)
            ev1.record()
            torch.cuda.synchronize()
            times.append(ev0.elapsed_time(ev1))
            assert got == want, "device files differ from cv2.imencode (%s)" % name
        ms = float(np.median(times))
        acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
        with torch.profiler.profile(activities=acts) as prof:
            for c in chunks:
                got = net.encode_pngs(c)
            torch.cuda.synchronize()
        assert got == want[-len(got):]
        kern = {}
        for e in prof.key_averages():
            if "png_enc" in e.key:
                k = e.key.split("png_enc_")[1].split("_kernel")[0]
                kern[k] = round(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) / 1e3, 3)
        kms = sum(kern.values())
        t0 = time.perf_counter()
        for _ in range(a.runs):
            host = [cv2.imencode(".png", f)[1].tobytes() for f in frames]
        one = (time.perf_counter() - t0) / a.runs * 1e3
        assert host == want
        t0 = time.perf_counter()
        for _ in range(a.runs):
            list(pool.map(lambda f: cv2.imencode(".png", f)[1], frames))
        many = (time.perf_counter() - t0) / a.runs * 1e3
        n = len(frames)
        res["batches"][name] = {
            "images": n, "out_MB": round(out_mb, 3),
            "device_call_ms": round(ms, 3), "device_call_range_ms": [round(min(times), 3), round(max(times), 3)],
            "device_images_per_s": round(n / ms * 1e3, 1),
            "kernel_ms": kern, "kernel_total_ms": round(kms, 3),
            "cv2_1thread_ms": round(one, 3), "cv2_1thread_images_per_s": round(n / one * 1e3, 1),
            "cv2_threads": os.cpu_count(), "cv2_threads_ms": round(many, 3),
            "cv2_threads_images_per_s": round(n / many * 1e3, 1)}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
