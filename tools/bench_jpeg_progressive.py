#!/usr/bin/env python
"""Progressive JPEG decoding on the device (DESIGN.md 2.18) on bench_jpeg.py's collection of 96 streams (bench_mixed.py's
frame shapes), written progressive by cv2 (its 10-scan script, no restart markers):
  decode : b200pose_net_decode_jpegs with the net's progressive switch on, into device memory in batches of 32 - the
           call's time from CUDA events around it (host parse, upload, kernels, status copy), and each kernel's time
           from torch.profiler (own pass)
  host   : cv2.imdecode on one thread and on os.cpu_count() threads
  e2e    : PoseEngine.infer_jpegs with jpeg_progressive on (device decoding) against off (cv2.imdecode fallback), bf16,
           dest 368, batch_cap 32, He-initialised weights, alternating, frames/s, with the person rows compared
with the card's name and power limit read in the same call.  One JSON line.

  python tools/bench_jpeg_progressive.py [--runs R]"""
import argparse
import concurrent.futures
import ctypes
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
from bench_jpeg import BATCH, card, collection  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    import cv2
    import torch
    _b200_alias.load_package()
    engine = importlib.import_module(_b200_alias.PKG + ".engine")
    nat = importlib.import_module(_b200_alias.PKG + "._native")
    from oracle import net_port
    assert torch.cuda.is_available(), "bench_jpeg_progressive needs a GPU"
    blobs = collection(progressive=True)
    assert all(not engine.jpeg_info(b)[2] and engine.jpeg_info(b, progressive=True)[2] for b in blobs)
    mb = sum(len(b) for b in blobs) / 1e6
    net = engine.NativeNet(0)
    net.load_state_dict_arrays([v.numpy() for v in net_port.he_state_dict(1234).values()])
    net.set_jpeg_progressive(True)
    batches = [blobs[i:i + BATCH] for i in range(0, len(blobs), BATCH)]
    shapes = [[engine.jpeg_info(b, progressive=True)[:2] for b in part] for part in batches]
    outs = [torch.empty(sum(h * w * 3 for h, w in s), dtype=torch.uint8, device="cuda") for s in shapes]
    tables = [engine.jpeg_table(part) for part in batches]
    stream = torch.cuda.current_stream().cuda_stream

    def decode(k):
        ptrs, sizes, keep = tables[k]
        nat.check(nat.lib().b200pose_net_decode_jpegs(net._h, ptrs, sizes, len(keep), ctypes.c_void_p(outs[k].data_ptr()),
                                                      1, ctypes.c_void_p(stream)), "decode")

    for k in range(len(batches)):
        decode(k)
    # the device frames equal cv2's
    arrs = [np.frombuffer(b, np.uint8) for b in blobs]
    same_frames = True
    for k, part in enumerate(batches):
        at, flat = 0, outs[k].cpu().numpy()
        for (h, w), b in zip(shapes[k], part):
            same_frames &= bool(np.array_equal(flat[at:at + h * w * 3].reshape(h, w, 3),
                                               cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)))
            at += h * w * 3
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2 * len(batches))]
    dev_ms, wall_ms = [], []
    for _ in range(a.runs):
        t0 = time.perf_counter()
        for k in range(len(batches)):
            ev[2 * k].record()
            decode(k)
            ev[2 * k + 1].record()
        torch.cuda.synchronize()
        wall_ms.append((time.perf_counter() - t0) * 1e3)
        dev_ms.append(sum(ev[2 * k].elapsed_time(ev[2 * k + 1]) for k in range(len(batches))))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in range(len(batches)):
            decode(k)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        if "jpeg_" in e.name and e.device_type.name == "CUDA":
            key = e.name.split("jpeg_")[1].split("_kernel")[0]
            kern[key] = kern.get(key, 0.0) + e.device_time / 1e3
    ktot = sum(kern.values()) or 1.0
    cv2.setNumThreads(1)
    one, many = [], []
    for _ in range(a.runs):
        t0 = time.perf_counter()
        for x in arrs:
            cv2.imdecode(x, cv2.IMREAD_COLOR)
        one.append(time.perf_counter() - t0)
        with concurrent.futures.ThreadPoolExecutor(os.cpu_count()) as ex:
            t0 = time.perf_counter()
            list(ex.map(lambda x: cv2.imdecode(x, cv2.IMREAD_COLOR), arrs))
            many.append(time.perf_counter() - t0)
    pe = engine.PoseEngine.from_net(net, mode="bf16", batch_cap=BATCH)
    e2e = {"switch_on": [], "switch_off": []}
    same = True
    for r in range(a.runs + 1):
        pe.set_jpeg_progressive(True)
        t0 = time.perf_counter()
        got = pe.infer_jpegs_arrays(blobs)
        t1 = time.perf_counter()
        pe.set_jpeg_progressive(False)
        want = pe.infer_jpegs_arrays(blobs)
        t2 = time.perf_counter()
        same = same and all(np.array_equal(g, w) for g, w in zip(got, want))
        if r:
            e2e["switch_on"].append(len(blobs) / (t1 - t0))
            e2e["switch_off"].append(len(blobs) / (t2 - t1))
    med = lambda v: float(np.median(v))
    print(json.dumps({
        "card": card(), "images": len(blobs), "compressed_MB": round(mb, 3), "batch": BATCH,
        "frames_equal_cv2": same_frames,
        "decode_call_ms_per_batch": round(med(dev_ms) / len(batches), 3),
        "decode_call_images_per_s": round(len(blobs) / (med(dev_ms) / 1e3), 1),
        "decode_call_images_per_s_spread": [round(len(blobs) / (v / 1e3), 1) for v in (max(dev_ms), min(dev_ms))],
        "decode_call_wall_ms_per_batch": round(med(wall_ms) / len(batches), 3),
        "decode_kernel_ms_per_batch": round(ktot / len(batches), 3),
        "kernel_ms_per_batch": {k: round(v / len(batches), 3) for k, v in kern.items()},
        "decode_kernel_images_per_s": round(len(blobs) / (ktot / 1e3), 1),
        "cv2_1thread_images_per_s": round(len(blobs) / med(one), 1),
        "cv2_threads": os.cpu_count(), "cv2_nthreads_images_per_s": round(len(blobs) / med(many), 1),
        "e2e_frames_per_s": {k: round(med(v), 1) for k, v in e2e.items()},
        "e2e_spread": {k: [round(float(np.min(v)), 1), round(float(np.max(v)), 1)] for k, v in e2e.items()},
        "e2e_rows_equal": bool(same)}))


if __name__ == "__main__":
    main()
