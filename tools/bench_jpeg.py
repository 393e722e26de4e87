#!/usr/bin/env python
"""JPEG decoding on the device (DESIGN.md 2.13) on a seeded collection of 96 JPEGs with bench_mixed.py's frame shapes
(short side 240 .. 480, five aspect ratios), smooth photo-like content, quality 75 .. 95, 80 % 4:2:0:
  decode : b200pose_net_decode_jpegs into device memory in batches of 32 - the call's time from CUDA events around it
           (host parse, upload, kernels, status copy), and the five kernels' time from torch.profiler (own pass): per
           batch, images/s and compressed MB/s of both, and the Huffman kernel's share of the kernel time
  host   : cv2.imdecode on one thread and on os.cpu_count() threads
  e2e    : PoseEngine.infer_jpegs against cv2.imdecode + infer_images (bf16, dest 368, batch_cap 32, He-initialised
           weights), alternating, frames/s, with the person rows of both compared
with the card's name and power limit read in the same call.  One JSON line.

  python tools/bench_jpeg.py [--runs R]"""
import argparse
import concurrent.futures
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
sys.path.insert(0, os.path.join(ROOT, "tools"))
import _b200_alias  # noqa: E402
from bench_mixed import mixed_frames  # noqa: E402

BATCH = 32


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                       text=True)
    return r.stdout.strip().split("\n")[0]


def collection(seed=7, progressive=False):
    """96 seeded JPEG streams of bench_mixed.py's shapes; progressive: written progressive by cv2 instead."""
    import cv2
    rng = np.random.default_rng(seed)
    blobs = []
    for f in mixed_frames():
        h, w = f.shape[:2]
        low = rng.integers(0, 256, (max(2, h // 24), max(2, w // 24), 3), dtype=np.uint8)
        img = cv2.resize(low, (w, h), interpolation=cv2.INTER_CUBIC)
        img = np.clip(img.astype(np.int16) + rng.integers(-12, 13, img.shape), 0, 255).astype(np.uint8)
        for _ in range(12):
            p = tuple(int(v) for v in rng.integers(0, [w, h]))
            q = tuple(int(v) for v in rng.integers(0, [w, h]))
            cv2.line(img, p, q, tuple(int(v) for v in rng.integers(0, 256, 3)), int(rng.integers(1, 6)))
        r = rng.random()
        sf = 0x221111 if r < 0.8 else (0x111111 if r < 0.9 else 0x211111)
        ok, buf = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, int(rng.integers(75, 96)),
                                            cv2.IMWRITE_JPEG_SAMPLING_FACTOR, sf,
                                            cv2.IMWRITE_JPEG_PROGRESSIVE, int(progressive)])
        blobs.append(buf.tobytes())
    return blobs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    import cv2
    import torch
    pkg = _b200_alias.load_package()
    engine = importlib.import_module(_b200_alias.PKG + ".engine")
    nat = importlib.import_module(_b200_alias.PKG + "._native")
    from oracle import net_port
    assert torch.cuda.is_available(), "bench_jpeg needs a GPU"
    blobs = collection()
    mb = sum(len(b) for b in blobs) / 1e6
    net = engine.NativeNet(0)
    net.load_state_dict_arrays([v.numpy() for v in net_port.he_state_dict(1234).values()])
    batches = [blobs[i:i + BATCH] for i in range(0, len(blobs), BATCH)]
    shapes = [[engine.jpeg_info(b)[:2] for b in part] for part in batches]
    outs = [torch.empty(sum(h * w * 3 for h, w in s), dtype=torch.uint8, device="cuda") for s in shapes]
    tables = [engine.jpeg_table(part) for part in batches]
    stream = torch.cuda.current_stream().cuda_stream

    def decode_all():
        for (ptrs, sizes, keep), out in zip(tables, outs):
            nat.check(nat.lib().b200pose_net_decode_jpegs(net._h, ptrs, sizes, len(keep), ctypes.c_void_p(out.data_ptr()),
                                                          1, ctypes.c_void_p(stream)), "decode")

    decode_all()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2 * len(batches))]
    dev_ms, wall_ms = [], []
    for _ in range(a.runs):
        t0 = time.perf_counter()
        tot = 0.0
        for k, ((ptrs, sizes, keep), out) in enumerate(zip(tables, outs)):
            ev[2 * k].record()
            nat.check(nat.lib().b200pose_net_decode_jpegs(net._h, ptrs, sizes, len(keep), ctypes.c_void_p(out.data_ptr()),
                                                          1, ctypes.c_void_p(stream)), "decode")
            ev[2 * k + 1].record()
        torch.cuda.synchronize()
        wall_ms.append((time.perf_counter() - t0) * 1e3)
        for k in range(len(batches)):
            tot += ev[2 * k].elapsed_time(ev[2 * k + 1])
        dev_ms.append(tot)
    # kernel split (own pass)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        decode_all()
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        if "jpeg_" in e.name and e.device_type.name == "CUDA":
            key = e.name.split("jpeg_")[1].split("_kernel")[0]
            kern[key] = kern.get(key, 0.0) + e.device_time / 1e3
    ktot = sum(kern.values()) or 1.0
    # host cv2
    cv2.setNumThreads(1)
    arrs = [np.frombuffer(b, np.uint8) for b in blobs]
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
    # end to end, alternating
    pe = engine.PoseEngine.from_net(net, mode="bf16", batch_cap=BATCH)
    e2e = {"infer_jpegs": [], "imdecode+infer_images": []}
    same = True
    for r in range(a.runs + 1):
        t0 = time.perf_counter()
        got = pe.infer_jpegs_arrays(blobs)
        t1 = time.perf_counter()
        want = pe.infer_images_arrays([cv2.imdecode(x, cv2.IMREAD_COLOR) for x in arrs])
        t2 = time.perf_counter()
        same = same and all(np.array_equal(g, w) for g, w in zip(got, want))
        if r:
            e2e["infer_jpegs"].append(len(blobs) / (t1 - t0))
            e2e["imdecode+infer_images"].append(len(blobs) / (t2 - t1))
    med = lambda v: float(np.median(v))
    spread = lambda v: [float(np.min(v)), float(np.max(v))]
    print(json.dumps({
        "card": card(), "images": len(blobs), "compressed_MB": round(mb, 3), "batch": BATCH,
        "decode_call_ms_per_batch": round(med(dev_ms) / len(batches), 3),
        "decode_call_images_per_s": round(len(blobs) / (med(dev_ms) / 1e3), 1),
        "decode_call_images_per_s_spread": [round(len(blobs) / (v / 1e3), 1) for v in (max(dev_ms), min(dev_ms))],
        "decode_call_MB_per_s": round(mb / (med(dev_ms) / 1e3), 1),
        "decode_call_wall_ms_per_batch": round(med(wall_ms) / len(batches), 3),
        "decode_kernel_ms_per_batch": round(ktot / len(batches), 3),
        "decode_kernel_images_per_s": round(len(blobs) / (ktot / 1e3), 1),
        "decode_kernel_MB_per_s": round(mb / (ktot / 1e3), 1),
        "kernel_ms": {k: round(v, 3) for k, v in kern.items()}, "huffman_share": round(kern.get("huff", 0) / ktot, 3),
        "cv2_1thread_images_per_s": round(len(blobs) / med(one), 1),
        "cv2_threads": os.cpu_count(), "cv2_nthreads_images_per_s": round(len(blobs) / med(many), 1),
        "e2e_frames_per_s": {k: round(med(v), 1) for k, v in e2e.items()},
        "e2e_spread": {k: [round(x, 1) for x in spread(v)] for k, v in e2e.items()},
        "e2e_rows_equal": bool(same)}))


if __name__ == "__main__":
    main()
