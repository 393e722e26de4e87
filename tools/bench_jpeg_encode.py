#!/usr/bin/env python
"""JPEG encoding on the device (DESIGN.md 2.14), quality 95, 4:2:0, three batches: 32 x 640x480, 32 x 1920x1080 and
bench_mixed.py's 96 mixed shapes as drawn frames (photo-like content with lines drawn on it), in calls of up to 32:
  device : b200pose_net_encode_jpegs from device frames to host bytes - the call's time from CUDA events around it
           (descriptor upload, five kernels, size copy and synchronisation, stream copy), images/s and output MB/s, and
           the five kernels' time from torch.profiler (own pass)
  host   : cv2.imencode on one thread and on os.cpu_count() threads
  run_eval's visualisation step per image, 32 COCO-sized (640x480) frames with 3 .. 8 persons each from synthetic
           maps: before - host draw_humans + cv2.imwrite per image; after - coco_eval.write_vis_device (one packed
           upload, b200pose_post_draw in place, encode from the same buffer, write), host clock around each including
           the file writes, alternating, with the files of both compared byte for byte
Every repetition checks that the device's bytes equal cv2's.  The card's name and power limit are read in the same
call.  One JSON line.

  python tools/bench_jpeg_encode.py [--runs R]"""
import argparse
import concurrent.futures
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
QUALITY, SAMPLING = 95, "420"


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                       text=True)
    return r.stdout.strip().split("\n")[0]


def drawn(h, w, rng):
    import cv2
    low = rng.integers(0, 256, (max(2, h // 24), max(2, w // 24), 3), dtype=np.uint8)
    img = cv2.resize(low, (w, h), interpolation=cv2.INTER_CUBIC)
    img = np.clip(img.astype(np.int16) + rng.integers(-12, 13, img.shape), 0, 255).astype(np.uint8)
    for _ in range(12):
        p = tuple(int(v) for v in rng.integers(0, [w, h]))
        q = tuple(int(v) for v in rng.integers(0, [w, h]))
        cv2.line(img, p, q, tuple(int(v) for v in rng.integers(0, 256, 3)), 3)
        cv2.circle(img, p, 3, tuple(int(v) for v in rng.integers(0, 256, 3)), 3)
    return img


def batches(seed=5):
    rng = np.random.default_rng(seed)
    return {"32x640x480": [drawn(480, 640, rng) for _ in range(BATCH)],
            "32x1920x1080": [drawn(1080, 1920, rng) for _ in range(BATCH)],
            "96_mixed": [drawn(f.shape[0], f.shape[1], rng) for f in mixed_frames()]}


def main():
    import cv2
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=10)
    a = ap.parse_args()
    _b200_alias.load_package()
    engine = importlib.import_module(_b200_alias.PKG + ".engine")
    net = engine.NativeNet(0)
    res = {"card": card(), "quality": QUALITY, "sampling": SAMPLING, "runs": a.runs, "batches": {}}
    params = [cv2.IMWRITE_JPEG_QUALITY, QUALITY, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, 0x221111]
    pool = concurrent.futures.ThreadPoolExecutor(os.cpu_count())
    for name, frames in batches().items():
        want = [cv2.imencode(".jpg", f, params)[1].tobytes() for f in frames]
        chunks = [[torch.from_numpy(f).cuda() for f in frames[i:i + BATCH]] for i in range(0, len(frames), BATCH)]
        out_mb = sum(len(w) for w in want) / 1e6
        for c in chunks:                                    # warm-up: every shape and buffer size
            net.encode_jpegs(c, QUALITY, SAMPLING)
        torch.cuda.synchronize()
        times = []
        for _ in range(a.runs):
            got = []
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            for c in chunks:
                got += net.encode_jpegs(c, QUALITY, SAMPLING)
            ev1.record()
            torch.cuda.synchronize()
            times.append(ev0.elapsed_time(ev1))
            assert got == want, "device streams differ from cv2.imencode (%s)" % name
        ms = float(np.median(times))
        acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
        with torch.profiler.profile(activities=acts) as prof:
            for c in chunks:
                got = net.encode_jpegs(c, QUALITY, SAMPLING)
            torch.cuda.synchronize()
        assert got == want[-len(got):]
        kern, api = {}, {}
        for e in prof.key_averages():
            if "jpeg_enc" in e.key:
                k = e.key.split("jpeg_enc_")[1].split("_kernel")[0]
                kern[k] = round(getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) / 1e3, 3)
            elif e.key.startswith("cuda") and e.cpu_time_total > 50:      # runtime calls of the host side, over 50 us
                api[e.key] = round(e.cpu_time_total / 1e3, 3)
        kms = sum(kern.values())
        t0 = time.perf_counter()                                # the call's host wall time, end to end
        for _ in range(a.runs):
            for c in chunks:
                net.encode_jpegs(c, QUALITY, SAMPLING)
        wall = (time.perf_counter() - t0) / a.runs * 1e3
        t0 = time.perf_counter()
        for _ in range(a.runs):
            host = [cv2.imencode(".jpg", f, params)[1].tobytes() for f in frames]
        one = (time.perf_counter() - t0) / a.runs * 1e3
        assert host == want
        t0 = time.perf_counter()
        for _ in range(a.runs):
            list(pool.map(lambda f: cv2.imencode(".jpg", f, params)[1], frames))
        many = (time.perf_counter() - t0) / a.runs * 1e3
        n = len(frames)
        res["batches"][name] = {
            "images": n, "out_MB": round(out_mb, 3),
            "device_call_ms": round(ms, 3), "device_images_per_s": round(n / ms * 1e3, 1),
            "device_out_MB_per_s": round(out_mb / ms * 1e3, 1),
            "kernel_ms": kern, "kernel_total_ms": round(kms, 3), "host_wall_ms": round(wall, 3),
            "runtime_api_cpu_ms": api,
            "kernel_images_per_s": round(n / kms * 1e3, 1) if kms else None,
            "cv2_1thread_ms": round(one, 3), "cv2_1thread_images_per_s": round(n / one * 1e3, 1),
            "cv2_threads": os.cpu_count(), "cv2_threads_ms": round(many, 3),
            "cv2_threads_images_per_s": round(n / many * 1e3, 1)}
    res["run_eval_vis"] = vis_step(engine, net, a.runs)
    print(json.dumps(res))


def vis_step(engine, net, runs):
    """run_eval's visualisation step, before and after, ms per image."""
    import tempfile
    import cv2
    from oracle import synth
    ev = importlib.import_module(_b200_alias.PKG + ".evaluate.coco_eval")
    common = importlib.import_module(_b200_alias.PKG + ".lib.utils.common")
    p2p = importlib.import_module(_b200_alias.PKG + ".lib.utils.paf_to_pose")
    n = BATCH
    post = engine.NativePost(0, batch_cap=n, peak_cap=1024, human_cap=256)
    maps = [synth.stick_figures(3 + k % 6, 100 + k)[:2] for k in range(n)]
    heat = np.ascontiguousarray(np.stack([m[0] for m in maps]))
    paf = np.ascontiguousarray(np.stack([m[1] for m in maps]))
    post.run(heat.ctypes.data, paf.ctypes.data, False, 1, n, 46, 46, 0.1)
    post.sync()
    rng = np.random.default_rng(9)
    frames = [drawn(480, 640, rng) for _ in range(n)]
    humans = [p2p.humans_from_rows(post.humans(i), 368, 368) for i in range(n)]
    before, after = [], []
    with tempfile.TemporaryDirectory() as d:
        host = [os.path.join(d, "host%d.jpg" % i) for i in range(n)]
        dev = [os.path.join(d, "dev%d.jpg" % i) for i in range(n)]
        for r in range(runs + 1):
            t0 = time.perf_counter()
            for i in range(n):
                cv2.imwrite(host[i], common.draw_humans(frames[i].copy(), humans[i]))
            t1 = time.perf_counter()
            ev.write_vis_device(post, net, frames, [(368, 368)] * n, dev, list(range(n)))
            t2 = time.perf_counter()
            if r:                                              # the first round warms both up
                before.append((t1 - t0) / n * 1e3)
                after.append((t2 - t1) / n * 1e3)
            for i in range(n):
                assert open(host[i], "rb").read() == open(dev[i], "rb").read(), "visualisation %d differs" % i
    return {"frames": "%d x 640x480, 3 .. 8 persons" % n,
            "before_host_draw_imwrite_ms_per_image": round(float(np.median(before)), 3),
            "after_device_draw_encode_write_ms_per_image": round(float(np.median(after)), 3),
            "before_range": [round(min(before), 3), round(max(before), 3)],
            "after_range": [round(min(after), 3), round(max(after), 3)]}


if __name__ == "__main__":
    main()
