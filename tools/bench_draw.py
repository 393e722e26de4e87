#!/usr/bin/env python
"""Drawing of detected persons (DESIGN.md 2.12) on 1920x1080 frames:
  kernel : b200pose_post_draw on device frames (CUDA events, plan + raster, per frame, batch of 8 frames) against the
           package's host draw_humans (imgcopy=False and True, one thread), with about 1, 8 and 30 person-like
           skeletons per frame (post-processing of synthetic stick figures on a 368 x 656 network input)
  stream : PoseStream frames/s on 1080p NV12 frames resident on the device, draw=True ('host'), 'device' and 'cuda'
           (wall clock over the whole stream, bf16, batch 8, He-initialised weights)
with the card's name, SM clocks and power limit read in the same call.  One JSON line per measurement.

  python tools/bench_draw.py [--frames F] [--iters I]"""
import argparse
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

H, W, NET = 1080, 1920, (368, 656)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=96, help="frames per PoseStream run")
    ap.add_argument("--iters", type=int, default=50, help="timed draw calls per case")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_draw needs a GPU")
    _b200_alias.load_package()
    eng = importlib.import_module(_b200_alias.PKG + ".engine")
    common = importlib.import_module(_b200_alias.PKG + ".lib.utils.common")
    p2p = importlib.import_module(_b200_alias.PKG + ".lib.utils.paf_to_pose")
    streaming = importlib.import_module(_b200_alias.PKG + ".streaming")
    from oracle import net_port, synth
    dev = card()
    n = 8
    rs = np.random.RandomState(0)
    base = rs.randint(0, 256, (n, H, W, 3)).astype(np.uint8)
    post = eng.NativePost(0, batch_cap=n, peak_cap=1024, human_cap=1024)
    for persons in (1, 8, 30):
        maps = [synth.stick_figures(persons, 100 * persons + i, h=NET[0] // 8, w=NET[1] // 8)[:2] for i in range(n)]
        heat = np.ascontiguousarray(np.stack([m[0] for m in maps]))
        paf = np.ascontiguousarray(np.stack([m[1] for m in maps]))
        post.run(heat.ctypes.data, paf.ctypes.data, False, 1, n, NET[0] // 8, NET[1] // 8, 0.1)
        post.sync()
        found = float(np.mean([len(post.humans(i)) for i in range(n)]))
        d = torch.from_numpy(base).cuda()
        st = torch.cuda.current_stream().cuda_stream
        args = (d.data_ptr(), True, n, [(H, W)] * n, [NET] * n, st)
        for _ in range(5):
            post.draw(*args)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.iters):
            post.draw(*args)
        e1.record()
        torch.cuda.synchronize()
        dev_ms = e0.elapsed_time(e1) / a.iters / n
        humans = [p2p.humans_from_rows(post.humans(i), NET[1], NET[0]) for i in range(n)]
        host = {}
        for imgcopy in (False, True):
            frames = [f.copy() for f in base]
            t0 = time.perf_counter()
            for _ in range(3):
                for f, hm in zip(frames, humans):
                    common.draw_humans(f, hm, imgcopy=imgcopy)
            host[imgcopy] = (time.perf_counter() - t0) / (3 * n) * 1e3
        print(json.dumps({"bench": "draw_kernel", "skeletons_per_frame": found, "device_ms_per_frame": round(dev_ms, 4),
                          "host_ms_per_frame": round(host[False], 3), "host_imgcopy_ms_per_frame": round(host[True], 3),
                          "frame": [H, W], "batch": n, "device": dev}), flush=True)

    sd = net_port.he_state_dict(1234)
    from lib.network.rtpose_vgg import get_model
    model = get_model("vgg19")
    model.load_state_dict(sd)
    model = model.cuda().float().eval()
    nv12 = []
    for i in range(8):
        bgr = np.random.RandomState(i).randint(0, 256, (H, W, 3)).astype(np.uint8)
        import cv2
        i420 = cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420)
        flat, q = i420.reshape(-1), (H // 2) * (W // 2)
        u, v = flat[H * W:H * W + q].reshape(H // 2, W // 2), flat[H * W + q:].reshape(H // 2, W // 2)
        nv12.append(torch.from_numpy(np.concatenate([i420[:H], np.stack([u, v], -1).reshape(H // 2, W)])).cuda())
    for rnd in range(2):
        for draw in (True, "device", "cuda"):
            frames = [nv12[k % 8] for k in range(a.frames)]
            t0 = time.perf_counter()
            k = 0
            for _, hs, drawn in streaming.PoseStream(model, frames, batch=8, format="nv12", draw=draw):
                k += 1
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            if rnd == 1:
                print(json.dumps({"bench": "pose_stream_nv12_device", "draw": "host" if draw is True else draw,
                                  "frames": k, "fps": round(k / dt, 1), "frame": [H, W], "batch": 8,
                                  "device": dev}), flush=True)


if __name__ == "__main__":
    main()
