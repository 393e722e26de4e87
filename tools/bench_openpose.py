#!/usr/bin/env python
"""OpenPose_Model(4, 2) against rtpose at 6 and 3 stages on bench.py's workload: seeded weights, batch 32 (--batch) of
seeded 368 x 368 uint8 frames on the device, fused post-processing, the three configurations alternating in one process
for R runs.  Then per configuration, from b200pose_net_profile (fastest of 5 profiled passes per launch): launches per
frame, and milliseconds, algorithmic and padded GFLOP/frame and TFLOP/s summed by layer kind; with the card's name and
power limit read in the same call.  Prints a table and ONE JSON line.

  python tools/bench_openpose.py [--mode bf16] [--runs R] [--steps K] [--warmup W] [--batch N]
"""
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

CONFIGS = ("openpose(4,2)", "rtpose6", "rtpose3")


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def kind_of(i, f, openpose):
    """Layer kind of launch i from its b200pose_net_debug_launch fields."""
    if i == 0:
        return "conv1_1"
    if i <= 11:
        return "trunk 3x3"
    if f[23] >= 0:
        return "head 1x1"
    if f[12] == 1:
        return "Mconv6 1x1" if openpose else "1x1"
    if openpose:
        return "dense 3x3 (96)" if f[15] == 48 else "dense 3x3 (128)"
    return "%dx%d" % (f[12], f[12])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="bf16")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=32)
    args = ap.parse_args()
    import torch
    _b200_alias.load_package()
    engine = importlib.import_module(_b200_alias.PKG + ".engine")
    nat = importlib.import_module(_b200_alias.PKG + "._native")
    syn = importlib.import_module(_b200_alias.PKG + ".synthetic")
    if not torch.cuda.is_available():
        raise SystemExit("bench_openpose.py needs a GPU")
    n, H, W = args.batch, 368, 368
    rt = engine.NativeNet(0)
    rt.load_state_dict_arrays(syn.he_state_arrays(1234))
    pes = {"openpose(4,2)": engine.openpose_engine(syn.openpose_state_dict(4, 2), 4, 2, 0, args.mode, batch_cap=n,
                                                   peak_cap=2048, human_cap=2048),
           "rtpose6": engine.PoseEngine.from_net(rt, args.mode, n, 2048, 2048, stages=6),
           "rtpose3": engine.PoseEngine.from_net(rt, args.mode, n, 2048, 2048, stages=3)}
    frames = torch.from_numpy(np.random.default_rng(0).integers(0, 256, (n, H, W, 3), dtype=np.uint8)).cuda()
    st = torch.cuda.Stream()

    def step(c):      # two runs in flight, as bench.py keeps them: fetch the previous one after submitting the next
        pe = pes[c]
        t = pe.infer_async_u8(frames.data_ptr(), True, n, H, W, 0.1, st.cuda_stream)
        if t > 0:
            pe.post.select(t - 1)
        return pe

    def finish(pe):
        pe.post.sync()
        pe.post.check_status(n)

    fps = {c: [] for c in CONFIGS}
    for c in CONFIGS:
        for _ in range(args.warmup):
            step(c)
        finish(pes[c])
    for _ in range(args.runs):
        for c in CONFIGS:
            finish(step(c))
            t0 = time.perf_counter()
            for _ in range(args.steps):
                pe = step(c)
            finish(pe)
            fps[c].append(n * args.steps / (time.perf_counter() - t0))
    prof = {}
    for c in CONFIGS:
        pe = pes[c]
        net = pe.net
        if net.openpose_stages is None:
            net.set_stages(pe.stages)
        net.forward_u8_ptr(frames.data_ptr(), True, n, H, W, nat.MODES[args.mode], [0] * 12, True, st.cuda_stream)
        st.synchronize()
        ms = np.zeros(256, np.float32)
        fl = np.zeros(256, np.float64)
        best = None
        for _ in range(5):
            cnt = nat.lib().b200pose_net_profile(net._h, ms.ctypes.data, fl.ctypes.data, 256, st.cuda_stream)
            assert cnt > 0, nat.lib().b200pose_last_error()
            best = ms[:cnt].copy() if best is None else np.minimum(best, ms[:cnt])
        kinds = {}
        fields = np.zeros(32, np.int32)
        for i in range(cnt):
            if nat.lib().b200pose_net_debug_launch(net._h, i, fields.ctypes.data, 32) < 27:     # fields written
                nat.check(1, "b200pose_net_debug_launch")
            f = fields.tolist()
            k = kind_of(i, f, net.openpose_stages is not None)
            # padded: what the kernel multiplies - 64-channel K blocks and whole n-tiles, per group
            padded = fl[i] if i == 0 else 2.0 * n * f[10] * f[11] * f[12] ** 2 * f[13] * 64 * f[14] * f[16] * f[15]
            e = kinds.setdefault(k, [0, 0.0, 0.0, 0.0])
            e[0] += 1
            e[1] += float(best[i])
            e[2] += float(fl[i])
            e[3] += float(padded)
        prof[c] = (cnt, kinds)
    rt.set_stages(6)
    name = card()
    print("%s; mode %s; batch %d x %dx%d uint8 on the device, fused post-processing; %d runs x %d steps per "
          "configuration, alternating" % (name, args.mode, n, H, W, args.runs, args.steps))
    for c in CONFIGS:
        cnt, kinds = prof[c]
        tot = [sum(v[i] for v in kinds.values()) for i in range(4)]
        print("\n%s: frames/s %s; %d launches per batch; net %.2f ms, %.1f GFLOP/frame (padded %.1f), %.1f TFLOP/s"
              % (c, " ".join("%.1f" % v for v in fps[c]), cnt, tot[1], tot[2] / n / 1e9, tot[3] / n / 1e9,
                 tot[2] / tot[1] / 1e9))
        print("  %-18s %8s %8s %12s %12s %8s" % ("kind", "launches", "ms", "GFLOP/frame", "padded", "TFLOP/s"))
        for k, (m, t, f, p) in kinds.items():
            print("  %-18s %8d %8.2f %12.2f %12.2f %8.1f" % (k, m, t, f / n / 1e9, p / n / 1e9, f / t / 1e9 if t else 0))
    print(json.dumps({"card": name, "mode": args.mode, "batch": n, "fps": fps,
                      "launches": {c: prof[c][0] for c in CONFIGS},
                      "kinds": {c: {k: {"launches": v[0], "ms": round(v[1], 3), "gflop_frame": round(v[2] / n / 1e9, 2),
                                        "padded_gflop_frame": round(v[3] / n / 1e9, 2)}
                                    for k, v in prof[c][1].items()} for c in CONFIGS}}))


if __name__ == "__main__":
    main()
