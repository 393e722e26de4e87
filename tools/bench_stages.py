#!/usr/bin/env python
"""Frames/s per refinement-stage count on bench.py's workload (seeded weights, batch 32 of seeded 368 x 368 uint8 frames on
the device, fused post-processing), k = 6 .. 1 alternating in one process for R runs; then per k the summed per-launch
milliseconds and TFLOP/s of the plan from b200pose_net_profile (algorithmic FLOPs), with the card's name and power limit
read in the same call.  Prints a table and ONE JSON line.

  python tools/bench_stages.py [--mode bf16] [--runs R] [--steps K] [--warmup W] [--batch N]
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

STAGES = (6, 5, 4, 3, 2, 1)


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


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
        raise SystemExit("bench_stages.py needs a GPU")
    net = engine.NativeNet(0)
    net.load_state_dict_arrays(syn.he_state_arrays(1234))
    pes = {k: engine.PoseEngine.from_net(net, args.mode, args.batch, 2048, 2048, stages=k) for k in STAGES}
    n, H, W = args.batch, 368, 368
    frames = torch.from_numpy(np.random.default_rng(0).integers(0, 256, (n, H, W, 3), dtype=np.uint8)).cuda()
    st = torch.cuda.Stream()

    def step(k):      # two runs in flight, as bench.py keeps them: fetch the previous one after submitting the next
        pe = pes[k]
        t = pe.infer_async_u8(frames.data_ptr(), True, n, H, W, 0.1, st.cuda_stream)
        if t > 0:
            pe.post.select(t - 1)
        return pe

    def finish(pe):
        pe.post.sync()
        pe.post.check_status(n)

    fps = {k: [] for k in STAGES}
    for k in STAGES:
        for _ in range(args.warmup):
            step(k)
        finish(pes[k])
    for _ in range(args.runs):
        for k in STAGES:
            finish(step(k))
            t0 = time.perf_counter()
            for _ in range(args.steps):
                pe = step(k)
            finish(pe)
            fps[k].append(n * args.steps / (time.perf_counter() - t0))
    prof = {}
    for k in STAGES:
        net.set_stages(k)
        net.forward_u8_ptr(frames.data_ptr(), True, n, H, W, nat.MODES[args.mode], [0] * 12, True, st.cuda_stream)
        st.synchronize()
        ms = np.zeros(64, np.float32)
        fl = np.zeros(64, np.float64)
        best = None
        for _ in range(5):     # per launch: the fastest of 5 profiled passes
            cnt = nat.lib().b200pose_net_profile(net._h, ms.ctypes.data, fl.ctypes.data, 64, st.cuda_stream)
            assert cnt > 0, nat.lib().b200pose_last_error()
            best = ms[:cnt].copy() if best is None else np.minimum(best, ms[:cnt])
        prof[k] = (float(best.sum()), float(fl[:cnt].sum()), cnt)
    net.set_stages(6)
    name = card()
    print("%s; mode %s; batch %d x %dx%d, fused post-processing; %d runs x %d steps per stage count, alternating"
          % (name, args.mode, n, H, W, args.runs, args.steps))
    print("stages  launches  GFLOP/frame  frames/s (runs)                 net ms  TFLOP/s")
    for k in STAGES:
        ms_sum, fl_sum, cnt = prof[k]
        print("%6d  %8d  %11.1f  %-30s  %6.2f  %7.1f" % (k, cnt, fl_sum / n / 1e9, " ".join("%.1f" % v for v in fps[k]),
                                                       ms_sum, fl_sum / ms_sum / 1e9))
    print(json.dumps({"card": name, "mode": args.mode, "batch": n, "fps": {str(k): fps[k] for k in STAGES},
                      "net_ms": {str(k): round(prof[k][0], 3) for k in STAGES},
                      "gflop_per_frame": {str(k): round(prof[k][1] / n / 1e9, 2) for k in STAGES},
                      "launches": {str(k): prof[k][2] for k in STAGES}}))


if __name__ == "__main__":
    main()
