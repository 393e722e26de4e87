#!/usr/bin/env python
"""Two arithmetic modes (default bf16 against fp8) on the network forward of bench.py's workload (seeded weights, batch 32
of seeded 368 x 368 uint8 frames), alternating the modes in one process: frames/s per run of each mode, then per-launch
milliseconds and TFLOP/s of both plans from b200pose_net_profile (algorithmic FLOPs), with the card's name and power
limit read in the same call.  Prints a table and ONE JSON line.

  python tools/bench_modes.py [--modes bf16 fp16] [--runs R] [--steps K] [--warmup W] [--batch N]
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



def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--modes", nargs=2, default=["bf16", "fp8"], metavar=("BASE", "OTHER"),
                    help="the two modes to alternate; times are reported as OTHER / BASE")
    args = ap.parse_args()
    MODES = tuple(args.modes)
    base, other = MODES
    import torch
    _b200_alias.load_package()
    engine = importlib.import_module(_b200_alias.PKG + ".engine")
    nat = importlib.import_module(_b200_alias.PKG + "._native")
    syn = importlib.import_module(_b200_alias.PKG + ".synthetic")
    net = engine.NativeNet(0)
    net.load_state_dict_arrays(syn.he_state_arrays(1234))
    n, H, W = args.batch, 368, 368
    frames = torch.from_numpy(np.random.default_rng(0).integers(0, 256, (n, H, W, 3), dtype=np.uint8)).cuda()
    st = torch.cuda.Stream()

    def step(mode):
        net.forward_u8_ptr(frames.data_ptr(), True, n, H, W, nat.MODES[mode], [0] * 12, True, st.cuda_stream)

    fps = {m: [] for m in MODES}
    for m in MODES:
        for _ in range(args.warmup):
            step(m)
    st.synchronize()
    for _ in range(args.runs):
        for m in MODES:
            step(m)
            st.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.steps):
                step(m)
            st.synchronize()
            fps[m].append(n * args.steps / (time.perf_counter() - t0))
    prof = {}
    for m in MODES:
        step(m)
        st.synchronize()
        ms = np.zeros(64, np.float32)
        fl = np.zeros(64, np.float64)
        best = None
        for _ in range(5):     # per launch: the fastest of 5 profiled passes
            k = nat.lib().b200pose_net_profile(net._h, ms.ctypes.data, fl.ctypes.data, 64, st.cuda_stream)
            assert k > 0, nat.lib().b200pose_last_error()
            best = ms[:k].copy() if best is None else np.minimum(best, ms[:k])
        prof[m] = (best, fl[:len(best)].copy())
    name = card()
    print("%s; batch %d x %dx%d; %d runs x %d steps per mode, alternating" % (name, n, H, W, args.runs, args.steps))
    for m in MODES:
        print("  %-5s frames/s: %s" % (m, " ".join("%.1f" % v for v in fps[m])))
    print("launch  GFLOP  %6s ms  TFLOP/s  %6s ms  TFLOP/s  %s/%s time" % (base, other, other, base))
    for i in range(len(prof[base][0])):
        (mb, fb), m8 = (prof[base][0][i], prof[base][1][i]), prof[other][0][i]
        print("%6d  %6.1f  %9.3f  %7.1f  %9.3f  %7.1f  %6.3f" % (i, fb / 1e9, mb, fb / mb / 1e9, m8, fb / m8 / 1e9, m8 / mb))
    tot = {m: (float(prof[m][0].sum()), float(prof[m][1].sum())) for m in MODES}
    for m in MODES:
        print("  %-5s all launches: %.3f ms, %.1f TFLOP/s" % (m, tot[m][0], tot[m][1] / tot[m][0] / 1e9))
    print(json.dumps({"card": name, "batch": n, "fps": fps,
                      "profile_ms": {m: [round(float(v), 4) for v in prof[m][0]] for m in MODES},
                      "gflop": [round(float(v) / 1e9, 3) for v in prof[base][1]]}))


if __name__ == "__main__":
    main()
