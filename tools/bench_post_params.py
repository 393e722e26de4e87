#!/usr/bin/env python
"""Post-processing time per batch for each parameter set of oracle/post_params.SETS, on bench.py's person-like
workload (workload_alt: synthetic.person_maps, batch 32 of 46 x 46 maps = 368 x 368 frames, 8 schematic persons per
frame, resident on the device).  Only b200pose_post_run runs (peaks, limbs, assembly); the sets alternate in one process
for R rounds of K timed runs each (CUDA events around K runs that end in a sync).  Prints a table and ONE JSON line
with the card's name, power limit and max SM clock read in the same call.

  python tools/bench_post_params.py [--runs R] [--steps K] [--warmup W] [--batch N]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import _b200_alias  # noqa: E402
from oracle import post_params  # noqa: E402

ORDER = ("default", "strict", "loose", "single", "wide")


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=32)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_post_params: needs a CUDA device")
    _b200_alias.load_package()
    eng = importlib.import_module(_b200_alias.PKG + ".engine")
    syn = importlib.import_module(_b200_alias.PKG + ".synthetic")
    n = args.batch
    heat, paf = syn.person_maps(n, 8, seed=7)
    h, w = heat.shape[2], heat.shape[3]
    d_heat, d_paf = torch.from_numpy(heat).cuda(), torch.from_numpy(paf).cuda()
    post = eng.NativePost(0, batch_cap=n)
    stream = torch.cuda.current_stream()
    sptr = stream.cuda_stream
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()

    def run():
        post.run(d_heat.data_ptr(), d_paf.data_ptr(), True, 0, n, h, w, 0.1, sptr)

    ms = {s: [] for s in ORDER}
    persons, status = {}, {}
    for r in range(args.runs):
        for s in ORDER:
            post.set_params(**post_params.params_of(s))
            for _ in range(args.warmup):
                run()
            post.sync()
            post.status_accum(reset=True)
            e0.record(stream)
            for _ in range(args.steps):
                run()
            post.sync()
            e1.record(stream)
            torch.cuda.synchronize()
            ms[s].append(e0.elapsed_time(e1) / args.steps)
            persons[s] = sum(len(post.humans(i)) for i in range(n)) / n
            status[s] = post.status_accum(reset=True)
    rec = {"card": card(), "batch": n, "maps": [h, w], "runs": args.runs, "steps": args.steps, "sets": {}}
    print("%-8s %8s %8s %8s %9s %7s  %s" % ("set", "min ms", "median", "max ms", "persons/f", "status", "params"))
    for s in ORDER:
        v = np.array(ms[s])
        rec["sets"][s] = {"ms_per_batch_min": round(float(v.min()), 4), "ms_per_batch_median": round(float(np.median(v)), 4),
                          "ms_per_batch_max": round(float(v.max()), 4), "persons_per_frame": round(persons[s], 2),
                          "status_bits": status[s], "params": post_params.params_of(s)}
        print("%-8s %8.3f %8.3f %8.3f %9.2f %7d  %s" % (s, v.min(), np.median(v), v.max(), persons[s], status[s],
                                                       post_params.SETS[s]))
    print(rec["card"])
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
