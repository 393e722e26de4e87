#!/usr/bin/env python
"""Post-processing time per batch for each peak refinement mode (cubic, gauss, none) and up-sampling factor (4, 8, 16)
of standalone runs (b200pose_post_run_scaled), on bench.py's person-like workload (workload_alt: synthetic.person_maps,
batch 32 of 46 x 46 maps = 368 x 368 frames, 8 schematic persons per frame, resident on the device).  The settings
alternate in one process for R rounds of K timed runs each (CUDA events around K runs that end in a sync).  Prints a
table and ONE JSON line with the card's name, power limit and max SM clock read in the same call.

  python tools/bench_refine.py [--runs R] [--steps K] [--warmup W] [--batch N]
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

MODES = ("cubic", "gauss", "none")
FACTORS = (4, 8, 16)


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
        raise SystemExit("bench_refine: needs a CUDA device")
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
    keys = [(m, f) for f in FACTORS for m in MODES]
    ms = {k: [] for k in keys}
    persons, status = {}, {}
    for r in range(args.runs):
        for mode, f in keys:
            post.set_refine(mode)
            for _ in range(args.warmup):
                post.run(d_heat.data_ptr(), d_paf.data_ptr(), True, 0, n, h, w, 0.1, sptr, upsample=f)
            post.sync()
            post.status_accum(reset=True)
            e0.record(stream)
            for _ in range(args.steps):
                post.run(d_heat.data_ptr(), d_paf.data_ptr(), True, 0, n, h, w, 0.1, sptr, upsample=f)
            post.sync()
            e1.record(stream)
            torch.cuda.synchronize()
            ms[(mode, f)].append(e0.elapsed_time(e1) / args.steps)
            persons[(mode, f)] = sum(len(post.humans(i)) for i in range(n)) / n
            status[(mode, f)] = post.status_accum(reset=True)
    rec = {"card": card(), "batch": n, "maps": [h, w], "runs": args.runs, "steps": args.steps, "settings": {}}
    print("%-6s %3s %8s %8s %8s %9s %7s" % ("mode", "f", "min ms", "median", "max ms", "persons/f", "status"))
    for mode, f in keys:
        v = np.array(ms[(mode, f)])
        rec["settings"]["%s_f%d" % (mode, f)] = {
            "ms_per_batch_min": round(float(v.min()), 4), "ms_per_batch_median": round(float(np.median(v)), 4),
            "ms_per_batch_max": round(float(v.max()), 4), "persons_per_frame": round(persons[(mode, f)], 2),
            "status_bits": status[(mode, f)]}
        print("%-6s %3d %8.3f %8.3f %8.3f %9.2f %7d" % (mode, f, v.min(), np.median(v), v.max(), persons[(mode, f)],
                                                       status[(mode, f)]))
    print(rec["card"])
    print(json.dumps(rec))


if __name__ == "__main__":
    main()
