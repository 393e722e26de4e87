#!/usr/bin/env python
"""Build compile-time tuning variants of libb200pose.so HERE (nvcc cross-compiles without a GPU) so that a GPU run only
measures:  python tools/variants.py build [name ...]   -> build/variants/libb200pose_<name>.so
           bash tools/run_variants.sh [name ...]       -> (on an H100) parity subset + bench line per variant
           python tools/variants.py report             -> table from build/variants/*.json
Each variant is the unmodified source with -D switches; `base` is the default build (its SASS equals the in-tree
library's, tools/sass_hash.py).  B200POSE_LIB=<path> makes the Python layer load a variant."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as g  # noqa: E402

VARIANTS = {
    "base": [],
    "bstages4": ["-DB2P_CONV_B_STAGES=4"],          # conv: 64 KB weight ring
    "range2048": ["-DB2P_LIMB_SMEM_RANGE=2048"],    # sort ranges of 2048 keys: 26 KB of shared memory, fits next to a conv CTA
    "lane32": ["-DB2P_LANE_SORT_KEYS=32"],          # one-lane partitions only below 33 keys
    "lane128": ["-DB2P_LANE_SORT_KEYS=128"],
    "peaks128": ["-DB2P_PEAK_THREADS=128"],         # 128-thread peak blocks (16 K registers: fit next to a conv CTA)
    "bstages3": ["-DB2P_CONV_B_STAGES=3"],          # conv: 48 KB weight ring
    "gather256": ["-DB2P_GATHER_THREADS=256"],      # 256-thread gather blocks (16 K registers)
    "fit": ["-DB2P_GATHER_THREADS=256", "-DB2P_PEAK_THREADS=128"],
    # conv weight ring (default: 96 KB, >= 3 stages -> N=128: 2 taps per stage, 3 stages)
    "ring96min6": ["-DB2P_CONV_MIN_B_STAGES=6"],                          # N=128: 1 tap per stage, 6 stages
    "ring96min2": ["-DB2P_CONV_MIN_B_STAGES=2"],                          # N=128: 3 taps per stage, 2 stages
}


def build(names):
    out_dir = os.path.join(ROOT, "build", "variants")
    os.makedirs(out_dir, exist_ok=True)
    srcs = [os.path.join(g.CSRC, s) for s in g.LIB_SOURCES]
    for name in names:
        lib = os.path.join(out_dir, "libb200pose_%s.so" % name)
        cmd = ([os.environ.get("NVCC", "nvcc")] + g.NVCC_FLAGS + VARIANTS[name]
               + ["-shared", "-Xcompiler", "-fPIC", "-o", lib] + srcs)
        r = subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        print("%-12s %s" % (name, "ok" if r.returncode == 0 else "FAILED\n" + r.stdout[-2000:]))


def report():
    d = os.path.join(ROOT, "build", "variants")
    for f in sorted(os.listdir(d)):
        if not f.endswith(".json"):
            continue
        try:
            line = [l for l in open(os.path.join(d, f)) if l.startswith("{")][-1]
            j = json.loads(line)
            print("%-12s %8.1f frames/s  e2e %8.1f  %.3f ms/step  conv frac %.3f" % (
                f[:-5], j["value"], j["e2e"]["value"], j["ms_per_step"], j["roofline"]["frac"]))
        except Exception as e:      # a variant that failed to run is part of the result
            print("%-12s no bench line (%s)" % (f[:-5], e))


if __name__ == "__main__":
    if len(sys.argv) >= 2 and sys.argv[1] == "build":
        build(sys.argv[2:] or list(VARIANTS))
    elif len(sys.argv) >= 2 and sys.argv[1] == "report":
        report()
    else:
        raise SystemExit(__doc__)
