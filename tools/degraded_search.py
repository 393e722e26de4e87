#!/usr/bin/env python
"""Searches seeded scenarios for one that makes the person assembly fall back to its full-scan row lookup (a peak held
by more than kListCap = 4 alive rows: `Assembler::degraded`, status bit 16), on the CPU through the host build of
csrc/post_core.h (build/libpostcore_host.so, made by `__graft_entry__.build()`).

  python tools/degraded_search.py [--fuzz N] [--fuzz-seed S] [--heat N] [--heat-seed S]

--fuzz: joint-list scenarios of oracle/synth.fuzz_field / fuzz_persons (seeds S .. S+N-1, fast);
--heat: heat-map scenarios of every oracle/synth.edge_maps kind at 46x46 through nms_port (N seeds per kind from S,
about 1.5 s each).  Prints every seed that degrades and the totals."""
import argparse
import ctypes
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import nms_port, synth  # noqa: E402

FP = ctypes.POINTER(ctypes.c_float)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--fuzz", type=int, default=10166)
    ap.add_argument("--fuzz-seed", type=int, default=50000)
    ap.add_argument("--heat", type=int, default=0)
    ap.add_argument("--heat-seed", type=int, default=1000)
    a = ap.parse_args()
    lib = ctypes.CDLL(os.path.join(ROOT, "build", "libpostcore_host.so"))
    lib.core_process.argtypes = [ctypes.c_int, FP, ctypes.c_int, FP, ctypes.c_long, ctypes.c_long, ctypes.c_long,
                                 ctypes.c_int, ctypes.c_int]

    def degraded(jl, paf, h, w):
        if len(jl) == 0:
            return False
        jl, paf = np.ascontiguousarray(jl), np.ascontiguousarray(paf)
        lib.core_process(len(jl), jl.ctypes.data_as(FP), h * 8, paf.ctypes.data_as(FP), 1, w * 38, 38, 3, 0)
        return bool(lib.core_degraded())

    found = []
    for seed in range(a.fuzz_seed, a.fuzz_seed + a.fuzz):
        rs = np.random.RandomState(seed)
        h, w = int(rs.choice([12, 23, 46])), int(rs.choice([23, 46, 53]))
        if seed % 2:
            h = max(h, 23)
            jl, paf = synth.fuzz_persons(rs, h, w)
        else:
            jl, paf = synth.fuzz_field(rs, h, w, ("uniform", "cluster", "ties")[(seed // 2) % 3])
        if degraded(jl, paf, h, w):
            found.append(("fuzz", seed))
            print("degraded: fuzz seed", seed, flush=True)
    for kind in synth.EDGE_KINDS:
        for seed in range(a.heat_seed, a.heat_seed + a.heat):
            heat, paf = synth.edge_maps(kind, seed, 46, 46)
            if degraded(nms_port.joint_list_from_nms(nms_port.nms(heat, 0.1)), paf, 46, 46):
                found.append((kind, seed))
                print("degraded: edge_maps", kind, seed, flush=True)
    print("searched %d fuzz scenarios (seeds %d..%d) and %d heat maps (%d per kind from seed %d): %d degrade"
          % (a.fuzz, a.fuzz_seed, a.fuzz_seed + a.fuzz - 1, a.heat * len(synth.EDGE_KINDS), a.heat, a.heat_seed,
             len(found)))


if __name__ == "__main__":
    main()
