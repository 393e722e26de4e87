#!/usr/bin/env python
"""Per-kernel SASS fingerprints of a built library: `python tools/sass_hash.py [--mask-params] [lib.so] > a.txt`, diff
two outputs to prove that a change (a refactor, a new entry point, code behind a compile-time switch) left the machine
code of the kernels that were validated on the GPU untouched.

--mask-params hashes the instruction text only (not the encoding column), replaces every c[0x0][...] operand with
c[0x0][P] and names the anonymous namespace `_GLOBAL__N_1` whatever path the file was compiled from.  A change to a kernel's
parameter struct moves the parameter offsets of every kernel that takes it; with the mask, kernels whose instructions are
otherwise the same hash the same.  Compare such outputs as multisets of hashes when kernel names change too."""
import argparse
import hashlib
import os
import re
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ap = argparse.ArgumentParser()
ap.add_argument("lib", nargs="?", default=os.path.join(ROOT, "pytorch_realtime_multi-person_pose_estimation_b200",
                                                       "libb200pose.so"))
ap.add_argument("--mask-params", action="store_true")
args = ap.parse_args()
out = subprocess.run(["cuobjdump", "-sass", args.lib], stdout=subprocess.PIPE, text=True, check=True).stdout
cur, table = None, {}
for line in out.splitlines():
    m = re.match(r"\s*Function : (\S+)", line)
    if m:
        cur = m.group(1)
        if args.mask_params:
            cur = re.sub(r"\d+_GLOBAL__N__[0-9a-f]+_\d+_\w+?_[0-9a-f]{8}", "12_GLOBAL__N_1", cur)
        table[cur] = hashlib.md5()
    elif cur and line.strip().startswith("/*"):      # instruction lines only
        if args.mask_params:
            line = re.sub(r"/\*\s*0x[0-9a-f]+\s*\*/", "", line)      # the encoding column
            line = re.sub(r"c\[0x0\]\[0x[0-9a-f]+\]", "c[0x0][P]", line)
            if not line.strip():
                continue
        table[cur].update(" ".join(line.split()).encode())      # column alignment varies with the widest line
for k in sorted(table):
    print(table[k].hexdigest()[:12], k)
