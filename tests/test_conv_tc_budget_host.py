"""CPU: the resource budget of every conv_tc_kernel instantiation, from ptxas (`-Xptxas -v`) with the library's flags.

One CTA of conv_tc_kernel runs per SM, next to the previous batch's post-processing kernels (DESIGN.md §2.1, §2.4), so
the kernel must stay within 189 952 B of shared memory: two patch stages, the weight ring and the barriers.  No
instantiation may spill, and none may have its wgmma serialised by ptxas (C7520)."""
import os
import re
import subprocess
import sys
import tempfile

from conftest import ROOT

sys.path.insert(0, ROOT)
import __graft_entry__ as g  # noqa: E402

SMEM_LIMIT = 189952
NVCC = os.environ.get("NVCC", "nvcc")


def _ptxas_log():
    r = subprocess.run([NVCC] + g.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(g.CSRC, "conv_tc.cu"),
                                                 "-o", os.devnull],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:]
    return r.stdout


def _dynamic_smem_bytes():
    """kConvTcSmemBytes, the dynamic shared memory every launch of conv_tc_kernel asks for (conv_tc.cuh)."""
    with tempfile.TemporaryDirectory() as d:
        src, exe = os.path.join(d, "smem.cu"), os.path.join(d, "smem")
        with open(src, "w") as f:
            f.write('#include <cstdio>\n#include "conv_tc.cuh"\n'
                    'int main() { std::printf("%d\\n", b2p::kConvTcSmemBytes); return 0; }\n')
        r = subprocess.run([NVCC, "-std=c++17", "-I", g.CSRC, "-o", exe, src], stdout=subprocess.PIPE,
                           stderr=subprocess.STDOUT, text=True, timeout=300)
        assert r.returncode == 0, r.stdout[-2000:]
        out = subprocess.run([exe], stdout=subprocess.PIPE, text=True, timeout=60)
        assert out.returncode == 0
        return int(out.stdout.strip())


def test_every_conv_tc_kernel_fits_its_budget():
    log = _ptxas_log()
    bodies = re.findall(r"Compiling entry function '(\S+)' for 'sm_90a'(.*?)(?=Compiling entry|\Z)", log, re.S)
    kernels = [(fn, body) for fn, body in bodies if "conv_tc_kernel" in fn]
    assert len(kernels) == 42
    dyn = _dynamic_smem_bytes()
    print("dynamic shared memory per CTA: %d B (limit %d B)" % (dyn, SMEM_LIMIT))
    bad = []
    for fn, body in kernels:
        regs = re.search(r"Used (\d+) registers", body)
        static = re.search(r"(\d+) bytes smem", body)
        smem = dyn + (int(static.group(1)) if static else 0)
        print("%-110s %3s registers, %d B shared" % (fn, regs.group(1) if regs else "?", smem))
        if "0 bytes spill stores, 0 bytes spill loads" not in body:
            bad.append((fn, "spills"))
        if smem > SMEM_LIMIT:
            bad.append((fn, "%d B of shared memory" % smem))
    serialised = [line for line in log.splitlines() if "C7520" in line]
    assert not serialised, "ptxas serialised wgmma (C7520):\n" + "\n".join(serialised)
    assert not bad, bad
