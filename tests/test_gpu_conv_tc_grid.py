"""GPU (-m gpu): conv_tc_kernel launched directly, every instantiation, at tile edges and at every grid size
(`build/test_conv_tc matrix`, tests/cuda/test_conv_tc.cu).

Each case of the harness's table runs with exact-integer operands, whose every stored word, residual word, fp32 map
element and amax / ea / overflow entry is known exactly, and (fp8 aside) with random operands under the interval rule
of its format.  Each runs at grid sizes 1, 2, 3, 7, S - 1, S and 2 S (S = SM count, clamped to the tile count): the run
at S is checked against the reference and every other run must equal it bit for bit, sentinels around every output
buffer included.  So a tile-schedule or persistent-loop bug (accumulator, residual sum, fp8 scale or ring state carried
from a CTA's previous tile) fails here even where the one grid size the library launches hides it.
tests/test_conv_tc_grid_host.py checks that the table covers every instantiation ptxas reports."""
import os
import re
import subprocess
import time

import pytest

from conftest import ROOT

pytestmark = pytest.mark.gpu

WORST = re.compile(r"^worst (\S+) (\d+) (uniform|ragged)( prelu)? : max\|v-r\|/e ([\d.]+) f32 ([\d.]+)$", re.M)


def test_every_instantiation_at_every_grid_size(built):
    exe = os.path.join(ROOT, "build", "test_conv_tc")
    t0 = time.time()
    r = subprocess.run([exe, "matrix"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    print(r.stdout)
    print("matrix run: %.1f s" % (time.time() - t0))
    m = re.search(r"^conv_tc matrix: (\d+) cases, (\d+) case-modes, ALL OK$", r.stdout, re.M)
    assert r.returncode == 0 and m, r.stdout[-3000:]
    listed = subprocess.run([exe, "list"], stdout=subprocess.PIPE, text=True, check=True).stdout.split("\n")
    cases = [tuple(line.split()[1:]) for line in listed if line.startswith("case ")]
    assert int(m.group(1)) == len(cases)
    # one OK line per case and operand mode: exact for every case, random for all but fp8
    assert len(re.findall(r"^case .* OK$", r.stdout, re.M)) == int(m.group(2)) == 2 * len(cases) - sum(
        c[0] == "fp8" for c in cases)
    # the worst |v - r| / e of the random operands, per instantiation: every non-fp8 one is reported
    worst = {(f, n, rg == "ragged", bool(pr)): (float(a), float(b)) for f, n, rg, pr, a, b in WORST.findall(r.stdout)}
    want = {(f, n, rg == "1", pr == "1") for f, n, rg, pr in cases if f != "fp8"}
    assert set(worst) == want
    for key in sorted(worst):
        print("conv_tc_kernel<%s, %s, ragged=%s, prelu=%s>: max|v-r|/e %.3f, fp32 maps %.3f" % (key + worst[key]))
