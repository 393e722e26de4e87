"""CPU: every conv_tc_kernel instantiation is a case of the standalone matrix (`build/test_conv_tc matrix`, run by
tests/test_gpu_conv_tc_grid.py).

`build/test_conv_tc list` prints each case's (format, N, ragged, PReLU) without touching a GPU.  That set must equal
the kernels ptxas reports for conv_tc.cu, so a new instantiation without a case in the harness fails on the CPU."""
import os
import subprocess

from conftest import ROOT
from test_conv_tc_matrix_host import decode
from test_fp8_host import _ptxas


def test_every_conv_tc_kernel_is_a_case_of_the_standalone_matrix(built):
    out = subprocess.run([os.path.join(ROOT, "build", "test_conv_tc"), "list"], stdout=subprocess.PIPE,
                         stderr=subprocess.STDOUT, text=True, timeout=60)
    assert out.returncode == 0, out.stdout
    table = set()
    for line in out.stdout.splitlines():
        fmt, n, ragged, prelu = line.split()[1:]
        table.add((fmt, int(n), ragged == "1", prelu == "1"))
    compiled = decode([fn for fn, _ in _ptxas("conv_tc.cu") if "conv_tc_kernel" in fn])
    assert len(set(compiled)) == len(compiled) == 42
    print("%d instantiations, %d with a case of the matrix" % (len(compiled), len(table & set(compiled))))
    assert not sorted(set(compiled) - table), "instantiations without a matrix case: %s" % sorted(set(compiled) - table)
    assert not sorted(table - set(compiled)), "matrix cases of no instantiation: %s" % sorted(table - set(compiled))
