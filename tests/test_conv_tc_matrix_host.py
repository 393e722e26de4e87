"""CPU: every conv_tc_kernel instantiation is a case of tests/test_gpu_conv_tc_matrix.py.

ptxas lists the kernels csrc/conv_tc.cu instantiates; each decodes to (format, N, ragged, PReLU) and the set must equal
the GPU matrix's case table, so that a new instantiation cannot go unchecked and a row cannot go missing."""
import re

from test_conv1_1_host import TC_FORMATS
from test_fp8_host import _ptxas
from test_gpu_conv_tc_matrix import CASES

ENTRY = re.compile(r"conv_tc_kernelILNS_8TcFormatE(\d+)ELi(\d+)ELb([01])ELb([01])EE")


def decode(names):
    """(format, N, ragged, PReLU) of each conv_tc_kernel entry ptxas compiled."""
    cases = []
    for fn in names:
        m = ENTRY.search(fn)
        assert m, fn
        fmt, n, ragged, prelu = m.groups()
        cases.append((TC_FORMATS[int(fmt)], int(n), ragged == "1", prelu == "1"))
    return cases


def test_every_conv_tc_kernel_is_a_case_of_the_gpu_matrix():
    names = [fn for fn, _ in _ptxas("conv_tc.cu") if "conv_tc_kernel" in fn]
    compiled = decode(names)
    print("%d conv_tc_kernel instantiations:" % len(compiled))
    for c in sorted(compiled):
        print("  conv_tc_kernel<%s, %d, ragged=%s, prelu=%s>" % c)
    assert len(set(compiled)) == len(compiled) == 42
    table = [c[:4] for c in CASES]
    assert len(set(table)) == len(table), "a case is listed twice"
    missing = sorted(set(compiled) - set(table))
    assert not missing, "instantiations without a case of the GPU matrix: %s" % missing
    extra = sorted(set(table) - set(compiled))
    assert not extra, "cases of the GPU matrix that no instantiation has: %s" % extra
