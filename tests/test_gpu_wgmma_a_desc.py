"""GPU (-m gpu): the wgmma A-operand descriptor rule of conv_tc_kernel (tests/cuda/test_wgmma_a_desc.cu)."""
import os
import subprocess

import pytest

from conftest import ROOT

pytestmark = pytest.mark.gpu


def test_patch_window_descriptor_equals_ldmatrix_fragments(built):
    """One tap at each dx of 0..6, with A read through a descriptor that starts dx pixels past a 1024-B boundary of the
    SWIZZLE_128B patch (base offset 0, as conv_tc_kernel builds it), is bit-identical to the same tap with ldmatrix
    fragments in registers, and those match a float64 reference."""
    r = subprocess.run([os.path.join(ROOT, "build", "test_wgmma_a_desc")], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=120)
    print(r.stdout)
    assert r.returncode == 0 and "ALL OK" in r.stdout
