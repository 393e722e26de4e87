"""CPU: the fp8 (e4m3) mode's host side (DESIGN.md §2.3) - the weight quantiser and the scale exponent rule of
csrc/fp8_core.h built for the host, the K order of the fp8 A fragments, the C ABI surface, and no spills in the new
kernels."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import fp8_check
from conftest import ROOT, pkg_module
from oracle import conv_check

CSRC = os.path.join(ROOT, "pytorch_realtime_multi-person_pose_estimation_b200", "csrc")


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("fp8") / "libfp8core.so")
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-o", so,
                    os.path.join(ROOT, "tests", "cuda", "fp8_host.cpp")], check=True)
    lib = ctypes.CDLL(so)
    lib.core_e4m3_rn.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_long]
    lib.core_fp8_exp.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_long]
    return lib


def test_host_e4m3_quantiser_equals_torch_on_every_bf16_in_range(core):
    """Every finite bf16 bit pattern in [-448, 448], subnormals included: the packer's e4m3 byte equals
    torch.float8_e4m3fn's."""
    _, f = fp8_check.e4m3_all_bf16_in_range()
    got = np.empty(f.shape, np.uint8)
    core.core_e4m3_rn(f.ctypes.data, got.ctypes.data, f.size)
    want = torch.from_numpy(f).to(torch.float8_e4m3fn).view(torch.uint8).numpy()
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, [(float(f[i]), int(got[i]), int(want[i])) for i in bad[:8]]
    assert f.size > 30000 and np.any(np.abs(f) < 2.0 ** -6) and np.any(f == 448.0)


def _exps(core, vals):
    bits = np.asarray(vals, np.float32).view(np.uint32)
    out = np.empty(bits.shape, np.int32)
    core.core_fp8_exp(bits.ctypes.data, out.ctypes.data, bits.size)
    return out.tolist()


def test_exponent_rule_edges(core):
    """ea = floor(log2(448 / amax)): powers of two, exactly 448, just above / below 1.75 * 2^k, 0, denormals, the
    clamp; every value keeps amax * 2^ea <= 448 < amax * 2^(ea + 1) inside the clamp."""
    tiny = np.float32(np.finfo(np.float32).tiny)
    cases = {1.0: 8, 2.0: 7, 0.5: 9, 448.0: 0, 449.0: -1, 224.0: 1, 1.75: 8, 1.7500001: 7, 1.7499999: 8, 0.0: 0,
             float(tiny): 63, float(tiny / 4): 63, 1e-30: 63, 3e38: -63, 2.0 ** -54: 62, 2.0 ** -55: 63, 2.0 ** -56: 63}
    got = _exps(core, list(cases))
    for (a, want), g in zip(cases.items(), got):
        assert g == want == fp8_check.exp_rule(np.float32(a)), (a, g, want)
    rs = np.random.RandomState(0)
    vals = np.concatenate([np.float32(2.0) ** rs.randint(-60, 60, 2000) * rs.uniform(1, 2, 2000).astype(np.float32),
                           rs.uniform(0, 500, 2000).astype(np.float32)]).astype(np.float32)
    for a, g in zip(vals, _exps(core, vals)):
        assert g == fp8_check.exp_rule(a), (a, g)
        if -63 < g < 63:
            assert float(a) * 2.0 ** g <= 448.0 < float(a) * 2.0 ** (g + 1)


def test_fp8_k_order_is_a_permutation_matching_the_bf16_fragments(core):
    """Byte j of fp8 A register 0 of lane q holds K index 4q + j: the bf16 k16 fragments hold row r's channels
    2q, 2q + 1 (register 0) and 2q + 8, 2q + 9 (register 2); K indices 16 .. 31 repeat this on the second k16 step."""
    perm = [core.core_k_to_channel(k) for k in range(32)]
    assert sorted(perm) == list(range(32))
    for q in range(4):
        assert perm[4 * q: 4 * q + 4] == [2 * q, 2 * q + 1, 2 * q + 8, 2 * q + 9]
        assert perm[16 + 4 * q: 20 + 4 * q] == [16 + 2 * q, 17 + 2 * q, 24 + 2 * q, 25 + 2 * q]


def test_fp8_abi_surface(built):
    nat = pkg_module("_native")
    with open(os.path.join(ROOT, "include", "b200pose.h")) as f:
        header = f.read()
    assert re.search(r"#define B200POSE_MODE_FP8 3\b", header)
    assert "int b200pose_net_debug_fp8(b200pose_net* net, int launch, int* act_exp, int n_img, int* w_exp, int cap);" in header
    assert "#define B200POSE_DEBUG_LAUNCH_FIELDS 27" in header
    assert nat.MODES["fp8"] == nat.MODE_FP8 == 3
    assert {"bf16", "bf16x3", "fp32"} <= set(nat.MODES) and nat.MODES["bf16"] == 0
    assert "b200pose_net_debug_fp8" in nat.EXPORTED
    lib = nat.lib()
    assert lib.b200pose_net_debug_fp8(None, 1, None, 0, None, 0) < 0
    assert b"fp8" in lib.b200pose_last_error()


def _ptxas(src):
    r = subprocess.run([os.environ.get("NVCC", "nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "-Xptxas", "-v", "-c", os.path.join(CSRC, src), "-o", os.devnull],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:]
    return re.findall(r"Compiling entry function '(\S+)' for 'sm_90a'(.*?)(?=Compiling entry|\Z)", r.stdout, re.S)


@pytest.mark.parametrize("src,name,count", [("conv_tc.cu", "conv_tc_kernelILNS_8TcFormatE2E", 6),      # TcFormat::kFp8
                                            ("conv_misc.cu", "conv_first_mma_kernelILi.ELNS_8TcFormatE2E", 5)])
def test_fp8_kernels_do_not_spill(built, src, name, count):
    bodies = [(fn, body) for fn, body in _ptxas(src) if re.search(name, fn)]
    assert len(bodies) == count
    for fn, body in bodies:
        assert "0 bytes spill stores, 0 bytes spill loads" in body, (fn, body)


MUTATIONS = ["ea", "ew", "slice", "shift", "per_tensor", "bias"]
# mutations the bound cannot see at a shape (see the test's docstring)
INVISIBLE = {(1, 64): {"per_tensor"}, (3, 128): {"per_tensor"}, (7, 128): {"per_tensor"}, (7, 192): {"per_tensor"}}


def _emulation_case(ks, cin, seed):
    """One image, ks x ks over `cin` channels of ReLU-like activations, 8 output channels of Gaussian weights."""
    g = torch.Generator().manual_seed(seed)
    x = torch.relu(torch.randn((1, cin, 12, 12), generator=g)).to(torch.float32)
    x = conv_check.bf16_round(x.double())
    w = (torch.randn((8, cin, ks, ks), generator=g) * 0.05).to(torch.float32)
    w[3] *= 1e-5                                          # a row far below the others: beyond e4m3's range of one scale
    b = (torch.randn(8, generator=g) * 0.5).to(torch.float32).double()
    ea = fp8_check.exp_rule(float(x.abs().max()))
    qw, ew = fp8_check.quantise_weights(w)
    r, S = fp8_check.reference(fp8_check.quantise(x, ea), ea, qw, ew, b, ks)
    e = fp8_check.bound_coef(ks, cin) * S
    return x, ea, qw, ew, b, r, e


def _ratio(got, r, e):
    v = conv_check.check_bf16(conv_check.bf16_round(got), r, e)
    return bool(v.ok.all()), v.ratio


@pytest.mark.parametrize("ks,cin", [(1, 64), (3, 128), (7, 128), (7, 192)])
def test_checker_accepts_the_emulated_kernel_and_rejects_mutations(ks, cin):
    """The float64 interval of tests/fp8_check.py accepts the host emulation of the fp8 conv_tc_kernel at the characterised
    accumulator precision (ACC_BITS, measured by build/test_conv_fp8 acc) and rejects a descale by ea + 1, one
    channel's ew off by one, a dropped k32 slice, a tap read one pixel off and a scaled bias at every shape here.  One
    mutation stays below the bound and the test states it: weights quantised with one scale per tensor.  It changes only
    the row whose weights are far below the others', whose output is then dominated by its bias, and |b| is part of the
    interval's S; the per-launch GPU check compares ew per row with the rule instead."""
    x, ea, qw, ew, b, r, e = _emulation_case(ks, cin, 7 * ks + cin)
    ok, ratio = _ratio(fp8_check.emulate(x, ea, qw, ew, b, ks), r, e)
    assert ok, ratio
    seen = {}
    for m in MUTATIONS:
        ok_m, ratio_m = _ratio(fp8_check.emulate(x, ea, qw, ew, b, ks, mutate=m), r, e)
        seen[m] = not ok_m
        print("%dx%d over %d channels: emulation %.3f of e; mutation %-10s %s (%.2f of e)"
              % (ks, ks, cin, ratio, m, "rejected" if not ok_m else "NOT visible", ratio_m))
    invisible = {m for m, v in seen.items() if not v}
    assert invisible == INVISIBLE[(ks, cin)], invisible
