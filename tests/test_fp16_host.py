"""CPU: the fp16 (IEEE binary16) mode's host side (DESIGN.md §2.3) - the weight packer's rounding built for the host, the
float64 rounding R16 of the per-launch checker on a brute-force set, the checker's power to reject the faults the bf16
checker rejects (on a CPU emulation of the kernel), the C ABI surface, and no spills in the new kernels."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest
import torch

import fp16_check
from conftest import ROOT, pkg_module
from oracle import conv_check
from test_oracle import _emulate_tc, _layer

CSRC = os.path.join(ROOT, "pytorch_realtime_multi-person_pose_estimation_b200", "csrc")


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("f16") / "libf16core.so")
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-o", so,
                    os.path.join(ROOT, "tests", "cuda", "f16_host.cpp")], check=True)
    lib = ctypes.CDLL(so)
    lib.core_f16_rn.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_long]
    return lib


def _f16_bits(core, f):
    f = np.ascontiguousarray(f, np.float32)
    out = np.empty(f.shape, np.uint16)
    core.core_f16_rn(f.ctypes.data, out.ctypes.data, f.size)
    return out


def _edge_floats():
    """Every binary16 value, the float32 midpoints between neighbours and one float32 ulp either side of each, both
    signs; the overflow threshold; NaN and inf."""
    h = np.arange(0, 0x7C00, dtype=np.uint16).view(np.float16).astype(np.float64)      # 0 .. 65504
    nxt = np.append(h[1:], 65536.0)
    mid = ((h + nxt) / 2).astype(np.float32)          # exact in float32 (12 significant bits)
    below = np.nextafter(mid, np.float32(0))
    above = np.nextafter(mid, np.float32(np.inf))
    pos = np.concatenate([h.astype(np.float32), mid, below, above,
                          np.float32([65519.99, 65520.0, 65536.0, 1e9, 3.4e38, 2.0 ** -25, 2.0 ** -26, 1e-30])])
    return np.concatenate([pos, -pos, np.float32([np.inf, -np.inf])])


def test_host_packer_rounding_equals_numpy_on_the_edges_and_every_weight(core, he_sd):
    """The packer's binary16 bits equal numpy's float32 -> float16 cast (one rounding) on every binary16 value, every
    midpoint and its float32 neighbours, the overflow threshold (65519.99 -> 65504, 65520 -> inf), and on every weight
    of the He state dict."""
    f = _edge_floats()
    got = _f16_bits(core, f)
    want = f.astype(np.float16).view(np.uint16)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, [(float(f[i]), hex(got[i]), hex(want[i])) for i in bad[:8]]
    assert _f16_bits(core, np.float32([65519.99]))[0] == 0x7BFF and _f16_bits(core, np.float32([65520.0]))[0] == 0x7C00
    nan = _f16_bits(core, np.float32([np.nan]))[0]
    assert (nan & 0x7C00) == 0x7C00 and (nan & 0x3FF) != 0
    w = np.concatenate([v.numpy().ravel() for k, v in he_sd.items() if k.endswith(".weight")]).astype(np.float32)
    assert np.array_equal(_f16_bits(core, w), w.astype(np.float16).view(np.uint16))


def test_r16_is_one_rounding_from_float64():
    """R16 of the checker on float64 values: every binary16 value is a fixed point, the float64 midpoints tie to even,
    one float64 ulp either side rounds away from the tie (a float64 -> float32 -> float16 cast gets some of these
    wrong), subnormals round on the 2^-24 grid, and the overflow threshold is 65520."""
    h = np.arange(0, 0x7C00, dtype=np.uint16).view(np.float16).astype(np.float64)
    nxt = np.append(h[1:], 65536.0)
    t = lambda a: torch.from_numpy(np.asarray(a, np.float64))       # noqa: E731
    assert torch.equal(fp16_check.f16_round(t(h)), t(h))
    assert torch.equal(fp16_check.f16_round(t(-h)), t(-h))
    mid = (h + nxt) / 2
    even = np.where((np.arange(h.size) & 1) == 0, h, nxt)          # of h, nxt: the one with an even mantissa
    even = np.where(nxt == 65536.0, np.inf, even)                  # 65520 ties to the even inf
    assert torch.equal(fp16_check.f16_round(t(mid)), t(even))
    down, up = np.nextafter(mid, 0), np.nextafter(mid, np.inf)
    assert torch.equal(fp16_check.f16_round(t(down)), t(h))
    want_up = np.where(nxt == 65536.0, np.inf, nxt)
    assert torch.equal(fp16_check.f16_round(t(up)), t(want_up))
    # double rounding would fail here: just above a midpoint by less than half a float32 ulp
    x = mid[1000:1010] + np.spacing(mid[1000:1010]) * 4
    assert not np.array_equal(x.astype(np.float32).astype(np.float16).astype(np.float64), nxt[1000:1010])
    assert torch.equal(fp16_check.f16_round(t(x)), t(nxt[1000:1010]))
    specials = t([65519.99, 65520.0, -65520.0, 1e300, 2.0 ** -25, 2.0 ** -25 * 1.0000001, 3 * 2.0 ** -25, 0.0])
    assert fp16_check.f16_round(specials).tolist() == [65504.0, np.inf, -np.inf, np.inf, 0.0, 2.0 ** -24,
                                                       2.0 ** -23, 0.0]
    assert torch.isnan(fp16_check.f16_round(t([np.nan])))[0]


def _f16_layer(kind, seed):
    """test_oracle's layers with binary16 operands: activations and weights rounded to binary16 once."""
    x, _, w, b, ks, relu, pool, phys = _layer(kind, seed)
    x16 = fp16_check.f16_round(torch.from_numpy(x.astype(np.float64))).numpy().astype(np.float32)
    return x16, w, b, ks, relu, pool, phys


def _check16(x, w, b, ks, relu, pool, phys, got):
    C = x.shape[3]
    wp = torch.zeros((w.shape[0], C, ks, ks), dtype=torch.float64)
    wp[:, torch.from_numpy(phys)] = fp16_check.round_weights(w)
    xt = torch.from_numpy(x.astype(np.float64)).permute(0, 3, 1, 2)
    r, S = conv_check.reference(xt, wp, torch.from_numpy(b.astype(np.float64)), ks)
    e = conv_check.U * conv_check.bound_coef(ks, C) * S
    return fp16_check.check_f16(got, r, e, relu, pool)


@pytest.mark.parametrize("kind", ["mconv1", "trunk"])
def test_fp16_checker_accepts_the_kernel_arithmetic_and_rejects_each_mutation(kind):
    """The fp16 interval accepts the kernel's fp32 accumulation emulated on binary16 operands and rejects the mutations
    the bf16 checker rejects: a dropped k16 slice, a tap one pixel off, a neighbour's bias, a wrong partial-tile column,
    two channels swapped and (pooled layer) the wrong pool neighbour."""
    x, w, b, ks, relu, pool, phys = _f16_layer(kind, 7)
    wp = np.zeros((w.shape[0], x.shape[3], ks, ks))
    wp[:, phys] = fp16_check.round_weights(w).numpy()

    def out16(v):
        return fp16_check.f16_round(conv_check.f_act(v, relu, pool))

    v = _emulate_tc(x, wp, b, ks, relu, pool)
    ok = _check16(x, w, b, ks, relu, pool, phys, out16(v))
    print("%s fp16: emulated kernel accepted, max |v - r| / e = %.3f" % (kind, ok.ratio))
    assert bool(ok.ok.all()), conv_check.describe(ok, out16(v), kind, pool)
    mutants = {
        "k16 slice of one tap dropped": _emulate_tc(x, wp, b, ks, relu, pool, skip=(1, ks * ks // 2 + 1, 2)),
        "one tap read one pixel off": _emulate_tc(x, wp, b, ks, relu, pool, shift=ks * ks - 1),
        "neighbour's bias": _emulate_tc(x, wp, b, ks, relu, pool, bias_roll=1),
    }
    last = v.clone()
    last[..., -1] = v[..., -2]
    mutants["last partial tile column wrong"] = last
    swapped = v.clone()
    swapped[:, [5, 6]] = v[:, [6, 5]]
    mutants["two channels of an n-tile swapped"] = swapped
    if pool:
        mutants["wrong pool neighbour"] = torch.roll(v, -1, 3)
    for name, mv in mutants.items():
        verdict = _check16(x, w, b, ks, relu, pool, phys, out16(mv))
        assert not bool(verdict.ok.all()), "%s: mutation '%s' passed the fp16 checker" % (kind, name)
        print("%s fp16: '%s' rejected (%d bad elements)" % (kind, name, int((~verdict.ok).sum())))
    # a bf16-rounded output (3 mantissa bits fewer) is not an fp16 output
    verdict = _check16(x, w, b, ks, relu, pool, phys, conv_check.bf16_round(conv_check.f_act(v, relu, pool)))
    assert not bool(verdict.ok.all())


def test_fp16_abi_surface(built):
    nat = pkg_module("_native")
    with open(os.path.join(ROOT, "include", "b200pose.h")) as f:
        header = f.read()
    assert re.search(r"#define B200POSE_MODE_FP16 4\b", header)
    assert "4 ran as bf16" in header
    assert "int b200pose_net_overflow(b200pose_net* net, int* flags, int n, void* cuda_stream);" in header
    assert "int b200pose_post_overflow(b200pose_post* post, int img);" in header
    assert re.search(r"#define B200POSE_DEBUG_LAUNCH_FORMAT 27\b", header)
    assert nat.MODES["fp16"] == nat.MODE_FP16 == 4
    assert nat.MODES["bf16"] == 0 and nat.MODES["fp8"] == 3
    assert {"b200pose_net_overflow", "b200pose_post_overflow"} <= set(nat.EXPORTED)
    lib = nat.lib()
    flags = np.zeros(1, np.int32)
    assert lib.b200pose_net_overflow(None, flags.ctypes.data, 1, None) < 0
    assert b"overflow" in lib.b200pose_last_error()
    assert lib.b200pose_post_overflow(None, 0) < 0


def test_model_precision_fp16_is_accepted_and_defaults_unchanged(built, monkeypatch):
    monkeypatch.delenv("B200POSE_MODE", raising=False)
    rtpose = pkg_module("lib.network.rtpose_vgg")
    model = rtpose.get_model("vgg19")
    assert model.precision == "bf16x3"
    model.precision = "fp16"
    assert model.precision in pkg_module("_native").MODES
    import inspect
    eng = pkg_module("engine")
    assert inspect.signature(eng.PoseEngine.__init__).parameters["mode"].default == "bf16"
    with pytest.raises(pkg_module("_native").B200PoseError, match=r"image\(s\) \[1\]"):
        eng.check_overflow_flags([False, True, False])
    eng.check_overflow_flags([False, False])


def _ptxas(src):
    r = subprocess.run([os.environ.get("NVCC", "nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "-Xptxas", "-v", "-c", os.path.join(CSRC, src), "-o", os.devnull],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:]
    return re.findall(r"Compiling entry function '(\S+)' for 'sm_90a'(.*?)(?=Compiling entry|\Z)", r.stdout, re.S)


@pytest.mark.parametrize("src,name,count", [("conv_tc.cu", "conv_tc_kernelILNS_8TcFormatE3E", 8),      # TcFormat::kFp16
                                            ("conv_misc.cu", "conv_first_mma_kernelILi.ELNS_8TcFormatE3E", 5)])
def test_fp16_kernels_do_not_spill(built, src, name, count):
    bodies = [(fn, body) for fn, body in _ptxas(src) if re.search(name, fn)]
    assert len(bodies) == count
    for fn, body in bodies:
        assert "0 bytes spill stores, 0 bytes spill loads" in body, (fn, body)
