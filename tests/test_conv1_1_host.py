"""CPU: conv1_1's kernels and the verdict of tests/test_gpu_conv1_1.py.

Every conv1_1 kernel csrc/conv_misc.cu instantiates (ptxas lists them) must be a case of the GPU test's (format, input
kind) matrix, so that a new instantiation cannot go unchecked.  And that verdict must be able to fail: it accepts a host
emulation of the kernel and rejects the emulation with each of the mistakes below.
"""
import itertools
import os
import re

import numpy as np
import pytest
import torch

import fp16_check
from conftest import pkg_module
from oracle import conv_check
from test_fp8_host import CSRC, _ptxas
from test_gpu_conv1_1 import FORMATS, INPUTS, conv1_1_verdict, normalise

TC_FORMATS = ["bf16", "bf16x3", "fp8", "fp16"]          # enum class TcFormat in csrc/tc_format.h, in order
ENTRY = re.compile(r"(conv_first_kernel|conv_first_mma_kernel)ILi(\d+)E(?:LNS_8TcFormatE(\d+)E)?E")
# conv_first_launch: the kernel each format runs
DISPATCH = {"Bf16": "conv_first_mma_kernel<kIn, TcFormat::kBf16>", "Bf16x3": "conv_first_kernel<kIn>",
            "Fp8": "conv_first_mma_kernel<kIn, TcFormat::kFp8>", "Fp16": "conv_first_mma_kernel<kIn, TcFormat::kFp16>"}


def test_every_conv1_1_kernel_is_a_case_of_the_gpu_matrix():
    with open(os.path.join(CSRC, "conv_misc.cu")) as f:
        src = f.read()
    launch = src[src.index("cudaError_t conv_first_launch("):]
    launch = launch[:launch.index("\n}\n")]
    assert dict(re.findall(r"case TcFormat::k(\w+):.*\n\s*(conv_first_\w+<kIn(?:, TcFormat::k\w+)?>)", launch)) == DISPATCH
    assert pkg_module("_native").PREPROCESS == {p: i for i, p in enumerate(INPUTS) if i > 0}
    names = [fn for fn, _ in _ptxas("conv_misc.cu") if "conv_first" in fn]
    cases = []
    for fn in names:
        m = ENTRY.search(fn)
        assert m, fn
        kernel, k_in, fmt = m.groups()
        cases.append(("bf16x3" if kernel == "conv_first_kernel" else TC_FORMATS[int(fmt)], INPUTS[int(k_in)]))
    print("%d conv1_1 kernels: %s" % (len(names), sorted(cases)))
    assert len(names) == 20
    assert sorted(cases) == sorted(itertools.product(FORMATS, INPUTS))


def _f32(t):
    return t.to(torch.float32).to(torch.float64)


def emulate(fmt, pre, src, sd, mutate=None):
    """Host emulation of conv1_1 on one frame.  src: uint8 BGR [H, W, 3] normalised by `pre`, or float32 [3, H, W]
    (pre == "fp32").  The accumulator starts at the bias; the mma.sync kernels (bf16, fp8, fp16) add two exact k16
    partials of K = 27 padded to 32 in fp32, conv_first_kernel (bf16x3) runs the fp32 FMA chain over the taps in
    (channel, ky, kx) order; then ReLU and the stores.  Returns float64 [1, 64, H, W] tensors of the stored values
    (bf16x3: hi and residual).

    mutate: None or one of "rb_swap" (R and B swapped: the channel reversal of vgg / inception forgotten, or one made
    where there is none), "zero_ring" (the padding ring around the frame holds a normalised uint8 0 instead of +0),
    "tap_shift" (the centre tap of channel 0 reads one pixel to the right), "bias" (each channel gets its neighbour's
    bias, 2q <-> 2q + 1) and "partial_tile" (the 8-column partial tile at x = 64 is stored from the first tile's
    columns)."""
    key = next(k for k in sd if k.endswith(".weight"))
    w = sd[key].to(torch.float32).to(torch.float64).reshape(64, 27)
    bias = sd[key[:-len("weight")] + "bias"].to(torch.float32).to(torch.float64)
    if pre == "fp32":
        x = src[[2, 1, 0]] if mutate == "rb_swap" else src
    else:
        x = normalise(pre, (src[:, :, ::-1] if mutate == "rb_swap" else src)[None])[0]
    H, W = x.shape[1:]
    xp = np.zeros((3, H + 2, W + 3), np.float32)           # the zero padding, and a column for the shifted tap
    if mutate == "zero_ring":
        xp[:] = normalise(pre, np.zeros((1, H + 2, W + 3, 3), np.uint8))[0]
    xp[:, 1:H + 1, 1:W + 1] = x
    a = torch.from_numpy(xp).to(torch.float64)
    if fmt in ("bf16", "fp8"):
        a, w = conv_check.bf16_round(a), conv_check.bf16_round(w)
    elif fmt == "fp16":
        a, w = fp16_check.f16_round(a), fp16_check.f16_round(w)
    if mutate == "bias":
        bias = bias[torch.arange(64) ^ 1]
    prods = []
    for k in range(27):
        c, ky, kx = k // 9, k % 9 // 3, k % 3
        kx += 1 if mutate == "tap_shift" and k == 4 else 0
        prods.append(a[c, ky:ky + H, kx:kx + W][None] * w[:, k].view(64, 1, 1))     # exact in float64
    acc = bias.view(64, 1, 1).expand(64, H, W)
    if fmt == "bf16x3":
        for p in prods:
            acc = _f32(acc + p)
    else:
        for s in range(2):
            acc = _f32(acc + sum(prods[16 * s: 16 * s + 16]))
    v = acc.clamp_min(0.0)
    if mutate == "partial_tile":
        v[:, :, 64:] = v[:, :, :W - 64].clone()
    if fmt == "bf16x3":
        hi = conv_check.bf16_round(v)
        return [hi[None], conv_check.bf16_round(_f32(v - hi))[None]]
    return [(fp16_check.f16_round(v) if fmt == "fp16" else conv_check.bf16_round(v))[None]]


MUTATIONS = ["rb_swap", "zero_ring", "tap_shift", "bias", "partial_tile"]
# the fp32 entry point has no normalisation: its padding is +0 whatever the kernel would normalise
NOT_APPLICABLE = {"fp32": {"zero_ring"}}
# (format, input kind) -> mutations the interval cannot see
INVISIBLE = {}


@pytest.mark.parametrize("pre", INPUTS)
@pytest.mark.parametrize("fmt", FORMATS)
def test_verdict_accepts_the_emulated_kernel_and_rejects_mutations(he_sd, fmt, pre):
    """One 8x72 frame: a full 64-wide tile and the partial 8-wide one."""
    H, W = 8, 72
    if pre == "fp32":
        src = (torch.rand((3, H, W), generator=torch.Generator().manual_seed(3)) - 0.5).numpy()
        x = src
    else:
        src = np.random.RandomState(3).randint(0, 256, (H, W, 3)).astype(np.uint8)
        x = normalise(pre, src[None])[0]
    v = conv1_1_verdict(fmt, he_sd, x, emulate(fmt, pre, src, he_sd), device="cpu")
    assert bool(v.ok.all()), v.ratio
    invisible = set()
    for m in MUTATIONS:
        if m in NOT_APPLICABLE.get(pre, ()):
            continue
        vm = conv1_1_verdict(fmt, he_sd, x, emulate(fmt, pre, src, he_sd, mutate=m), device="cpu")
        bad = int((~vm.ok).sum())
        print("%s %s: emulation %.3f of e; mutation %-12s %s (%d of %d elements outside)"
              % (fmt, pre, v.ratio, m, "rejected" if bad else "NOT visible", bad, vm.ok.numel()))
        if not bad:
            invisible.add(m)
    assert invisible == INVISIBLE.get((fmt, pre), set())
