"""Reference rules of the fp8 (e4m3) mode (DESIGN.md §2.3), written independently of csrc/fp8_core.h: the scale exponent
rule, e4m3 quantisation (torch.float8_e4m3fn) and the per-launch error bound of conv_tc_kernel in fp8.

A launch's e4m3 operands qa = e4m3(a * 2^ea), qw = e4m3(w * 2^ew) have exact products in fp32.  Each tap runs two k32
wgmmas into a fresh accumulator (the second adds to the first) and the tap's partial is added to an fp32 sum (RN).
Hopper does not document how an fp8 wgmma accumulates; it is modelled as keeping ACC_BITS bits relative to the
largest of its 32 products and the incoming accumulator, truncating each term: a k32 step errs by at most
33 * 2^-ACC_BITS times the sum of the magnitudes it adds.  Over a tap's two steps that is 2 * 33 * 2^-ACC_BITS * S_tap,
and the fp32 sum of T tap partials adds 2^-22 * (T + 16) * S as in oracle/conv_check.py.
"""
import math

import numpy as np
import torch

from oracle import conv_check

E4M3_MAX = 448.0
EXP_CLAMP = 63
ACC_BITS = 13


def exp_rule(amax):
    """floor(log2(448 / amax)) clamped to [-63, 63], 0 for amax == 0 - by exact power-of-two comparisons."""
    a = float(amax)
    if a == 0.0:
        return 0
    if a < 2.0 ** -126:                  # denormal: the quotient is >= 2^134
        return EXP_CLAMP
    e = int(math.floor(math.log2(E4M3_MAX / a)))
    while math.ldexp(a, e) > E4M3_MAX:
        e -= 1
    while math.ldexp(a, e + 1) <= E4M3_MAX:
        e += 1
    return max(-EXP_CLAMP, min(EXP_CLAMP, e))


def quantise(x64, e):
    """e4m3(x * 2^e) as float64 (x: float64 tensor of fp32-representable values; the scaling is exact)."""
    return (x64 * 2.0 ** e).to(torch.float32).to(torch.float8_e4m3fn).to(torch.float64)


def quantise_weights(w32):
    """fp32 OIHW weights -> (float64 e4m3 values of w * 2^ew, ew per output channel)."""
    w = torch.as_tensor(w32).to(torch.float32)
    ew = [exp_rule(float(w[o].abs().max())) for o in range(w.shape[0])]
    q = torch.stack([quantise(w[o].double(), ew[o]) for o in range(w.shape[0])])
    return q, ew


def reference(qa, ea, qw, ew, b, ks):
    """r and S of the quantised convolution: sum(qa 2^-ea * qw 2^-ew) + b, float64."""
    scale = torch.tensor([2.0 ** -e for e in ew], dtype=torch.float64, device=qw.device).view(-1, 1, 1, 1)
    return conv_check.reference(qa * 2.0 ** -ea, qw * scale, b, ks)


def bound_coef(ks, cin):
    """e = bound_coef * S for a ks x ks launch over `cin` (padded) channels, in units of 1 (not 2^-22)."""
    taps = ks * ks * (cin // 64)
    return 2 * 33 * 2.0 ** -ACC_BITS + conv_check.U * (taps + 16)


def e4m3_all_bf16_in_range():
    """Every finite bf16 bit pattern with |x| <= 448, as float32."""
    u = np.arange(1 << 16, dtype=np.uint32)
    f = (u << np.uint32(16)).view(np.float32)
    keep = np.isfinite(f) & (np.abs(f) <= E4M3_MAX)
    return u[keep].astype(np.uint16), f[keep]


def emulate(x64, ea, qw, ew, b, ks, acc_bits=None, mutate=None):
    """Host emulation of conv_tc_kernel in fp8 for one image (x64: float64 [1, C, H, W] bf16 values; qw: e4m3 values of
    w * 2^ew [O, C, ks, ks]): exact e4m3 products; per (channel block, tap) two k32 steps into a fresh accumulator that
    keeps `acc_bits` bits (ACC_BITS) relative to the largest of its terms and the incoming value, truncating each term
    toward zero (the characterised behaviour, DESIGN.md §3); the tap partials summed in fp32 (RN) in the kernel's
    order; v = sum * 2^-(ea + ew) + b in fp32.  Returns v (float64, before ReLU / pool / bf16 rounding).

    mutate: None or one of "ea" (descale by ea + 1), "ew" (output channel 0 descaled by ew + 1), "slice" (the second
    k32 step of channel block 0, centre tap, dropped), "shift" (the centre tap reads one pixel to the right),
    "per_tensor" (weights quantised with one scale for the whole tensor), "bias" (bias scaled by 2)."""
    acc_bits = ACC_BITS if acc_bits is None else acc_bits
    O, C = qw.shape[0], qw.shape[1]
    _, _, H, W = x64.shape
    pad = ks // 2
    qa = quantise(x64, ea)[0]                                       # [C, H, W] = e4m3(a 2^ea)
    if mutate == "per_tensor":
        wt = qw * torch.tensor([2.0 ** -e for e in ew], dtype=torch.float64).view(-1, 1, 1, 1)
        e1 = exp_rule(float(wt.abs().max()))
        qw = quantise(wt, e1)
        ew = [e1] * O
    xp = torch.nn.functional.pad(qa, (pad, pad + 1, pad, pad))
    total = torch.zeros((O, H, W), dtype=torch.float32)
    centre = (ks * ks) // 2
    for cb in range(C // 64):
        for t in range(ks * ks):
            dy, dx = t // ks, t % ks
            if mutate == "shift" and t == centre:
                dx += 1
            win = xp[cb * 64:(cb + 1) * 64, dy:dy + H, dx:dx + W]             # [64, H, W]
            acc = torch.zeros((O, H, W), dtype=torch.float64)
            for s in range(2):
                if mutate == "slice" and cb == 0 and t == centre and s == 1:
                    continue
                p = win[None, 32 * s:32 * s + 32] * qw[:, cb * 64 + 32 * s: cb * 64 + 32 * s + 32, t // ks, t % ks][:, :, None, None]
                big = torch.maximum(acc.abs(), p.abs().amax(1))
                q = torch.where(big > 0, torch.exp2(torch.floor(torch.log2(big.clamp_min(1e-300))) - acc_bits),
                                torch.ones_like(big))
                acc = torch.trunc(acc / q) * q + (torch.trunc(p / q[:, None]) * q[:, None]).sum(1)
            total = total + acc.to(torch.float32)
    e_out = torch.tensor([2.0 ** -(ea + 1 if mutate == "ea" else ea) * 2.0 ** -(e + (1 if mutate == "ew" and o == 0 else 0))
                          for o, e in enumerate(ew)], dtype=torch.float32).view(-1, 1, 1)
    bias = (b * (2.0 if mutate == "bias" else 1.0)).to(torch.float32).view(-1, 1, 1)
    return (total * e_out + bias).to(torch.float64)[None]
