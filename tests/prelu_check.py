"""ORACLE (test infrastructure only).  The per-launch interval check of oracle/conv_check.py for outputs that pass
through OpenPose_Model's per-channel PReLU, f(v) = v > 0 ? v : s * v, computed by the kernels as one float32 multiply
after the bias.

conv_check bounds an output by [R(f(r - e)), R(f(r + e))], which holds for ReLU and the 2x2 max because they are
monotone.  With a negative slope PReLU is not, so the interval of f over [r - e, r + e] is taken from its extremes: the
two ends and, when 0 lies inside, f(0) = 0 (f is linear on each side of 0).  The device value is R(fl32(f(v))) for some
fp32 v in [r - e, r + e]; fl32 and the bf16 rounding R are monotone, so it lies in
[R(fl32(min f)), R(fl32(max f))].  bf16x3 outputs (hi, lo) use conv_check's slack w = 2^-16 max |f| on the same
extremes.  No PReLU layer pools, so there is no pool here."""
import torch

from oracle import conv_check


def prelu(v, slope):
    """f(v) per channel of NCHW float64 v; slope: [C]."""
    s = torch.as_tensor(slope, dtype=torch.float64, device=v.device).view(1, -1, 1, 1)
    return torch.where(v > 0, v, s * v)


def _f32(x):
    return x.to(torch.float32).to(torch.float64)


def _scale(e, slope):
    """e times f's Lipschitz constant max(1, |s|) per channel."""
    s = torch.as_tensor(slope, dtype=torch.float64, device=e.device).abs().clamp_min(1.0).view(1, -1, 1, 1)
    return (e * s).clamp_min(1e-300)


def extremes(r, e, slope):
    """(min f, max f) over [r - e, r + e] per element."""
    a, b = prelu(r - e, slope), prelu(r + e, slope)
    lo, hi = torch.minimum(a, b), torch.maximum(a, b)
    straddle = (r - e < 0) & (r + e > 0)
    zero = torch.zeros_like(r)
    return torch.where(straddle, torch.minimum(lo, zero), lo), torch.where(straddle, torch.maximum(hi, zero), hi)


def check_bf16(got, r, e, slope):
    """got: bf16 values (float64, NCHW); r, e: before the bias-add rounding and the PReLU."""
    fmin, fmax = extremes(r, e, slope)
    lo, hi = conv_check.bf16_round(_f32(fmin)), conv_check.bf16_round(_f32(fmax))
    ok = (got >= lo) & (got <= hi)
    # distance from f(r) to the reals that round to `got`, over f's largest change across the interval (e times
    # max(1, |s|)): a lower bound of |v - r| / e, as conv_check reports it
    d = ((prelu(r, slope) - got).abs() - conv_check.bf16_ulp(got) / 2).clamp_min(0.0)
    ratio = float((d / _scale(e, slope)).max()) if d.numel() else 0.0
    return conv_check.Verdict(ok, ratio, lo, hi)


def check_split(hi_p, lo_p, r, e, slope):
    v = hi_p + lo_p
    fmin, fmax = extremes(r, e, slope)
    w = conv_check.SPLIT_SLACK * torch.maximum(fmin.abs(), fmax.abs())
    a, b = fmin - w, fmax + w
    ok = (v >= a) & (v <= b) & (lo_p.abs() <= conv_check.bf16_ulp(hi_p) / 2)
    d = ((v - prelu(r, slope)).abs() - w).clamp_min(0.0)
    ratio = float((d / _scale(e, slope)).max()) if d.numel() else 0.0
    return conv_check.Verdict(ok, ratio, a, b)
