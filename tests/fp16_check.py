"""Per-launch check of the fp16 mode (DESIGN.md §2.3): oracle/conv_check.py's interval with binary16 rounding.

An fp16 launch is a bf16 launch with other operands: binary16 activations and weights, whose products are exact in fp32,
and the same fp32 accumulation.  So the bound is the bf16 one, e = 2^-22 * (K/16 + 16) * S, with r and S from a float64
convolution of the launch's own binary16 input planes and of the fp32 weights rounded to binary16 once.  A stored output
is accepted iff R16(f(r - e)) <= got <= R16(f(r + e)), with f = ReLU then the 2x2 max and R16 = round to nearest even
on the binary16 grid, subnormals included, overflow to +-inf.

R16 is one rounding straight from float64: a float64 -> float32 -> float16 cast rounds twice and can land one binary16
ulp off at the midpoints (tests/test_fp16_host.py)."""
import numpy as np
import torch

from oracle import conv_check

F16_MAX = 65504.0
_SUB = 2.0 ** -24          # binary16 subnormal step
_MIN_NORMAL = 2.0 ** -14


def f16_round(x):
    """float64 -> the nearest binary16 value (ties to even), as float64; subnormals kept, beyond 65504 + ulp/2: +-inf."""
    x = x.to(torch.float64).contiguous()
    u = x.view(torch.int64)
    normal = ((u + ((1 << 41) - 1) + ((u >> 42) & 1)) & ~((1 << 42) - 1)).view(torch.float64)    # 10 mantissa bits
    normal = torch.where(normal.abs() > F16_MAX, torch.copysign(torch.full_like(x, float("inf")), x), normal)
    sub = torch.round(x / _SUB) * _SUB        # exact scaling by a power of two; torch.round: ties to even
    out = torch.where(x.abs() < _MIN_NORMAL, sub, normal)
    return torch.where(torch.isnan(x), x, out)


def f16_ulp(x):
    """binary16 ulp of binary16-valued x (the subnormal step below 2^-14; inf for inf), from the exponent bits."""
    x = x.to(torch.float64).contiguous()
    ex = (x.view(torch.int64) >> 52) & 0x7FF
    ulp = ((ex - 10).clamp_min(1) << 52).view(torch.float64)
    return torch.where(x.abs() < _MIN_NORMAL, torch.full_like(x, _SUB), ulp)


def f16_to_f64(u16, device="cpu"):
    """uint16 binary16 bit patterns (numpy) -> float64 tensor (exact)."""
    f = np.ascontiguousarray(u16, dtype=np.uint16).view(np.float16).astype(np.float64)
    return torch.from_numpy(f).to(device)


def round_weights(w):
    """fp32 weights -> float64 binary16 values: one rounding from the fp32 value, like the library's packer."""
    return f16_round(torch.as_tensor(w).to(torch.float32).to(torch.float64))


def check_f16(got, r, e, relu=False, pool=False):
    """got: binary16 values (float64, NCHW, after pool); r, e: pre-activation, pre-pool."""
    lo = f16_round(conv_check.f_act(r - e, relu, pool))
    hi = f16_round(conv_check.f_act(r + e, relu, pool))
    ok = (got >= lo) & (got <= hi)
    d = ((conv_check.f_act(r, relu, pool) - got).abs() - f16_ulp(got) / 2).clamp_min(0.0)
    e_out = torch.nn.functional.max_pool2d(e, 2) if pool else e
    ratio = float((d / e_out.clamp_min(1e-300)).max()) if d.numel() else 0.0
    return conv_check.Verdict(ok, ratio, lo, hi)
