"""ORACLE (test infrastructure only - never imported by the product path).

Per-launch reference check of the tensor-core convolutions of the bf16 / bf16x3 plans.

A launch reads bf16 activation planes and writes bf16 planes (the stage heads also write fp32 maps).  From the launch's
own input planes and weights derived from the state dict, a float64 convolution gives, for every output before it is
rounded, the exact value r = sum(a * w) + b of the bf16 operands, and S = sum|a * w| + |b| bounds every partial sum of
the device's accumulation.  The device's fp32 value v then satisfies |v - r| <= e, with

    e = 2^-22 * (K/16 + 16) * S              wgmma / mma.sync: one fp32 add of an exact 16-product partial per k16 step
    e = 2^-22 * (Kc/16 + 16 + chunks) * S    K-chunked mode: chunks of Kc accumulated as above, summed in fp32 (RN)
    e = 2^-22 * (K + 1) * S                  CUDA-core fp32 FMA chain (conv1_1 in bf16x3 mode)

(bf16 x bf16 products are exact in fp32; K counts the padded K the kernel runs, all three terms in bf16x3 mode.)
2^-22 (twice the fp32 unit roundoff) allows for tensor-core adders that truncate instead of rounding.  Hopper's internal
accumulation is not documented, so that factor is an assumption: every check reports max |v - r| / e.

ReLU, the 2x2 max and round-to-nearest are monotone, so
  * a bf16 output is accepted iff R(f(r - e)) <= got <= R(f(r + e))   (f = ReLU then 2x2 max, R = bf16 RNE);
  * an fp32 head map iff |got - r| <= e;
  * a bf16x3 output (hi, lo) iff f(r - e) - w <= hi + lo <= f(r + e) + w with w = 2^-16 |f(r)| (hi + lo represents v
    to 2^-17 |v|) and |lo| <= ulp(hi) / 2.
Everything is torch float64 and runs on any device; float64 accumulation (error <= K * 2^-53 * S) is 2^-25 below e.
"""
import math
from collections import namedtuple

import numpy as np
import torch
import torch.nn.functional as F

U = 2.0 ** -22
SPLIT_SLACK = 2.0 ** -16
TILE_W, TILE_H = 8, 16          # output tile of conv_tc_kernel (pre-pool pixels)

Verdict = namedtuple("Verdict", "ok ratio lo hi")


def bf16_to_f64(u16, device="cpu"):
    """uint16 bf16 bit patterns (numpy) -> float64 tensor."""
    u = np.ascontiguousarray(u16, dtype=np.uint16).astype(np.uint32) << np.uint32(16)
    return torch.from_numpy(u.view(np.float32)).to(device=device, dtype=torch.float64)


def bf16_round(x):
    """Round-to-nearest-even of float64 values to bf16 precision (one rounding, straight from float64)."""
    x = x.to(torch.float64).contiguous()
    u = x.view(torch.int64)
    u = (u + ((1 << 44) - 1) + ((u >> 45) & 1)) & ~((1 << 45) - 1)
    return u.view(torch.float64)


def bf16_ulp(x):
    """bf16 ulp of bf16-valued x (0 for x == 0), built from the exponent bits: exact on every device (torch.ldexp goes
    through pow, which need not return powers of two exactly)."""
    x = x.to(torch.float64).contiguous()
    ex = (x.view(torch.int64) >> 52) & 0x7FF
    ulp = ((ex - 7).clamp_min(1) << 52).view(torch.float64)
    return torch.where(x == 0, torch.zeros_like(x), ulp)


def split_weights(w):
    """fp32 weights -> (hi, lo) float64: hi = bf16(w), lo = bf16(w - hi) (w - hi is exact)."""
    w = torch.as_tensor(w).to(torch.float32).to(torch.float64)
    hi = bf16_round(w)
    return hi, bf16_round(w - hi)


def reference(x_hi, w_hi, b, ks, x_lo=None, w_lo=None):
    """r and S of a stride-1 'same' conv.  x: float64 NCHW, w: float64 OIHW, b: float64 [O].  With x_lo / w_lo: the three
    bf16x3 terms A_hi W_hi + A_hi W_lo + A_lo W_hi (nothing else)."""
    if x_lo is None:
        X, Wr, Ws = x_hi, w_hi, w_hi.abs()
    else:
        X = torch.cat([x_hi, x_lo], 1)
        Wr = torch.cat([w_hi + w_lo, w_hi], 1)
        Ws = torch.cat([w_hi.abs() + w_lo.abs(), w_hi.abs()], 1)
    r = F.conv2d(X, Wr, b, padding=ks // 2)
    S = F.conv2d(X.abs(), Ws, b.abs(), padding=ks // 2)
    return r, S


def bound_coef(ks, cin, split=False, chunk=False, fma=False):
    """The factor c of e = 2^-22 * c * S for a launch: ks x ks taps over `cin` (padded) input channels."""
    taps = ks * ks
    nterms = 3 if split else 1
    K = nterms * taps * cin
    if fma:
        return K + 1
    if chunk:
        if ks == 7:                      # one chunk per filter row
            kc, chunks = 7 * 64, nterms * (cin // 64) * 7
        else:                            # one chunk per (64-channel block, term)
            kc, chunks = taps * 64, nterms * (cin // 64)
        return math.ceil(kc / 16) + 16 + chunks
    return math.ceil(K / 16) + 16


def f_act(v, relu, pool):
    if relu:
        v = v.clamp_min(0.0)
    if pool:
        v = F.max_pool2d(v, 2)
    return v


def _e_out(e, pool):
    return F.max_pool2d(e, 2) if pool else e


def check_bf16(got, r, e, relu=False, pool=False):
    """got: bf16 values (float64, NCHW, after pool); r, e: pre-activation, pre-pool."""
    lo = bf16_round(f_act(r - e, relu, pool))
    hi = bf16_round(f_act(r + e, relu, pool))
    ok = (got >= lo) & (got <= hi)
    # distance from f(r) to the set of reals that round to `got`, over e: a lower bound of |v - r| / e
    d = ((f_act(r, relu, pool) - got).abs() - bf16_ulp(got) / 2).clamp_min(0.0)
    ratio = float((d / _e_out(e, pool).clamp_min(1e-300)).max()) if d.numel() else 0.0
    return Verdict(ok, ratio, lo, hi)


def check_split(hi_p, lo_p, r, e, relu=False, pool=False):
    v = hi_p + lo_p
    fr = f_act(r, relu, pool)
    w = SPLIT_SLACK * fr.abs()
    a = f_act(r - e, relu, pool) - w
    b = f_act(r + e, relu, pool) + w
    ok = (v >= a) & (v <= b) & (lo_p.abs() <= bf16_ulp(hi_p) / 2)
    d = ((v - fr).abs() - w).clamp_min(0.0)
    ratio = float((d / _e_out(e, pool).clamp_min(1e-300)).max()) if d.numel() else 0.0
    return Verdict(ok, ratio, a, b)


def check_f32(got, r, e):
    err = (got - r).abs()
    ok = err <= e
    ratio = float((err / e.clamp_min(1e-300)).max()) if err.numel() else 0.0
    return Verdict(ok, ratio, r - e, r + e)


def describe(verdict, got, name, pool=False, limit=5):
    """Failure report: count, the first elements with their intervals, and where the bad elements sit relative to the
    kernel's 8 (w) x 16 (h) pixel tiles and 16-channel k-slices."""
    bad = (~verdict.ok).nonzero()
    if bad.numel() == 0:
        return "%s: ok" % name
    s = 2 if pool else 1
    y, x, c = bad[:, 2].cpu() * s, bad[:, 3].cpu() * s, bad[:, 1].cpu()
    edge = ((x % TILE_W == 0) | ((x + s - 1) % TILE_W == TILE_W - 1) | (y % TILE_H == 0) |
            ((y + s - 1) % TILE_H == TILE_H - 1))
    lines = ["%s: %d of %d elements outside the interval; %.0f%% at tile edges (a uniform spread puts ~%.0f%% there); "
             "bad channels %s; bad tile columns (x %% 8) %s" % (
                 name, bad.shape[0], verdict.ok.numel(), 100.0 * float(edge.float().mean()),
                 100.0 * (1 - (1 - 2.0 * s / TILE_W) * (1 - 2.0 * s / TILE_H)),
                 sorted(set(c.tolist()))[:16], sorted(set((x % TILE_W).tolist())))]
    for idx in bad[:limit].tolist():
        t = tuple(idx)
        lines.append("  [n=%d c=%d y=%d x=%d] got %.9g, interval [%.9g, %.9g]" % (
            t[0], t[1], t[2], t[3], float(got[t]), float(verdict.lo[t]), float(verdict.hi[t])))
    return "\n".join(lines)
