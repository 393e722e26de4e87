"""CPU: the PReLU interval rule (tests/prelu_check.py) that tests/test_gpu_openpose_layers.py trusts must be able to
fail.  The kernel's fp32 arithmetic, emulated on the host (test_oracle's tensor-core emulation, then the PReLU as one
float32 multiply after the bias), must pass on two OpenPose_Model layers; each planted mistake must be caught:
the neighbour channel's slope, PReLU before the bias, ReLU instead of PReLU, a slot-pad lane read as non-zero, and the
features / PAF order of a stage input swapped."""
import numpy as np
import pytest
import torch

import prelu_check
from oracle import conv_check
from test_oracle import _emulate_tc

# the concat buffer [PAF 0..37 | . | heat 40..58 | . | features 64..191] read as torch.cat([features, paf])
FEAT_PAF = np.r_[64:192, 0:38]
PAF_FEAT = np.r_[0:38, 64:192]          # the same channels packed as torch.cat([paf, features])
SLOTS96 = np.r_[0:96, 128:224, 256:352]  # a dense block's three 96-channel outputs in 128-channel slots


def _layer(kind, seed=3):
    """(x NHWC float32 bf16 values, x_lo, w OIHW fp32, b, slope, ks, phys): stage_input = an L2 stage >= 2 Mconv1_0
    (166 -> 128, 3x3) on the concat buffer; dense96 = Mconv2_0 of a first stage (288 -> 96) on three 96-channel slots."""
    rs = np.random.RandomState(seed)
    if kind == "stage_input":
        n, H, W, C, cout, phys = 1, 16, 20, 192, 128, FEAT_PAF
    else:
        n, H, W, C, cout, phys = 1, 16, 20, 384, 96, SLOTS96
    cin, ks = len(phys), 3
    full = np.zeros((n, H, W, C), np.float64)
    full[..., phys] = rs.randn(n, H, W, cin)          # PReLU outputs: both signs
    x = conv_check.bf16_round(torch.from_numpy(full)).numpy().astype(np.float32)
    x_lo = conv_check.bf16_round(torch.from_numpy(full - x)).numpy().astype(np.float32)
    w = (rs.randn(cout, cin, ks, ks) * np.sqrt(1.26 / (cin * ks * ks))).astype(np.float32)
    b = (rs.rand(cout) * 0.2 - 0.1).astype(np.float32)
    slope = (rs.rand(cout) * 2.0 - 0.5).astype(np.float32)
    return x, x_lo, w, b, slope, ks, phys


def _packed(w, C, phys):
    """bf16 hi / lo weights on the physical input channels (zero K rows elsewhere), float64 OIHW."""
    w_hi, w_lo = conv_check.split_weights(w)
    hi = np.zeros((w.shape[0], C) + w.shape[2:])
    lo = np.zeros_like(hi)
    hi[:, phys], lo[:, phys] = w_hi.numpy(), w_lo.numpy()
    return hi, lo


def _prelu_f32(v, slope):
    """The kernel's epilogue on v = fp32(acc + bias): v > 0 ? v : fl32(slope * v)."""
    s = torch.from_numpy(slope.astype(np.float64)).view(1, -1, 1, 1)
    return torch.where(v > 0, v, (s * v).to(torch.float32).to(torch.float64))


def _verdict(x, x_lo, w, b, slope, ks, phys, got_hi, got_lo=None):
    C = x.shape[3]
    hi, lo = _packed(w, C, phys)
    xt = torch.from_numpy(x.astype(np.float64)).permute(0, 3, 1, 2)
    bt = torch.from_numpy(b.astype(np.float64))
    split = got_lo is not None
    if split:
        r, S = conv_check.reference(xt, torch.from_numpy(hi), bt, ks,
                                    torch.from_numpy(x_lo.astype(np.float64)).permute(0, 3, 1, 2), torch.from_numpy(lo))
    else:
        r, S = conv_check.reference(xt, torch.from_numpy(hi), bt, ks)
    e = conv_check.U * conv_check.bound_coef(ks, C, split=split, chunk=split) * S
    if split:
        return prelu_check.check_split(got_hi, got_lo, r, e, slope)
    return prelu_check.check_bf16(got_hi, r, e, slope)


def test_extremes_of_a_non_monotone_prelu():
    """With slope -0.5 on [-2, 1]: f(-2) = 1, f(1) = 1, and f(0) = 0 is the minimum - not in [f(r - e), f(r + e)]."""
    r, e = torch.full((1, 1, 1, 1), -0.5, dtype=torch.float64), torch.full((1, 1, 1, 1), 1.5, dtype=torch.float64)
    lo, hi = prelu_check.extremes(r, e, [-0.5])
    assert float(lo) == 0.0 and float(hi) == 1.0
    lo, hi = prelu_check.extremes(r, torch.full_like(e, 0.25), [1.5])     # [-0.75, -0.25], slope 1.5: no zero inside
    assert float(lo) == -1.125 and float(hi) == -0.375


@pytest.mark.parametrize("kind", ["stage_input", "dense96"])
def test_prelu_checker_accepts_the_kernel_arithmetic_and_rejects_each_mutation(kind):
    x, x_lo, w, b, slope, ks, phys = _layer(kind)
    C = x.shape[3]
    hi, lo = _packed(w, C, phys)
    v = _emulate_tc(x, hi, b, ks, 0, 0)
    good = conv_check.bf16_round(_prelu_f32(v, slope))
    ok = _verdict(x, x_lo, w, b, slope, ks, phys, good)
    print("%s bf16: emulated kernel accepted, max |v - r| / e = %.3f" % (kind, ok.ratio))
    assert bool(ok.ok.all()), conv_check.describe(ok, good, kind)
    assert float((v < 0).double().mean()) > 0.2 and (slope < 0).any() and (slope > 1).any()

    acc = _emulate_tc(x, hi, np.zeros_like(b), ks, 0, 0)          # the accumulator before the bias
    bias = torch.from_numpy(b.astype(np.float64)).view(1, -1, 1, 1)
    mutants = {
        "the neighbour channel's slope": _prelu_f32(v, np.roll(slope, 1)),
        "PReLU before the bias": (_prelu_f32(acc, slope) + bias).to(torch.float32).to(torch.float64),
        "ReLU instead of PReLU": v.clamp_min(0.0),
    }
    if kind == "dense96":
        # the producer stored all 128 lanes of slot 0 (stale values in lanes 96..127) and the packer left those K rows
        # non-zero (each repeats the slot's last channel)
        xm = x.copy()
        xm[..., 96:128] = xm[..., 95:96] + 0.5
        wm = hi.copy()
        wm[:, 96:128] = hi[:, 95:96]
        mutants["a slot-pad lane read as non-zero"] = _prelu_f32(_emulate_tc(xm, wm, b, ks, 0, 0), slope)
    else:
        swapped, _ = _packed(w, C, PAF_FEAT)
        mutants["features / PAF order swapped"] = _prelu_f32(_emulate_tc(x, swapped, b, ks, 0, 0), slope)
    for name, mv in mutants.items():
        got = conv_check.bf16_round(mv)
        verdict = _verdict(x, x_lo, w, b, slope, ks, phys, got)
        assert not bool(verdict.ok.all()), "%s: mutation '%s' passed the checker" % (kind, name)
        print("%s bf16: '%s' rejected (%d bad elements)" % (kind, name, int((~verdict.ok).sum())))

    # bf16x3: the three-term, K-chunked emulation passes; a wrong slope does not
    for slopes, should_pass in ((slope, True), (np.roll(slope, 1), False)):
        fv = _prelu_f32(_emulate_tc(x, hi, b, ks, 0, 0, x_lo=x_lo, w_lo=lo, chunk=True), slopes)
        g_hi = conv_check.bf16_round(fv)
        g_lo = conv_check.bf16_round((fv - g_hi).to(torch.float32).to(torch.float64))
        verdict = _verdict(x, x_lo, w, b, slope, ks, phys, g_hi, g_lo)
        assert bool(verdict.ok.all()) == should_pass, (kind, should_pass, conv_check.describe(verdict, g_hi + g_lo, kind))
        print("%s bf16x3 (%s slope): %s, max |v - r| / e = %.3f" % (kind, "own" if should_pass else "neighbour's",
                                                                  "accepted" if should_pass else "rejected", verdict.ratio))
