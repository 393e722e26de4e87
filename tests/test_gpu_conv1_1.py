"""GPU (-m gpu): conv1_1 in every tensor-core format and with every input kind, against a float64 reference.

conv1_1 is the one launch whose kernel changes with both the arithmetic format and the input.  csrc/conv_misc.cu builds
20 of them: conv_first_kernel<kIn> (bf16x3: fp32 FMA chain and a residual plane) and conv_first_mma_kernel<kIn, F> for F
in bf16, fp8 and fp16, each for fp32 NCHW input and for uint8 frames with the rtpose, vgg, inception or ssd
normalisation fused into the tile load.  Every (format, input kind) case checks each output element of all 64 channels
with its format's interval (oracle/conv_check.py, tests/fp16_check.py):

  * the reference operand is the numpy normalisation of lib/datasets/preprocessing.py (or the fp32 input), rounded once
    to the format's operand type - bf16 for bf16 and fp8, R16 for fp16 - and kept in fp32 for bf16x3's FMA chain, whose
    weights stay fp32 as well;
  * uniform batches: 1x8x8 (one mostly idle 64x4 tile), 2x64x72 (a full tile and an 8-wide one), 3x24x136 (two tiles
    and 8 columns, three images) and 1x368x496; for uint8 frames also the ragged batch of tests/test_gpu_ragged.py on its
    248x264 canvas, each frame on its own extent against its own reference, every 16-bit word outside it 0x0000.

An interval cannot see a 1-ulp difference in a normalised input, so that is checked bit for bit: the fused uint8 entry
point must store the planes the fp32 entry point stores for the host-normalised frames.  fp8's conv1_1 is the bf16
kernel plus the amax record: its planes must equal bf16's, and the exponent launch 1 uses must be the rule applied to
them.  fp16 must report no overflow.  tests/test_conv1_1_host.py lists the 20 kernels from ptxas and shows that this
verdict rejects a host emulation of the kernel with seeded mistakes.
"""
import time

import numpy as np
import pytest
import torch

import fp8_check
import fp16_check
from conftest import pkg_module
from oracle import conv_check
from test_gpu_fp8 import _debug_fp8
from test_gpu_fp16 import _nchw16, check_plan_fp16
from test_gpu_layers import Hooks, _forward, _nchw, check_plan, layer_net  # noqa: F401 (fixture)
from test_gpu_ragged import SHAPES as RAGGED

pytestmark = pytest.mark.gpu
REF = "cuda"

FORMATS = ["bf16", "bf16x3", "fp8", "fp16"]
INPUTS = ["fp32", "rtpose", "vgg", "inception", "ssd"]          # kIn = 0 .. 4 (csrc/preprocess_core.h)
UNIFORM = [(1, 8, 8), (2, 64, 72), (3, 24, 136), (1, 368, 496)]
CANVAS = (max(h for h, _ in RAGGED), max(w for _, w in RAGGED))
T1 = 0                                                          # conv1_1's output buffer (test_gpu_layers.BUFS)


def normalise(pre, frames):
    """float32 [n, 3, H, W]: the numpy normalisation `pre` of uint8 BGR frames [n, H, W, 3]."""
    fn = getattr(pkg_module("lib.datasets.preprocessing"), pre + "_preprocess")
    return np.stack([fn(f) for f in frames]).astype(np.float32)


def conv1_1_verdict(fmt, sd, x, got, device=REF):
    """The interval check of conv1_1's output over one frame.  x: float32 [3, h, w], the input as the kernel loads it
    (zero padding at the frame's border); got: float64 [1, 64, h, w] tensors of the stored values, hi and residual plane
    in bf16x3."""
    key = next(k for k in sd if k.endswith(".weight"))
    w32 = sd[key]
    b = sd[key[:-len("weight")] + "bias"].double().to(device)
    xin = torch.from_numpy(x[None].astype(np.float64)).to(device)
    if fmt == "bf16x3":         # fp32 CUDA-core FMA chain on the fp32 input and weights
        r, S = conv_check.reference(xin, w32.double().to(device), b, 3)
        return conv_check.check_split(got[0], got[1], r, conv_check.U * conv_check.bound_coef(3, 3, fma=True) * S, relu=True)
    coef = conv_check.U * conv_check.bound_coef(3, 3)           # mma.sync: K = 27 in two k16 steps
    if fmt == "fp16":
        r, S = conv_check.reference(fp16_check.f16_round(xin), fp16_check.round_weights(w32).to(device), b, 3)
        return fp16_check.check_f16(got[0], r, coef * S, relu=True)
    r, S = conv_check.reference(conv_check.bf16_round(xin), conv_check.split_weights(w32)[0].to(device), b, 3)
    return conv_check.check_bf16(got[0], r, coef * S, relu=True)


def _planes(hooks, fmt, img, H, W):
    """uint16 [H, W, 64] planes conv1_1 stored for image img (bf16x3: hi and residual)."""
    return [hooks.act(T1, p, img, H, W) for p in ((0, 1) if fmt == "bf16x3" else (0,))]


def _values(fmt, u16):
    return _nchw16(u16) if fmt == "fp16" else _nchw(u16)


def _run(net, fmt, pre, src):
    """A forward of src through the fp32 entry point (pre == "fp32": float32 [n, 3, H, W]) or the fused uint8 one
    (uint8 [n, H, W, 3]).  Returns the device input, which the hooks' re-runs read: keep it alive."""
    if pre == "fp32":
        return _forward(net, torch.from_numpy(src), fmt)
    nat = pkg_module("_native")
    n, H, W, _ = src.shape
    xd = torch.from_numpy(src).cuda()
    net.forward_u8_ptr(xd.data_ptr(), True, n, H, W, nat.MODES[fmt], [0] * 12, True, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return xd


def _ea_fails(ea, planes, extents, label):
    """fp8: launch 1's activation exponent of each image against the rule on max |stored bf16| inside its extent."""
    fails = []
    for img, (p, (h, w)) in enumerate(zip(planes, extents)):
        amax = float(conv_check.bf16_to_f64(p[0][:h, :w]).abs().max())
        if ea[img] != fp8_check.exp_rule(amax):
            fails.append("%s image %d: launch 1 ea %d, rule %d (amax %r)" % (label, img, ea[img], fp8_check.exp_rule(amax), amax))
    return fails


def _check_uniform(net, sd, fmt, pre, shape):
    nat = pkg_module("_native")
    n, H, W = shape
    shape_label = "%s %dx%dx%d" % (pre, n, H, W)          # the plan checkers add the format
    label = fmt + " " + shape_label
    seed = H * 1000 + W + n
    if pre == "fp32":
        src = x = (torch.rand((n, 3, H, W), generator=torch.Generator().manual_seed(seed)) - 0.5).numpy()
    else:
        src = np.random.RandomState(seed).randint(0, 256, (n, H, W, 3)).astype(np.uint8)
        x = normalise(pre, src)
    xd = _run(net, fmt, pre, src)
    hooks = Hooks(net)
    assert hooks.describe(0)["in_u8"] == (0 if pre == "fp32" else nat.PREPROCESS[pre]), label
    if fmt == "fp16":
        assert not net.overflow(n).any(), label
    if fmt == "fp8":
        ea = _debug_fp8(hooks, 1, n)[0]
    if fmt == "fp16":
        fails, worst = check_plan_fp16(hooks, sd, x, n, H, W, range(n), shape_label, launches=1)
        ratio = worst[0]
    else:
        fails, rows = check_plan(hooks, sd, x, n, H, W, range(n), fmt, launches=1, label=shape_label)
        ratio = rows[0]["ratio_out"]
    got = [_planes(hooks, fmt, img, H, W) for img in range(n)]
    if fmt == "fp8":
        fails += _ea_fails(ea, got, [(H, W)] * n, label)
    # bit-exact: the planes of the same input through another path
    others = [] if pre == "fp32" else [("the fp32 entry point on the host-normalised frames", fmt, "fp32", x)]
    if fmt == "fp8":
        others.append(("the bf16 mode", "bf16", pre, src))
    for what, fmt2, pre2, src2 in others:
        xd2 = _run(net, fmt2, pre2, src2)
        h2 = Hooks(net)
        h2.run(1)
        for img in range(n):
            if not all(np.array_equal(a, b) for a, b in zip(got[img], _planes(h2, fmt2, img, H, W))):
                fails.append("%s image %d: conv1_1 planes differ from %s" % (label, img, what))
        del xd2
    del xd
    return fails, ratio


def _check_ragged(net, sd, fmt, pre):
    """The ragged batch after a batch of canvas-size frames: conv1_1 leaves nothing of those outside the frames."""
    nat = pkg_module("_native")
    Hc, Wc = CANVAS
    st = torch.cuda.current_stream().cuda_stream
    rs = np.random.RandomState(17)

    def run(frames):
        packed = torch.from_numpy(np.concatenate([f.ravel() for f in frames])).cuda()
        net.forward_ragged_u8_ptr(packed.data_ptr(), True, [f.shape[:2] for f in frames], nat.MODES[fmt], [0] * 12, True, st)
        torch.cuda.synchronize()

    run([rs.randint(0, 256, (Hc, Wc, 3)).astype(np.uint8) for _ in RAGGED])
    frames = [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in RAGGED]
    run(frames)
    n = len(frames)
    label = "%s %s ragged" % (fmt, pre)
    hooks = Hooks(net)
    assert hooks.describe(0)["in_u8"] == nat.PREPROCESS[pre], label
    if fmt == "fp16":
        assert not net.overflow(n).any(), label
    got = [_planes(hooks, fmt, img, Hc, Wc) for img in range(n)]    # as the forward left them
    fails, ratio = [], 0.0
    if fmt == "fp8":
        fails += _ea_fails(_debug_fp8(hooks, 1, n)[0], got, RAGGED, label)
    for img, (f, (h, w)) in enumerate(zip(frames, RAGGED)):
        where = "%s frame %d (%dx%d)" % (label, img, h, w)
        v = conv1_1_verdict(fmt, sd, normalise(pre, f[None])[0], [_values(fmt, p[:h, :w]) for p in got[img]])
        if not bool(v.ok.all()):
            fails.append(conv_check.describe(v, _values(fmt, got[img][0][:h, :w]), where))
        ratio = max(ratio, v.ratio)
        for k, p in enumerate(got[img]):
            if p[h:].any() or p[:h, w:].any():
                fails.append("%s: plane %d is not 0x0000 outside the frame" % (where, k))
    return fails, ratio


@pytest.mark.parametrize("pre", INPUTS)
@pytest.mark.parametrize("fmt", FORMATS)
def test_conv1_1_matches_the_float64_reference(layer_net, he_sd, fmt, pre):
    t0 = time.time()
    fails, ratios = [], {}
    layer_net.set_preprocess("rtpose" if pre == "fp32" else pre)
    try:
        for shape in UNIFORM:
            f, ratios["%dx%dx%d" % shape] = _check_uniform(layer_net, he_sd, fmt, pre, shape)
            fails += f
        if pre != "fp32":                       # the ragged entry point takes uint8 frames
            f, ratios["ragged"] = _check_ragged(layer_net, he_sd, fmt, pre)
            fails += f
    finally:
        layer_net.set_preprocess("rtpose")
    print("\nconv1_1 %s %s: max |v - r| / e %.3f (%s); checked in %.1f s" % (
        fmt, pre, max(ratios.values()), ", ".join("%s %.3f" % kv for kv in ratios.items()), time.time() - t0))
    assert not fails, "\n".join(fails[:12]) + ("\n... %d failures in all" % len(fails) if len(fails) > 12 else "")
