"""GPU (-m gpu): every instantiation of conv_tc_kernel<F, N, kRagged, kPrelu>, each run by a plan that selects it and
checked launch by launch against a float64 reference of its own inputs.

conv_tc_launch picks the kernel from the plan's format, the launch's n-tile, whether the forward carries an extents
table (a ragged batch) and whether the layer has PReLU slopes (OpenPose_Model).  add_plan narrows the n-tile on small
batches, so which kernels a plan runs depends on its shape; the end-to-end and per-plan suites do not say which ones
they reach.  Here each case of CASES names a net, a format and a batch, and asserts that the plan the library built
(b200pose_net_debug_launch) has at least one launch of that format and n-tile with (or without) PReLU - the arithmetic
that chose the batch is not trusted.  Every such launch is then re-run (b200pose_net_debug_run, which replays a ragged
batch's extents table) and checked on every frame with tests/ragged_check.py: inside the frame's extent, the format's
interval around a float64 convolution of the launch's own input planes cropped to the frame (oracle/conv_check.py,
tests/prelu_check.py, tests/fp8_check.py, tests/fp16_check.py); outside it, +0; channels outside the launch's slice
unchanged.  A ragged batch runs after a batch of canvas-size frames, so nothing outside a frame is +0 by accident.
tests/test_conv_tc_matrix_host.py checks that CASES lists exactly the instantiations ptxas reports.
"""
import time

import numpy as np
import pytest
import torch

import fp8_check
import fp16_check
import openpose_port
import prelu_check
import ragged_check
import test_gpu_layers as rt_layers
import test_gpu_openpose_layers as op_layers
from conftest import pkg_module
from oracle import conv_check
from test_gpu_fp8 import _debug_fp8
from test_gpu_fp16 import _describe_all

pytestmark = pytest.mark.gpu
REF = "cuda"

# Plans: (net, uniform (n, H, W) or ragged frame sizes).  Two frames of one ragged batch may not have one size: a batch
# of equal sizes runs as a uniform one.
PLANS = {
    "rtpose 1x184x248": ("rtpose", (1, 184, 248)),
    "rtpose ragged 184x248+176x232": ("rtpose", [(184, 248), (176, 232)]),
    "openpose 1x368x368": ("openpose", (1, 368, 368)),
    "openpose ragged 368x368+368x352": ("openpose", [(368, 368), (368, 352)]),
    "openpose ragged 184x248+176x232": ("openpose", [(184, 248), (176, 232)]),
}
RT_U, RT_R = "rtpose 1x184x248", "rtpose ragged 184x248+176x232"
OP_U, OP_R368, OP_R184 = "openpose 1x368x368", "openpose ragged 368x368+368x352", "openpose ragged 184x248+176x232"

# One row per instantiation: (format, N, ragged, PReLU, plan).
CASES = [
    ("bf16", 128, False, False, RT_U),
    ("bf16", 64, False, False, RT_U),
    ("bf16", 48, False, False, RT_U),
    ("bf16", 32, False, False, RT_U),
    ("bf16", 128, True, False, RT_R),
    ("bf16", 64, True, False, RT_R),
    ("bf16", 48, True, False, RT_R),
    ("bf16", 32, True, False, RT_R),
    ("fp16", 128, False, False, RT_U),
    ("fp16", 64, False, False, RT_U),
    ("fp16", 48, False, False, RT_U),
    ("fp16", 32, False, False, RT_U),
    ("fp16", 128, True, False, RT_R),
    ("fp16", 64, True, False, RT_R),
    ("fp16", 48, True, False, RT_R),
    ("fp16", 32, True, False, RT_R),
    ("bf16x3", 64, False, False, RT_U),
    ("bf16x3", 48, False, False, RT_U),
    ("bf16x3", 32, False, False, RT_U),
    ("bf16x3", 64, True, False, RT_R),
    ("bf16x3", 48, True, False, RT_R),
    ("bf16x3", 32, True, False, RT_R),
    ("fp8", 64, False, False, RT_U),
    ("fp8", 48, False, False, RT_U),
    ("fp8", 32, False, False, RT_U),
    ("fp8", 64, True, False, RT_R),
    ("fp8", 48, True, False, RT_R),
    ("fp8", 32, True, False, RT_R),
    ("bf16", 128, False, True, OP_U),
    ("bf16", 64, False, True, OP_U),
    ("bf16", 48, False, True, OP_U),
    ("bf16", 32, False, True, OP_U),
    ("bf16", 128, True, True, OP_R368),
    ("bf16", 64, True, True, OP_R368),
    ("bf16", 48, True, True, OP_R184),
    ("bf16", 32, True, True, OP_R184),
    ("bf16x3", 64, False, True, OP_U),
    ("bf16x3", 48, False, True, OP_U),
    ("bf16x3", 32, False, True, OP_U),
    ("bf16x3", 64, True, True, OP_R368),
    ("bf16x3", 48, True, True, OP_R184),
    ("bf16x3", 32, True, True, OP_R184),
]


def case_id(c):
    return "%s-N%d-%s%s" % (c[0], c[1], "ragged" if c[2] else "uniform", "-prelu" if c[3] else "")


def launch_format(f):
    """The arithmetic format of a launch from its fields: split (bf16x3), binary16 (fp16), chunked (bf16x3, fp8)."""
    if f["split"]:
        return "bf16x3"
    if f["format"]:
        return "fp16"
    return "fp8" if f["chunk"] else "bf16"


def _table(kind):
    """The launch table of the net in one shape: convs, in_ch, off and maps per group, act ('relu', 'prelu' or None),
    slope keys per group, buffers and pool."""
    if kind == "rtpose":
        return [dict(t, act="relu" if t["relu"] else None, slopes=[None] * len(t["convs"]))
                for t in rt_layers.launch_table()]
    return [dict(convs=[t["conv"]], in_ch=[t["in_ch"]], off=[t["off"]], maps=[t["map"]], act=t["act"],
                 slopes=[t["slope"]], in_buf=t["in_buf"], out_buf=t["out_buf"], pool=t["pool"])
            for t in op_layers.launch_table(op_layers.L2, op_layers.L1)]


@pytest.fixture(scope="module")
def nets(built, he_sd):
    eng = pkg_module("engine")
    rt = eng.NativeNet(0)
    rt.load_state_dict_arrays([v.numpy() for v in he_sd.values()])
    op_sd = openpose_port.he_state_dict(op_layers.L2, op_layers.L1)
    op = eng.NativeNet.openpose(0, op_layers.L2, op_layers.L1)
    op.load_state_dict_arrays([v.numpy() for v in op_sd.values()])
    return {"rtpose": (rt, he_sd, rt_layers), "openpose": (op, op_sd, op_layers)}


def run_plan(net, mode, batch, seed):
    """A forward of the plan's batch.  Returns (device input to keep alive, n, H, W, extents per image)."""
    nat = pkg_module("_native")
    st = torch.cuda.current_stream().cuda_stream
    if isinstance(batch, tuple):
        n, H, W = batch
        x = (torch.rand((n, 3, H, W), generator=torch.Generator().manual_seed(seed)) - 0.5).cuda().contiguous()
        net.forward_ptr(x.data_ptr(), True, n, H, W, nat.MODES[mode], [0] * 12, True, st)
        torch.cuda.synchronize()
        return x, n, H, W, [(H, W)] * n
    n, H, W = len(batch), max(h for h, _ in batch), max(w for _, w in batch)
    rs = np.random.RandomState(seed)
    # canvas-size frames first: the ragged batch then runs on buffers that hold data beyond every frame
    full = torch.from_numpy(rs.randint(0, 256, (n, H, W, 3)).astype(np.uint8)).cuda()
    net.forward_u8_ptr(full.data_ptr(), True, n, H, W, nat.MODES[mode], [0] * 12, True, st)
    frames = [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in batch]
    packed = torch.from_numpy(np.concatenate([f.ravel() for f in frames])).cuda()
    net.forward_ragged_u8_ptr(packed.data_ptr(), True, list(batch), nat.MODES[mode], [0] * 12, True, st)
    torch.cuda.synchronize()
    return packed, n, H, W, list(batch)


def _values(fmt, u16, ch=None, device=REF):
    t = (fp16_check.f16_to_f64(u16, device) if fmt == "fp16" else conv_check.bf16_to_f64(u16, device)).permute(2, 0, 1)[None]
    return t if ch is None else t[:, torch.as_tensor(ch, device=device)]


def verdicts_for(fmt, sd, t, f, ea=None, ew=None, device=REF):
    """The caller side of ragged_check.check_image for one launch: the format's interval checks of every group's output
    (and fp32 map) from a float64 convolution of the cropped input planes; fp8 also checks the activation exponent
    against the rule on the frame's own region and the weight exponents against the rule on the state dict."""
    ks, cin = f["ksize"], f["cin_blocks"] * 64
    split = fmt == "bf16x3"

    def verdicts(src, got, maps):
        out, fails = [], []
        if fmt == "fp8":
            read = np.unique(np.concatenate(t["in_ch"]))
            amax = float(conv_check.bf16_to_f64(src[0][..., read]).abs().max()) if src[0].size else 0.0
            if ea != fp8_check.exp_rule(amax):
                return out, ["ea %d, rule on the frame's input %d (amax %r)" % (ea, fp8_check.exp_rule(amax), amax)]
        rows = f["n_tiles"] * f["n_tile"]
        for g, conv in enumerate(t["convs"]):
            w32 = sd[conv + ".weight"]
            b = sd[conv + ".bias"].double().to(device)
            off, valid = t["off"][g], w32.shape[0]
            xin = _values(fmt, src[0], t["in_ch"][g], device)
            gv = _values(fmt, got[0][..., off:off + valid], device=device)
            if fmt == "fp16":
                r, S = conv_check.reference(xin, fp16_check.round_weights(w32).to(device), b, ks)
                e = conv_check.U * conv_check.bound_coef(ks, cin) * S
            elif fmt == "fp8":
                qw, ew_ref = fp8_check.quantise_weights(w32)
                if list(ew[g * rows: g * rows + valid]) != ew_ref:
                    fails.append("group %d: weight exponents differ from the rule" % g)
                    continue
                qa = fp8_check.quantise(xin, int(ea))
                r, S = fp8_check.reference(qa, int(ea), qw.to(device), ew_ref, b, ks)
                e = fp8_check.bound_coef(ks, cin) * S
            else:
                w_hi, w_lo = conv_check.split_weights(w32)
                xin_lo = _values(fmt, src[1], t["in_ch"][g], device) if split else None
                r, S = conv_check.reference(xin, w_hi.to(device), b, ks, xin_lo, w_lo.to(device) if split else None)
                e = conv_check.U * conv_check.bound_coef(ks, cin, split=split, chunk=bool(f["chunk"])) * S
            lo = _values(fmt, got[1][..., off:off + valid], device=device) if split else None
            if t["act"] == "prelu":
                slope = sd[t["slopes"][g]].double()
                v = prelu_check.check_split(gv, lo, r, e, slope) if split else prelu_check.check_bf16(gv, r, e, slope)
            elif fmt == "fp16":
                v = fp16_check.check_f16(gv, r, e, f["relu"], f["pool"])
            elif split:
                v = conv_check.check_split(gv, lo, r, e, f["relu"], f["pool"])
            else:
                v = conv_check.check_bf16(gv, r, e, f["relu"], f["pool"])
            out.append(("group %d (%s)" % (g, conv), v, gv + lo if split else gv))
            if t["maps"][g] >= 0:
                m = torch.from_numpy(maps[g].astype(np.float64)).to(device)[None]
                out.append(("group %d fp32 map %d" % (g, t["maps"][g]), conv_check.check_f32(m, r, e), m))
        return out, fails
    return verdicts


def check_launch(hooks, layers, sd, fmt, i, t, n, H, W, exts, label):
    """Launch i of the plan the last forward built, on every image.  Returns (failures, worst ratio)."""
    f = _describe_all(hooks, i)
    planes = (0, 1) if fmt == "bf16x3" else (0,)
    out_c = layers.BUF_C[f["out_buf"]]
    hooks.run(i)
    before = [[hooks.act(f["out_buf"], p, img, H, W) for p in planes] for img in range(n)]
    hooks.run(i + 1)
    ea, ew = None, None                 # fp8: the activation exponent per image, the weight exponents per row
    if fmt == "fp8":
        ea, ew = _debug_fp8(hooks, i, n)
    written, pad = np.zeros(out_c, bool), []
    for g, conv in enumerate(t["convs"]):
        store, mine = min(f["store%d" % g], f["n_tile"]), np.zeros(out_c, bool)
        for nt in range(f["n_tiles"]):
            mine[t["off"][g] + nt * f["n_tile"]: t["off"][g] + nt * f["n_tile"] + store] = True
        written |= mine
        pad += [int(c) for c in np.nonzero(mine)[0] if c >= t["off"][g] + sd[conv + ".weight"].shape[0]]
    fails, worst = [], 0.0
    for img in range(n):
        src = [hooks.act(f["in_buf"], p, img, H, W) for p in planes]
        after = [hooks.act(f["out_buf"], p, img, H, W) for p in planes]
        maps = [hooks._read(layers.NUM_MAPS_BUF + m, 0, img, (sd[c + ".weight"].shape[0], H // 8, W // 8), np.float32)
                for c, m in zip(t["convs"], t["maps"]) if m >= 0]
        ver = verdicts_for(fmt, sd, t, f, None if ea is None else int(ea[img]), ew)
        fl, ratio = ragged_check.check_image(ver, src, after, before[img], exts[img], f["H"], H, f["pool"], written,
                                             pad, maps, "%s launch %d (%s) image %d" % (label, i, t["convs"][0], img))
        fails += fl
        worst = max(worst, ratio)
    return fails, worst


@pytest.mark.parametrize("case", CASES, ids=[case_id(c) for c in CASES])
def test_instantiation_runs_and_matches_the_float64_reference(nets, case):
    fmt, N, ragged, prelu, plan = case
    kind, batch = PLANS[plan]
    assert isinstance(batch, list) == ragged, case
    net, sd, layers = nets[kind]
    t0 = time.time()
    keep, n, H, W, exts = run_plan(net, fmt, batch, seed=N + 7 * len(plan))
    hooks = layers.Hooks(net)
    table = _table(kind)
    if fmt == "fp16":
        assert not net.overflow(n).any(), "%s: an image is flagged for fp16 overflow" % plan
    chosen = []
    for i in range(1, len(table)):
        f = _describe_all(hooks, i)
        t = table[i]
        assert (f["in_buf"], f["out_buf"], f["pool"], f["groups"]) == (t["in_buf"], t["out_buf"], t["pool"],
                                                                       len(t["convs"])), (i, f, t)
        if launch_format(f) == fmt and f["n_tile"] == N and (t["act"] == "prelu") == prelu:
            chosen.append(i)
    assert chosen, "%s %s: no launch runs conv_tc_kernel<%s, %d, %s, %s>" % (plan, fmt, fmt, N, ragged, prelu)
    fails, worst = [], 0.0
    for i in chosen:
        fl, r = check_launch(hooks, layers, sd, fmt, i, table[i], n, H, W, exts, "%s %s" % (plan, fmt))
        fails += fl
        worst = max(worst, r)
    del keep
    print("\nconv_tc_kernel<%s, %d, %s, %s>: %s, launches %s; worst |v - r| / e %.3f; %.1f s"
          % (fmt, N, ragged, prelu, plan, chosen, worst, time.time() - t0))
    assert not fails, "\n".join(fails[:12]) + ("\n... %d failures in all" % len(fails) if len(fails) > 12 else "")
