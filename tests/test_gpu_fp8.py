"""GPU (-m gpu): the fp8 (e4m3) tensor-core mode (DESIGN.md §2.3).

Every one of the 51 tensor-core launches is checked against a float64 convolution of its own quantised operands: the
launch's real bf16 input planes (b200pose_net_debug_read) scaled by the activation exponent the hook reports
(b200pose_net_debug_fp8), which must equal the rule recomputed from that input, and the fp32 state dict quantised per
output channel (tests/fp8_check.py).  Then the per-image properties the bf16 mode has: batch rows and ragged frames
independent of each other, deterministic runs, graph replay equal to plain launches, and the same launch count.
"""
import time

import numpy as np
import pytest
import torch

import fp8_check
from conftest import golden, pkg_module
from oracle import conv_check
from test_gpu_layers import BUF_C, Hooks, _nchw, _forward, launch_table, layer_net  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu
REF = "cuda"
SHAPES = [((1, 8, 8), (0,)), ((2, 64, 72), (0, 1)), ((1, 184, 248), (0,)), ((1, 368, 368), (0,)),
          ((2, 368, 496), (0, 1)), ((8, 368, 368), (0, 7)), ((32, 368, 368), (0, 31))]


def _debug_fp8(hooks, i, n):
    ea = np.zeros(n, np.int32)
    ew = np.zeros(4096, np.int32)
    rows = hooks.lib.b200pose_net_debug_fp8(hooks.net._h, i, ea.ctypes.data, n, ew.ctypes.data, ew.size)
    assert rows > 0, hooks.lib.b200pose_last_error()
    return ea, ew[:rows]


def check_plan_fp8(hooks, sd, n, H, W, imgs, label):
    table = launch_table()
    fails, worst = [], {}
    for i in range(1, 52):
        f, t = hooks.describe(i), table[i]
        hooks.run(i + 1)
        ea, ew = _debug_fp8(hooks, i, n)
        ks = f["ksize"]
        rows_per_group = f["n_tiles"] * f["n_tile"]
        nb = f["out_buf"]
        for img in imgs:
            src = hooks.act(f["in_buf"], 0, img, H, W)
            after = hooks.act(nb, 0, img, H, W)
            # ---- the activation exponent: max |bf16| over the channels the launch reads, this image only
            read = np.unique(np.concatenate(t["in_ch"]))
            amax = float(np.abs(conv_check.bf16_to_f64(src[..., read]).cpu().numpy()).max())
            want = fp8_check.exp_rule(amax)
            if ea[img] != want:
                fails.append("%s launch %d image %d: ea %d, rule on the input %d (amax %r)" % (label, i, img, ea[img], want, amax))
                continue
            written = np.zeros(BUF_C[nb], bool)
            for g, conv in enumerate(t["convs"]):
                w32 = sd[conv + ".weight"]
                qw, ew_ref = fp8_check.quantise_weights(w32)
                got_ew = ew[g * rows_per_group: g * rows_per_group + w32.shape[0]].tolist()
                if got_ew != ew_ref:
                    fails.append("%s launch %d group %d: weight exponents differ from the rule" % (label, i, g))
                    continue
                b = sd[conv + ".bias"].double().to(REF)
                qa = fp8_check.quantise(_nchw(src, t["in_ch"][g]), int(ea[img]))
                r, S = fp8_check.reference(qa, int(ea[img]), qw.to(REF), ew_ref, b, ks)
                e = fp8_check.bound_coef(ks, f["cin_blocks"] * 64) * S
                off, valid = t["off"][g], w32.shape[0]
                got = _nchw(after[..., off:off + valid])
                v = conv_check.check_bf16(got, r, e, f["relu"], f["pool"])
                where = "%s fp8 launch %d (%s) image %d group %d" % (label, i, conv, img, g)
                if not bool(v.ok.all()):
                    fails.append(conv_check.describe(v, got, where, f["pool"]))
                worst[i] = max(worst.get(i, 0.0), v.ratio)
                if t["maps"][g] >= 0:
                    m = torch.from_numpy(hooks.stage_map(t["maps"][g], img, H, W).astype(np.float64)).to(REF)[None]
                    vm = conv_check.check_f32(m, r, e)
                    if not bool(vm.ok.all()):
                        fails.append(conv_check.describe(vm, m, where + " fp32 map"))
                    worst[i] = max(worst[i], vm.ratio)
                store = min(f["store%d" % g], f["n_tile"])
                mine = np.zeros_like(written)
                for nt in range(f["n_tiles"]):
                    mine[off + nt * f["n_tile"]: off + nt * f["n_tile"] + store] = True
                written |= mine
                pad = [int(c) for c in np.nonzero(mine)[0] if c >= off + valid]
                if pad and np.any(after[..., pad] & 0x7FFF):
                    fails.append("%s: pad channels %s are not 0" % (where, pad))
            prev = hooks.prev.get(img)
            if prev is not None and not written.all() and not np.array_equal(after[..., ~written], prev[..., ~written]):
                fails.append("%s launch %d image %d: channels outside the launch's slice changed" % (label, i, img))
        if i < 51:
            nxt = hooks.describe(i + 1)["out_buf"]
            hooks.prev = {img: hooks.act(nxt, 0, img, H, W) for img in imgs}
    return fails, worst


@pytest.mark.parametrize("shape,imgs", SHAPES, ids=["%dx%dx%d" % s for s, _ in SHAPES])
def test_every_fp8_launch_matches_its_quantised_float64_reference(layer_net, he_sd, shape, imgs):
    t0 = time.time()
    n, H, W = shape
    x = torch.rand((n, 3, H, W), generator=torch.Generator().manual_seed(H * 1000 + W + n)) - 0.5
    xd = _forward(layer_net, x, "fp8")
    hooks = Hooks(layer_net)
    hooks.prev = {}
    fails, worst = check_plan_fp8(hooks, he_sd, n, H, W, imgs, "%dx%dx%d" % shape)
    del xd
    print("\n%dx%dx%d fp8: per-launch max |v - r| / e: %s" % (shape + (" ".join("%d:%.3f" % kv for kv in sorted(worst.items())),)))
    print("  worst %.3f; checked in %.1f s" % (max(worst.values()) if worst else -1, time.time() - t0))
    assert not fails, "\n".join(fails[:12]) + ("\n... %d failures in all" % len(fails) if len(fails) > 12 else "")


def _maps(net, x, mode, stream=None):
    nat = pkg_module("_native")
    n, _, H, W = x.shape
    outs = [torch.empty((n, 38 if i % 2 == 0 else 19, H // 8, W // 8), device="cuda") for i in range(12)]
    st = stream or torch.cuda.current_stream()
    with torch.cuda.stream(st):
        net.forward_ptr(x.data_ptr(), True, n, H, W, nat.MODES[mode], [o.data_ptr() for o in outs], True, st.cuda_stream)
    st.synchronize()
    return [o.cpu() for o in outs]


def test_fp8_batch_rows_are_independent_deterministic_and_graph_replay_equal(layer_net):
    x = (torch.rand((8, 3, 64, 72), generator=torch.Generator().manual_seed(3)) - 0.5).cuda()
    x[3] *= 40.0            # a frame with a much larger range must not change the others' scales
    batch = _maps(layer_net, x, "fp8")
    for i in (0, 3, 7):
        alone = _maps(layer_net, x[i:i + 1].contiguous(), "fp8")
        for b, a in zip(batch, alone):
            assert torch.equal(b[i:i + 1], a), "frame %d in a batch of 8 differs from the frame alone" % i
    s = torch.cuda.Stream()
    runs = [_maps(layer_net, x, "fp8", s) for _ in range(3)]       # plain, plain (graph captured), graph replay
    for r in runs:
        for a, b in zip(r, batch):
            assert torch.equal(a, b)


@pytest.mark.parametrize("flip", [False, True])
def test_fp8_ragged_frames_equal_each_frame_alone(layer_net, flip):
    nat = pkg_module("_native")
    shapes = [(64, 72), (48, 80), (64, 40)]
    rs = np.random.RandomState(9)
    frames = [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in shapes]
    if flip:
        frames = frames + [np.ascontiguousarray(f[:, ::-1]) for f in frames]
        shapes = shapes + shapes
    packed = torch.from_numpy(np.concatenate([f.reshape(-1) for f in frames])).cuda()
    Hc, Wc = max(h for h, _ in shapes), max(w for _, w in shapes)
    outs = [torch.empty((len(shapes), 38 if i % 2 == 0 else 19, Hc // 8, Wc // 8), device="cuda") for i in range(12)]
    layer_net.forward_ragged_u8_ptr(packed.data_ptr(), True, shapes, nat.MODES["fp8"], [o.data_ptr() for o in outs], True,
                                    torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    for i, (f, (h, w)) in enumerate(zip(frames, shapes)):
        fd = torch.from_numpy(f).cuda()
        alone = [torch.empty((1, 38 if k % 2 == 0 else 19, h // 8, w // 8), device="cuda") for k in range(12)]
        layer_net.forward_u8_ptr(fd.data_ptr(), True, 1, h, w, nat.MODES["fp8"], [o.data_ptr() for o in alone], True,
                                 torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        for k in range(12):
            assert torch.equal(outs[k][i:i + 1, :, :h // 8, :w // 8], alone[k]), (i, k)
            assert not torch.any(outs[k][i, :, h // 8:, :]) and not torch.any(outs[k][i, :, :, w // 8:])


def test_fp8_launch_count_equals_bf16(layer_net):
    nat = pkg_module("_native")
    x = (torch.rand((2, 3, 64, 72), generator=torch.Generator().manual_seed(4)) - 0.5).cuda()
    deltas = {}
    for mode in ("bf16", "fp8"):
        _maps(layer_net, x, mode)
        c0 = nat.launch_count()
        _maps(layer_net, x, mode)
        deltas[mode] = nat.launch_count() - c0
    assert deltas["fp8"] == deltas["bf16"] == 52


def test_fp8_end_to_end_deviation_on_net_368(layer_net):
    """Regression guard only (the per-launch checks above are the correctness evidence): per stage max-abs and relative
    RMS of fp8 and bf16 against the fp32 mode on the golden net_368 input."""
    g = golden("net_368")
    x = (torch.rand((1, 3, 368, 368), generator=torch.Generator().manual_seed(int(g["seed"]))) - 0.5).cuda()
    ref = _maps(layer_net, x, "fp32")
    rows = {}
    for mode in ("bf16", "fp8"):
        got = _maps(layer_net, x, mode)
        rows[mode] = [(float((a - r).abs().max()), float(((a - r) ** 2).mean().sqrt() / (r ** 2).mean().sqrt()))
                      for a, r in zip(got, ref)]
    print("\nstage  map   bf16 max-abs  rel-rms    fp8 max-abs  rel-rms")
    for k in range(12):
        print("%5d  %-4s  %11.3e  %8.2e  %11.3e  %8.2e" % (k // 2 + 1, "paf" if k % 2 == 0 else "heat", rows["bf16"][k][0],
                                                          rows["bf16"][k][1], rows["fp8"][k][0], rows["fp8"][k][1]))
    worst_abs = max(r[0] for r in rows["fp8"])
    worst_rms = max(r[1] for r in rows["fp8"])
    print("fp8 worst max-abs %.3e, worst relative RMS %.3e" % (worst_abs, worst_rms))
    assert worst_abs < FP8_MAX_ABS_BAR and worst_rms < FP8_REL_RMS_BAR


# twice the first measurement (H100 80GB HBM3, 400 W: max-abs 0.869, relative RMS 0.242; DESIGN.md §6)
FP8_MAX_ABS_BAR = 1.74
FP8_REL_RMS_BAR = 0.48


def test_fp8_frames_of_a_32_batch_equal_each_frame_alone(layer_net):
    x = (torch.rand((32, 3, 64, 72), generator=torch.Generator().manual_seed(8)) - 0.5).cuda()
    x[5] *= 50.0
    x[20] *= 0.01
    batch = _maps(layer_net, x, "fp8")
    for i in range(32):
        alone = _maps(layer_net, x[i:i + 1].contiguous(), "fp8")
        for b, a in zip(batch, alone):
            assert torch.equal(b[i:i + 1], a), "frame %d of 32 differs from the frame alone" % i


def _fp8_engine(net):
    return pkg_module("engine").PoseEngine.from_net(net, mode="fp8", batch_cap=16, peak_cap=1024, human_cap=2048)


def test_fp8_ragged_inference_with_and_without_flip_equals_each_frame_alone(layer_net):
    """b200pose_infer_raw_u8_ragged in fp8 (flip through the fused mirror and merge) against b200pose_infer_raw_u8 on
    each frame alone."""
    from test_gpu_ragged import RAW, _alone_persons
    pe = _fp8_engine(layer_net)
    rs = np.random.RandomState(23)
    frames = [rs.randint(0, 256, s + (3,)).astype(np.uint8) for s in RAW]
    for flip in (False, True):
        want = [_alone_persons(pe, f, flip, 0.1) for f in frames]
        assert sum(len(r) for r, _ in want) > 0
        packed = np.concatenate([f.ravel() for f in frames])
        pe.infer_raw_ragged_async_u8(packed.ctypes.data, False, [f.shape[:2] for f in frames], 184, 8, 0.1, flip)
        got = pe.fetch_arrays()
        for i in range(len(frames)):
            np.testing.assert_array_equal(got[i], want[i][0], err_msg="flip=%s frame %d" % (flip, i))
            np.testing.assert_array_equal(pe.post.peaks(i), want[i][1], err_msg="flip=%s frame %d" % (flip, i))


@pytest.mark.parametrize("flip", [False, True])
def test_fp8_ragged_multiscale_equals_uniform_multiscale_of_each_frame_alone(layer_net, flip):
    import test_gpu_ragged_multiscale as ms
    pe = _fp8_engine(layer_net)
    frames = ms._frames(ms.RAW, 31)
    want = [ms._alone(pe, f, flip) for f in frames]
    assert sum(len(w[0]) for w in want) > 0
    ms._assert_frames_equal(ms._ragged(pe, frames, flip), want, ms.RAW, "fp8 flip=%s" % flip)


def test_fp8_fused_infer_u8_equals_forward_u8_then_post_run(layer_net):
    nat = pkg_module("_native")
    pe = _fp8_engine(layer_net)
    img = np.random.RandomState(12).randint(0, 256, (4, 184, 184, 3)).astype(np.uint8)
    xd = torch.from_numpy(img).cuda()
    st = torch.cuda.current_stream().cuda_stream
    pe.infer_async_u8(xd.data_ptr(), True, 4, 184, 184, 0.1, st)
    fused = [r.copy() for r in pe.fetch_arrays()]
    fused_peaks = [pe.post.peaks(i) for i in range(4)]
    outs = [torch.empty((4, 38 if i % 2 == 0 else 19, 23, 23), device="cuda") for i in range(12)]
    layer_net.forward_u8_ptr(xd.data_ptr(), True, 4, 184, 184, nat.MODES["fp8"], [o.data_ptr() for o in outs], True, st)
    torch.cuda.synchronize()
    post = pkg_module("engine").NativePost(0, batch_cap=4, peak_cap=1024, human_cap=2048)
    post.run(outs[11].data_ptr(), outs[10].data_ptr(), True, 0, 4, 23, 23, 0.1)
    post.sync()
    assert sum(len(r) for r in fused) > 0
    for i in range(4):
        np.testing.assert_array_equal(post.humans(i), fused[i], err_msg="image %d" % i)
        np.testing.assert_array_equal(post.peaks(i), fused_peaks[i], err_msg="image %d" % i)


def test_fp8_launch_count_of_every_entry_point_equals_bf16(layer_net):
    nat = pkg_module("_native")
    rs = np.random.RandomState(2)
    u8 = torch.from_numpy(rs.randint(0, 256, (2, 64, 72, 3)).astype(np.uint8)).cuda()
    f32 = (torch.rand((2, 3, 64, 72), generator=torch.Generator().manual_seed(2)) - 0.5).cuda()
    raw = [rs.randint(0, 256, s + (3,)).astype(np.uint8) for s in [(90, 120), (120, 90), (100, 100)]]
    packed = np.concatenate([f.ravel() for f in raw])
    same = np.ascontiguousarray(np.stack([raw[2], raw[2]]))
    st = torch.cuda.current_stream().cuda_stream

    def calls(pe, mode):
        m = nat.MODES[mode]
        return {
            "net_forward": lambda: layer_net.forward_ptr(f32.data_ptr(), True, 2, 64, 72, m, [0] * 12, True, st),
            "net_forward_u8": lambda: layer_net.forward_u8_ptr(u8.data_ptr(), True, 2, 64, 72, m, [0] * 12, True, st),
            "net_forward_ragged_u8": lambda: layer_net.forward_ragged_u8_ptr(
                u8.data_ptr(), True, [(64, 72), (64, 64)], m, [0] * 12, True, st),
            "infer": lambda: (pe.infer_async(f32.data_ptr(), True, 2, 64, 72, 0.1, st), pe.fetch_arrays()),
            "infer_u8": lambda: (pe.infer_async_u8(u8.data_ptr(), True, 2, 64, 72, 0.1, st), pe.fetch_arrays()),
            "infer_flip": lambda: (pe.infer_flip_async(f32.data_ptr(), True, 2, 64, 72, 0.1, st), pe.fetch_arrays()),
            "infer_u8_flip": lambda: (pe.infer_flip_async_u8(u8.data_ptr(), True, 2, 64, 72, 0.1, st), pe.fetch_arrays()),
            "infer_raw_u8": lambda: (pe.infer_raw_async_u8(same.ctypes.data, False, 2, 100, 100, 96, 8, 0.1, True),
                                     pe.fetch_arrays()),
            "infer_raw_u8_ragged": lambda: (pe.infer_raw_ragged_async_u8(packed.ctypes.data, False,
                                                                         [f.shape[:2] for f in raw], 96, 8, 0.1, True),
                                            pe.fetch_arrays()),
            "infer_raw_u8_multiscale": lambda: (pe.infer_raw_multiscale_async_u8(
                same.ctypes.data, False, 2, 100, 100, (0.5, 1.0), 96, 8, 0.1, True), pe.fetch_arrays()),
            "infer_raw_u8_multiscale_ragged": lambda: (pe.infer_raw_multiscale_ragged_async_u8(
                packed.ctypes.data, False, [f.shape[:2] for f in raw], (0.5, 1.0), 96, 8, 0.1, True), pe.fetch_arrays()),
        }

    # launches per call: conv1_1 + 51 tensor-core layers per forward, 1 crop (crop_with_factor or the ragged frame copy)
    # and 1 mirror of the raw frames, 2 flip merges and 2 resize-accumulates (heat, PAF) per scale, 3 of post-processing
    # (peaks, limbs, assembly); the raw entry points all run with flip, the multi-scale ones at 2 scales
    fwd, crop, mirror, merge, resize, post = 52, 1, 1, 2, 2, 3
    want = {
        "net_forward": fwd,
        "net_forward_u8": fwd,
        "net_forward_ragged_u8": crop + fwd,
        "infer": fwd + post,
        "infer_u8": fwd + post,
        "infer_flip": mirror + fwd + merge + post,
        "infer_u8_flip": mirror + fwd + merge + post,
        "infer_raw_u8": mirror + crop + fwd + merge + post,
        "infer_raw_u8_ragged": mirror + crop + fwd + merge + post,
        "infer_raw_u8_multiscale": mirror + 2 * (crop + fwd + merge + resize) + post,
        "infer_raw_u8_multiscale_ragged": mirror + 2 * (crop + fwd + merge + resize) + post,
    }
    deltas = {}
    for mode in ("bf16", "fp8"):
        pe = pkg_module("engine").PoseEngine.from_net(layer_net, mode=mode, batch_cap=8, peak_cap=1024, human_cap=2048)
        for name, fn in calls(pe, mode).items():
            fn()
            torch.cuda.synchronize()
            c0 = nat.launch_count()
            fn()
            torch.cuda.synchronize()
            deltas[(mode, name)] = nat.launch_count() - c0
    assert set(want) == set(calls(None, "bf16"))
    for name in want:
        assert deltas[("fp8", name)] == deltas[("bf16", name)] == want[name], \
            (name, deltas[("fp8", name)], deltas[("bf16", name)], want[name])


def test_fp8_harness_exact_integer_cases_and_accumulator_characterisation(built):
    """build/test_conv_fp8: the exact-integer cases (indexing and K order, no rounding assumption), then the accumulator
    characterisation, which must give the constants tests/fp8_check.py bounds with: ACC_BITS bits kept relative to the
    largest term (also across the two k32 steps of a tap), each term truncated toward zero."""
    import os
    import subprocess
    from conftest import ROOT
    exe = os.path.join(ROOT, "build", "test_conv_fp8")
    r = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    print(r.stdout)
    assert r.returncode == 0 and "ALL OK" in r.stdout
    r = subprocess.run([exe, "acc"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    print(r.stdout)
    line = [l for l in r.stdout.splitlines() if l.startswith("ACC ")]
    assert r.returncode == 0 and line
    got = dict(kv.split("=") for kv in line[0].split()[1:])
    assert got == {"bits": str(fp8_check.ACC_BITS), "cross_step_bits": str(fp8_check.ACC_BITS), "per_term": "1",
                   "rounds": "0"}, got
