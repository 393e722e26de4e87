"""GPU (-m gpu): the fp16 (IEEE binary16) tensor-core mode (DESIGN.md §2.3).

Every launch of the fp16 plan - conv1_1 and the 51 tensor-core launches - is checked against a float64 convolution of
its own binary16 input planes (b200pose_net_debug_read) and of the fp32 state dict rounded to binary16, with the bf16
mode's accumulation bound (tests/fp16_check.py).  Then the per-image properties the other modes have (ragged frames,
flip, multi-scale, determinism, graph replay, launch count), the end-to-end gain over bf16 on the golden net_368 input,
and the overflow report: an image whose activations leave binary16's range raises, names the image, and leaves the
next clean run unaffected.
"""
import time

import numpy as np
import pytest
import torch

import fp16_check
from conftest import golden, pkg_module
from oracle import conv_check, glue_port
from test_gpu_layers import (BUF_C, FIELDS, SHAPES, Hooks, _forward, launch_table, layer_net)  # noqa: F401 (fixture)

pytestmark = pytest.mark.gpu
REF = "cuda"


def _nchw16(u16, ch=None):
    t = fp16_check.f16_to_f64(u16, REF).permute(2, 0, 1)[None]
    return t if ch is None else t[:, torch.as_tensor(ch, device=REF)]


def _describe_all(hooks, i):
    """All fields of launch i, the 16-bit format field included."""
    f = np.zeros(len(FIELDS) + 1, np.int32)
    got = hooks.lib.b200pose_net_debug_launch(hooks.net._h, i, f.ctypes.data, len(f))
    assert got == len(f), hooks.lib.b200pose_last_error()
    return dict(zip(FIELDS + ["format"], f.tolist()))


def check_plan_fp16(hooks, sd, x_in, n, H, W, imgs, label, launches=52):
    """x_in: the network input as conv1_1 sees it before rounding (float32 numpy [n, 3, H, W])."""
    table = launch_table()
    fails, worst = [], {}
    prev = {}
    for i in range(launches):
        f, t = _describe_all(hooks, i), table[i]
        assert f["format"] == 1 and f["split"] == 0 and f["chunk"] == 0, (i, f)
        hooks.run(i + 1)
        ks = f["ksize"]
        nb = f["out_buf"]
        for img in imgs:
            after = hooks.act(nb, 0, img, H, W)
            src = None if i == 0 else hooks.act(f["in_buf"], 0, img, H, W)
            written = np.zeros(BUF_C[nb], bool)
            for g, conv in enumerate(t["convs"]):
                w32 = sd[conv + ".weight"]
                b = sd[conv + ".bias"].double().to(REF)
                if i == 0:
                    xin = fp16_check.f16_round(torch.from_numpy(x_in[img:img + 1].astype(np.float64)).to(REF))
                    cin = 3
                else:
                    xin = _nchw16(src, t["in_ch"][g])
                    cin = f["cin_blocks"] * 64
                r, S = conv_check.reference(xin, fp16_check.round_weights(w32).to(REF), b, ks)
                e = conv_check.U * conv_check.bound_coef(ks, cin) * S
                off, valid = t["off"][g], w32.shape[0]
                got = _nchw16(after[..., off:off + valid])
                v = fp16_check.check_f16(got, r, e, f["relu"], f["pool"])
                where = "%s fp16 launch %d (%s) image %d group %d" % (label, i, conv, img, g)
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
            if img in prev and not written.all() and not np.array_equal(after[..., ~written], prev[img][..., ~written]):
                fails.append("%s launch %d image %d: channels outside the launch's slice changed" % (label, i, img))
        if i + 1 < launches:
            nxt = hooks.describe(i + 1)["out_buf"]
            prev = {img: hooks.act(nxt, 0, img, H, W) for img in imgs}
    return fails, worst


@pytest.mark.parametrize("shape,imgs", SHAPES, ids=["%dx%dx%d" % s for s, _ in SHAPES])
def test_every_fp16_launch_matches_its_float64_reference(layer_net, he_sd, shape, imgs):
    t0 = time.time()
    n, H, W = shape
    x = torch.rand((n, 3, H, W), generator=torch.Generator().manual_seed(H * 1000 + W + n)) - 0.5
    xd = _forward(layer_net, x, "fp16")
    fails, worst = check_plan_fp16(Hooks(layer_net), he_sd, x.numpy(), n, H, W, imgs, "%dx%dx%d" % shape)
    del xd
    print("\n%dx%dx%d fp16: per-launch max |v - r| / e: %s" % (shape + (" ".join("%d:%.3f" % kv for kv in sorted(worst.items())),)))
    print("  worst %.3f; checked in %.1f s" % (max(worst.values()), time.time() - t0))
    assert not fails, "\n".join(fails[:12]) + ("\n... %d failures in all" % len(fails) if len(fails) > 12 else "")


@pytest.mark.parametrize("pre", ["rtpose", "vgg", "inception", "ssd"])
def test_fp16_conv1_1_on_uint8_frames(layer_net, he_sd, pre):
    """conv1_1 with each normalisation fused into its load: the binary16 operand is R16 of the normalised value."""
    nat = pkg_module("_native")
    img = np.random.RandomState(5).randint(0, 256, (2, 64, 72, 3)).astype(np.uint8)
    pp = pkg_module("lib.datasets.preprocessing")       # the numpy functions the fused loads restate bit for bit
    prep = {"rtpose": glue_port.rtpose_preprocess, "vgg": glue_port.vgg_preprocess,
            "inception": pp.inception_preprocess, "ssd": pp.ssd_preprocess}[pre]
    x = np.stack([prep(i) for i in img]).astype(np.float32)
    layer_net.set_preprocess(pre)
    try:
        xd = torch.from_numpy(img).cuda()
        layer_net.forward_u8_ptr(xd.data_ptr(), True, 2, 64, 72, nat.MODES["fp16"], [0] * 12, True,
                                 torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        hooks = Hooks(layer_net)
        assert hooks.describe(0)["in_u8"] == nat.PREPROCESS[pre]
        fails, worst = check_plan_fp16(hooks, he_sd, x, 2, 64, 72, (0, 1), "u8 " + pre, launches=1)
    finally:
        layer_net.set_preprocess("rtpose")
    print("conv1_1 %s fp16: max |v - r| / e %.3f" % (pre, worst[0]))
    assert not fails, "\n".join(fails[:12])


def _maps(net, x, mode, stream=None):
    nat = pkg_module("_native")
    n, _, H, W = x.shape
    outs = [torch.empty((n, 38 if i % 2 == 0 else 19, H // 8, W // 8), device="cuda") for i in range(12)]
    st = stream or torch.cuda.current_stream()
    with torch.cuda.stream(st):
        net.forward_ptr(x.data_ptr(), True, n, H, W, nat.MODES[mode], [o.data_ptr() for o in outs], True, st.cuda_stream)
    st.synchronize()
    return [o.cpu() for o in outs]


# Twice the first measurement (H100 80GB HBM3, 700 W: worst relative RMS 2.35e-3, worst max-abs 8.60e-3 over the 12
# maps; bf16 / fp16 relative RMS 8.1 - 9.1 per map; DESIGN.md §6).
FP16_REL_RMS_BAR = 0.0047
FP16_MAX_ABS_BAR = 0.0172


def test_fp16_end_to_end_deviation_on_net_368_is_below_bf16(layer_net):
    """Per stage map, relative RMS and max-abs of fp16 and bf16 against the fp32 mode on the golden net_368 input: fp16
    must be closer than bf16 on every one of the 12 maps (the binary16 rounding unit is 8x finer)."""
    g = golden("net_368")
    x = (torch.rand((1, 3, 368, 368), generator=torch.Generator().manual_seed(int(g["seed"]))) - 0.5).cuda()
    ref = _maps(layer_net, x, "fp32")
    rows = {}
    for mode in ("bf16", "fp16"):
        got = _maps(layer_net, x, mode)
        rows[mode] = [(float((a - r).abs().max()), float(((a - r) ** 2).mean().sqrt() / (r ** 2).mean().sqrt()))
                      for a, r in zip(got, ref)]
    print("\nstage  map   bf16 max-abs  rel-rms   fp16 max-abs  rel-rms   bf16/fp16 rel-rms")
    for k in range(12):
        b, h = rows["bf16"][k], rows["fp16"][k]
        print("%5d  %-4s  %11.3e  %8.2e  %11.3e  %8.2e  %6.1f" % (k // 2 + 1, "paf" if k % 2 == 0 else "heat", b[0], b[1],
                                                                 h[0], h[1], b[1] / h[1]))
    worst_abs = max(r[0] for r in rows["fp16"])
    worst_rms = max(r[1] for r in rows["fp16"])
    print("fp16 worst max-abs %.3e, worst relative RMS %.3e" % (worst_abs, worst_rms))
    for k in range(12):
        assert rows["fp16"][k][1] < rows["bf16"][k][1], (k, rows["fp16"][k], rows["bf16"][k])
    assert worst_abs < FP16_MAX_ABS_BAR and worst_rms < FP16_REL_RMS_BAR


def test_fp16_batch_rows_are_independent_deterministic_and_graph_replay_equal(layer_net):
    x = (torch.rand((8, 3, 64, 72), generator=torch.Generator().manual_seed(3)) - 0.5).cuda()
    batch = _maps(layer_net, x, "fp16")
    for i in (0, 3, 7):
        alone = _maps(layer_net, x[i:i + 1].contiguous(), "fp16")
        for b, a in zip(batch, alone):
            assert torch.equal(b[i:i + 1], a), "frame %d in a batch of 8 differs from the frame alone" % i
    s = torch.cuda.Stream()
    runs = [_maps(layer_net, x, "fp16", s) for _ in range(3)]       # plain, plain (graph captured), graph replay
    for r in runs:
        for a, b in zip(r, batch):
            assert torch.equal(a, b)


def test_fp16_graph_replay_equals_plain_launches_without_graphs(built, he_sd, monkeypatch):
    """B200POSE_GRAPH=0 (plain launches) against a net that captures and replays the small-batch graph."""
    eng = pkg_module("engine")
    x = (torch.rand((2, 3, 64, 72), generator=torch.Generator().manual_seed(6)) - 0.5).cuda()
    out = {}
    for g in ("0", "1"):
        monkeypatch.setenv("B200POSE_GRAPH", g)
        net = eng.NativeNet(0)
        net.load_state_dict_arrays([v.numpy() for v in he_sd.values()])
        s = torch.cuda.Stream()
        out[g] = [_maps(net, x, "fp16", s) for _ in range(3)][-1]
        del net
    for a, b in zip(out["0"], out["1"]):
        assert torch.equal(a, b)


@pytest.mark.parametrize("flip", [False, True])
def test_fp16_ragged_frames_equal_each_frame_alone(layer_net, flip):
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
    layer_net.forward_ragged_u8_ptr(packed.data_ptr(), True, shapes, nat.MODES["fp16"], [o.data_ptr() for o in outs],
                                    True, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    for i, (f, (h, w)) in enumerate(zip(frames, shapes)):
        fd = torch.from_numpy(f).cuda()
        alone = [torch.empty((1, 38 if k % 2 == 0 else 19, h // 8, w // 8), device="cuda") for k in range(12)]
        layer_net.forward_u8_ptr(fd.data_ptr(), True, 1, h, w, nat.MODES["fp16"], [o.data_ptr() for o in alone], True,
                                 torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        for k in range(12):
            assert torch.equal(outs[k][i:i + 1, :, :h // 8, :w // 8], alone[k]), (i, k)
            assert not torch.any(outs[k][i, :, h // 8:, :]) and not torch.any(outs[k][i, :, :, w // 8:])


def _fp16_engine(net):
    return pkg_module("engine").PoseEngine.from_net(net, mode="fp16", batch_cap=16, peak_cap=1024, human_cap=2048)


def test_fp16_ragged_inference_with_and_without_flip_equals_each_frame_alone(layer_net):
    from test_gpu_ragged import RAW, _alone_persons
    pe = _fp16_engine(layer_net)
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
            assert not pe.post.overflow(i)


@pytest.mark.parametrize("flip", [False, True])
def test_fp16_ragged_multiscale_equals_uniform_multiscale_of_each_frame_alone(layer_net, flip):
    import test_gpu_ragged_multiscale as ms
    pe = _fp16_engine(layer_net)
    frames = ms._frames(ms.RAW, 31)
    want = [ms._alone(pe, f, flip) for f in frames]
    assert sum(len(w[0]) for w in want) > 0
    ms._assert_frames_equal(ms._ragged(pe, frames, flip), want, ms.RAW, "fp16 flip=%s" % flip)


def test_fp16_fused_flip_equals_composed_flip(layer_net):
    """b200pose_infer_u8_flip against the composed path: forward of the frames and of their mirrors, then
    b200pose_flip_merge, then b200pose_post_run."""
    nat = pkg_module("_native")
    pe = _fp16_engine(layer_net)
    img = np.random.RandomState(12).randint(0, 256, (2, 184, 184, 3)).astype(np.uint8)
    both = np.ascontiguousarray(np.concatenate([img, img[:, :, ::-1]]))
    xd = torch.from_numpy(img).cuda()
    st = torch.cuda.current_stream().cuda_stream
    pe.infer_flip_async_u8(xd.data_ptr(), True, 2, 184, 184, 0.1, st)
    fused = [r.copy() for r in pe.fetch_arrays()]
    bd = torch.from_numpy(both).cuda()
    outs = [torch.empty((4, 38 if i % 2 == 0 else 19, 23, 23), device="cuda") for i in range(12)]
    layer_net.forward_u8_ptr(bd.data_ptr(), True, 4, 184, 184, nat.MODES["fp16"], [o.data_ptr() for o in outs], True, st)
    torch.cuda.synchronize()
    heat, paf = outs[11].cpu().numpy(), outs[10].cpu().numpy()
    post = pkg_module("engine").NativePost(0, batch_cap=4, peak_cap=1024, human_cap=2048)
    mp, mh = post.flip_merge(heat[:2], heat[2:], paf[:2], paf[2:], layout=0)
    post.run(mh.ctypes.data, mp.ctypes.data, False, 0, 2, 23, 23, 0.1)
    post.sync()
    assert sum(len(r) for r in fused) > 0
    for i in range(2):
        np.testing.assert_array_equal(post.humans(i), fused[i], err_msg="image %d" % i)


def test_fp16_launch_count_equals_bf16(layer_net):
    nat = pkg_module("_native")
    x = (torch.rand((2, 3, 64, 72), generator=torch.Generator().manual_seed(4)) - 0.5).cuda()
    deltas = {}
    for mode in ("bf16", "fp16"):
        _maps(layer_net, x, mode)
        c0 = nat.launch_count()
        _maps(layer_net, x, mode)
        deltas[mode] = nat.launch_count() - c0
    assert deltas["fp16"] == deltas["bf16"] == 52


def test_fp16_and_the_other_modes_alternate_on_one_shape(layer_net):
    """The fp16 plan shares the activation buffers with the other modes' plans of the same shape: alternating modes
    gives each mode its own maps again, bit for bit."""
    x = (torch.rand((1, 3, 64, 72), generator=torch.Generator().manual_seed(11)) - 0.5).cuda()
    first = {m: _maps(layer_net, x, m) for m in ("bf16", "fp16", "fp8", "bf16x3")}
    for m in ("fp16", "bf16", "fp16"):
        for a, b in zip(_maps(layer_net, x, m), first[m]):
            assert torch.equal(a, b), m
    assert not all(torch.equal(a, b) for a, b in zip(first["fp16"], first["bf16"]))


# ---------------------------------------------------------------------------------------------------------- overflow
def _hot_sd(he_sd):
    """conv1_1 scaled so that its largest weight is 60 000: every weight is still a binary16 value, but its outputs on
    inputs in [-0.5, 0.5] reach far beyond 65 504."""
    sd = {k: v.clone() for k, v in he_sd.items()}
    first = next(k for k in sd if k.endswith(".weight"))
    factor = 60000.0 / float(sd[first].abs().max())
    sd[first] *= factor
    sd[first[:-len("weight")] + "bias"] *= factor
    return sd


@pytest.fixture(scope="module")
def hot_net(built, he_sd):
    net = pkg_module("engine").NativeNet(0)
    net.load_state_dict_arrays([v.numpy() for v in _hot_sd(he_sd).values()])
    return net


def test_fp16_overflow_is_flagged_per_image_and_cleared_by_the_next_forward(layer_net):
    """[clean, overflowing, clean]: only the middle image is flagged; then a clean batch on the same net reports none.
    The flags are an arithmetic report, not a device fault: the run itself succeeds."""
    x = (torch.rand((3, 3, 64, 72), generator=torch.Generator().manual_seed(21)) - 0.5).cuda()
    x[1] *= 1e5
    _maps(layer_net, x, "fp16")
    assert layer_net.overflow(3).tolist() == [False, True, False]
    with pytest.raises(pkg_module("_native").B200PoseError, match=r"image\(s\) \[1\]"):
        layer_net.check_overflow(3)
    maps = _maps(layer_net, x[[0, 2]].contiguous(), "fp16")
    assert layer_net.overflow(2).tolist() == [False, False]
    assert all(bool(torch.isfinite(m).all()) for m in maps)
    _maps(layer_net, x, "bf16")                   # other modes report nothing
    assert layer_net.overflow(3).tolist() == [False, False, False]


def test_fp16_overflow_raises_through_forward_and_get_outputs(he_sd):
    rtpose = pkg_module("lib.network.rtpose_vgg")
    coco = pkg_module("evaluate.coco_eval")
    nat = pkg_module("_native")
    model = rtpose.get_model("vgg19")
    model.load_state_dict(_hot_sd(he_sd))
    model = model.cuda().eval()
    model.precision = "fp16"
    x = (torch.rand((2, 3, 64, 64), generator=torch.Generator().manual_seed(2)) - 0.5).cuda()
    with pytest.raises(nat.B200PoseError, match=r"fp16 overflow.*image\(s\) \[0, 1\]"):
        model(x)
    img = np.random.RandomState(3).randint(0, 256, (90, 120, 3)).astype(np.uint8)
    with pytest.raises(nat.B200PoseError, match=r"fp16 overflow.*image\(s\) \[0\]"):
        coco.get_outputs(img, model, "rtpose")
    model.precision = "bf16"                      # the same weights in bf16: finite, no error
    (paf, heat), _ = model(x)
    assert bool(torch.isfinite(paf).all()) and bool(torch.isfinite(heat).all())
    model.load_state_dict(he_sd)                  # clean weights: fp16 runs again on the same module
    model.precision = "fp16"
    (paf, heat), _ = model(x)
    assert bool(torch.isfinite(paf).all())
    coco.get_outputs(img, model, "rtpose")


def test_fp16_overflow_raises_through_engine_fetch_and_names_the_image(layer_net, hot_net):
    nat = pkg_module("_native")
    eng = pkg_module("engine")
    pe = eng.PoseEngine.from_net(layer_net, mode="fp16", batch_cap=8, peak_cap=1024, human_cap=2048)
    x = (torch.rand((3, 3, 64, 72), generator=torch.Generator().manual_seed(22)) - 0.5).cuda()
    x[1] *= 1e5
    st = torch.cuda.current_stream().cuda_stream
    pe.infer_async(x.data_ptr(), True, 3, 64, 72, 0.1, st)
    with pytest.raises(nat.B200PoseError, match=r"image\(s\) \[1\]"):
        pe.fetch()
    pe.infer_flip_async(x.data_ptr(), True, 3, 64, 72, 0.1, st)       # the mirror of frame 1 counts for frame 1
    with pytest.raises(nat.B200PoseError, match=r"image\(s\) \[1\]"):
        pe.fetch_arrays(check=False)
    clean = x[[0, 2]].contiguous()
    pe.infer_async(clean.data_ptr(), True, 2, 64, 72, 0.1, st)
    pe.fetch()
    assert [pe.post.overflow(i) for i in range(2)] == [False, False]
    # every frame of a net whose conv1_1 overflows, through the raw-frame, ragged and multi-scale entry points
    hot = eng.PoseEngine.from_net(hot_net, mode="fp16", batch_cap=8, peak_cap=1024, human_cap=2048)
    rs = np.random.RandomState(4)
    frames = [rs.randint(0, 256, s + (3,)).astype(np.uint8) for s in [(90, 120), (120, 90)]]
    packed = np.concatenate([f.ravel() for f in frames])
    calls = [lambda: hot.infer_raw_ragged_async_u8(packed.ctypes.data, False, [f.shape[:2] for f in frames], 96, 8),
             lambda: hot.infer_raw_multiscale_ragged_async_u8(packed.ctypes.data, False, [f.shape[:2] for f in frames],
                                                              (0.5, 1.0), 96, 8, 0.1, True)]
    for call in calls:
        call()
        with pytest.raises(nat.B200PoseError, match=r"image\(s\) \[0, 1\]"):
            hot.fetch()


@pytest.mark.parametrize("bad", [float("nan"), float("inf"), 1e6])
def test_fp16_non_finite_input_is_flagged(layer_net, bad):
    """An fp32 input that is not finite in binary16 (NaN, inf, beyond 65 504) makes NaN sums in conv1_1 that the ReLU
    would turn into finite zeros; the input fragments are checked, so the image is flagged all the same."""
    x = (torch.rand((3, 3, 64, 72), generator=torch.Generator().manual_seed(23)) - 0.5).cuda()
    x[1, :, 20, 30] = bad
    x[1, 1, 20, 30] = -bad
    _maps(layer_net, x, "fp16")
    assert layer_net.overflow(3).tolist() == [False, True, False]


def test_fp16_refuses_weights_beyond_binary16(built, he_sd):
    """A weight that rounds to inf in binary16 would give NaN sums the ReLU can hide: an fp16 plan with such weights is
    refused with an error naming the conv, and the other modes still run on the same net."""
    nat = pkg_module("_native")
    x = (torch.rand((1, 3, 64, 72), generator=torch.Generator().manual_seed(24)) - 0.5).cuda()
    for conv in (0, 5):
        sd = {k: v.clone() for k, v in he_sd.items()}
        key = [k for k in sd if k.endswith(".weight")][conv]
        sd[key].view(-1)[7] = 1e5
        net = pkg_module("engine").NativeNet(0)
        net.load_state_dict_arrays([v.numpy() for v in sd.values()])
        with pytest.raises(nat.B200PoseError, match=r"conv %d has weight 100000, beyond binary16" % conv):
            _maps(net, x, "fp16")
        _maps(net, x, "bf16")
        with pytest.raises(nat.B200PoseError, match="beyond binary16"):
            _maps(net, x, "fp16")
