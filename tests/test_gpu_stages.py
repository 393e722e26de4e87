"""GPU (-m gpu): the stage count (b200pose_net_set_stages, NativeNet.set_stages, PoseEngine(stages=k), rtpose_model.stages).
A forward of k stages runs the trunk and stages 1 .. k: its 2k maps are the first 2k maps of a six-stage forward bit for
bit, it makes 7 tensor-core launches fewer per stage it skips, and every fused entry point post-processes stage k's maps."""
import os

import numpy as np
import pytest
import torch

from conftest import assert_humans_equal, pkg_module
from oracle import glue_port, pafprocess_oracle

pytestmark = pytest.mark.gpu

MODES = ["bf16", "bf16x3", "fp16", "fp8", "fp32"]
SCALES = (0.5, 1.0, 1.5, 2.0)


def _nat():
    return pkg_module("_native")


@pytest.fixture(scope="module")
def arrays(built, he_sd):
    return [v.numpy() for v in he_sd.values()]


@pytest.fixture(scope="module")
def net(arrays):
    n = pkg_module("engine").NativeNet(0)
    n.load_state_dict_arrays(arrays)
    return n


def _launches_skipped(mode, k):
    """Launches a k-stage forward makes fewer than a six-stage one: 7 tensor-core launches per stage; the fp32 path runs
    a stage's two branches as 2 x 7 launches and converts its maps into the concat buffer with 2 more (stages 1 .. 5 of
    a six-stage forward, 1 .. k - 1 of a k-stage one)."""
    return 16 * (6 - k) if mode == "fp32" else 7 * (6 - k)


def _forward(net, mode, frames, k, stream, shapes=None):
    """Maps 0 .. 2k-1 (device tensors) of a k-stage forward of uint8 frames [n,H,W,3] (shapes: a ragged batch, frames
    packed back to back) and the launches it made."""
    nat = _nat()
    net.set_stages(k)
    if shapes is None:
        n, H, W = frames.shape[:3]
    else:
        n, H, W = len(shapes), max(s[0] for s in shapes), max(s[1] for s in shapes)
    outs = [torch.empty((n, 38 if i % 2 == 0 else 19, H // 8, W // 8), device="cuda") for i in range(2 * k)]
    ptrs = [o.data_ptr() for o in outs] + [0] * (12 - 2 * k)
    torch.cuda.synchronize()
    l0 = nat.launch_count()
    if shapes is None:
        net.forward_u8_ptr(frames.data_ptr(), True, n, H, W, nat.MODES[mode], ptrs, True, stream.cuda_stream)
    else:
        net.forward_ragged_u8_ptr(frames.data_ptr(), True, shapes, nat.MODES[mode], ptrs, True, stream.cuda_stream)
    stream.synchronize()
    return outs, nat.launch_count() - l0


def _profile_launches(net, stream):
    nat = _nat()
    ms, fl = np.zeros(64, np.float32), np.zeros(64, np.float64)
    return nat.lib().b200pose_net_profile(net._h, ms.ctypes.data, fl.ctypes.data, 64, stream.cuda_stream)


def _fp8_exponents(net, n, launches):
    """Per tensor-core launch 1 .. launches of the last fp8 forward: the activation exponent of each image."""
    nat = _nat()
    out = []
    for i in range(1, launches + 1):
        ea, ew = np.zeros(n, np.int32), np.zeros(1024, np.int32)
        rows = nat.lib().b200pose_net_debug_fp8(net._h, i, ea.ctypes.data, n, ew.ctypes.data, 1024)
        assert rows > 0, nat.lib().b200pose_last_error()
        out.append(ea)
    return out


def _plan_input(plan):
    rs = np.random.RandomState({"small": 3, "b32": 4, "ragged": 5}[plan])
    if plan == "small":
        return torch.from_numpy(rs.randint(0, 256, (2, 64, 72, 3)).astype(np.uint8)).cuda(), None
    if plan == "b32":
        return torch.from_numpy(rs.randint(0, 256, (32, 368, 368, 3)).astype(np.uint8)).cuda(), None
    shapes = [(64, 80), (96, 64), (48, 48)]
    packed = np.concatenate([rs.randint(0, 256, s + (3,)).astype(np.uint8).ravel() for s in shapes])
    return torch.from_numpy(packed).cuda(), shapes


@pytest.mark.parametrize("plan", ["small", "b32", "ragged"])
@pytest.mark.parametrize("mode", MODES)
def test_stage_k_maps_are_the_first_2k_maps_of_six_stages(net, mode, plan):
    """Small plans (PDL-chained) run twice on a real stream, so that the second call replays a captured graph."""
    frames, shapes = _plan_input(plan)
    n = len(shapes) if shapes else frames.shape[0]
    side = torch.cuda.Stream()
    full, full_launches = _forward(net, mode, frames, 6, side, shapes)
    if plan == "small":
        again, _ = _forward(net, mode, frames, 6, side, shapes)
        assert all(torch.equal(a, b) for a, b in zip(again, full))
    if mode == "fp8":      # before the profile: its re-run of a ragged plan covers the whole canvas
        full_ea = _fp8_exponents(net, n, 51)
    if mode != "fp32":
        assert _profile_launches(net, side) == 52
    assert float(full[-1].abs().max()) > 0
    for k in range(1, 6):
        for rep in range(2 if plan == "small" else 1):
            outs, launches = _forward(net, mode, frames, k, side, shapes)
            assert len(outs) == 2 * k
            for i, (a, b) in enumerate(zip(outs, full)):
                assert torch.equal(a, b), (mode, plan, k, rep, i)
            assert full_launches - launches == _launches_skipped(mode, k), (mode, plan, k, launches, full_launches)
        if mode == "fp8":
            for i, (a, b) in enumerate(zip(_fp8_exponents(net, n, 16 + 7 * (k - 1)), full_ea)):
                np.testing.assert_array_equal(a, b, err_msg="launch %d, k=%d" % (i + 1, k))
        if mode != "fp32":
            assert _profile_launches(net, side) == 17 + 7 * (k - 1)
    net.set_stages(6)


# ------------------------------------------------------------------------------------------------ fused entry points
def _stage_maps(net, mode, crops, k):
    """Stage k's (heat, paf) of a six-stage forward of padded uint8 frames [n,H,W,3], NCHW host float32."""
    outs, _ = _forward(net, mode, torch.from_numpy(np.ascontiguousarray(crops)).cuda(), 6, torch.cuda.current_stream())
    return outs[2 * k - 1].cpu().numpy(), outs[2 * k - 2].cpu().numpy()


def _post(ref, heat, paf):
    """Device post-processing of NCHW host maps: per image the person rows and peaks."""
    n, _, h, w = heat.shape
    heat, paf = np.ascontiguousarray(heat), np.ascontiguousarray(paf)
    ref.run(heat.ctypes.data, paf.ctypes.data, False, 0, n, h, w, 0.1)
    ref.sync()
    return [ref.humans(i).copy() for i in range(n)], [ref.peaks(i) for i in range(n)]


def _fused(pe, n):
    rows = [r.copy() for r in pe.fetch_arrays()]
    return rows, [pe.post.peaks(i) for i in range(n)]


def _debug_maps(pe, n, h, w):
    nat = _nat()
    heat, paf = np.empty((n, 19, h, w), np.float32), np.empty((n, 38, h, w), np.float32)
    nat.check(nat.lib().b200pose_post_debug_maps(pe.post._h, heat.ctypes.data, heat.size, paf.ctypes.data, paf.size),
              "b200pose_post_debug_maps")
    return heat, paf


def _assert_same(got, want, what):
    for i, (g, w) in enumerate(zip(got[0], want[0])):
        np.testing.assert_array_equal(g, w, err_msg="%s rows of image %d" % (what, i))
    for i, (g, w) in enumerate(zip(got[1], want[1])):
        np.testing.assert_array_equal(g, w, err_msg="%s peaks of image %d" % (what, i))


def _crop(net, frames, dest):
    return net.crop_with_factor(np.ascontiguousarray(frames), dest, 8)[0]


@pytest.mark.parametrize("mode", MODES)
def test_fused_entry_points_post_process_stage_k(net, mode):
    eng = pkg_module("engine")
    ref = eng.NativePost(0, batch_cap=8, peak_cap=1024, human_cap=2048)
    rs = np.random.RandomState(61)
    frames = rs.randint(0, 256, (2, 96, 128, 3)).astype(np.uint8)
    raw = rs.randint(0, 256, (2, 90, 123, 3)).astype(np.uint8)
    mixed = [rs.randint(0, 256, s + (3,)).astype(np.uint8) for s in ((90, 123), (120, 100))]
    peaks = 0
    for k in (1, 3):
        pe = eng.PoseEngine.from_net(net, mode=mode, batch_cap=4, peak_cap=1024, human_cap=2048, stages=k)
        # infer (fp32 NCHW input) and infer_u8
        x = np.ascontiguousarray(np.stack([glue_port.rtpose_preprocess(f) for f in frames]), dtype=np.float32)
        pe.infer_async(x.ctypes.data, False, 2, 96, 128)
        got = _fused(pe, 2)
        outs = [torch.empty((2, 38 if i % 2 == 0 else 19, 12, 16), device="cuda") for i in range(12)]
        net.set_stages(6)
        xd = torch.from_numpy(x).cuda()
        net.forward_ptr(xd.data_ptr(), True, 2, 96, 128, pe.mode, [o.data_ptr() for o in outs], True, 0)
        torch.cuda.synchronize()
        want = _post(ref, outs[2 * k - 1].cpu().numpy(), outs[2 * k - 2].cpu().numpy())
        _assert_same(got, want, "%s k=%d infer" % (mode, k))
        pe.infer_async_u8(frames.ctypes.data, False, 2, 96, 128)
        want = _post(ref, *_stage_maps(net, mode, frames, k))
        _assert_same(_fused(pe, 2), want, "%s k=%d infer_u8" % (mode, k))
        peaks += sum(len(p) for p in want[1])
        # infer_u8_flip: stage k of both orientations, merged as handle_paf_and_heat does
        pe.infer_flip_async_u8(frames.ctypes.data, False, 2, 96, 128)
        got = _fused(pe, 2)
        heat, paf = _stage_maps(net, mode, np.concatenate([frames, frames[:, :, ::-1]]), k)
        mp, mh = ref.flip_merge(heat[:2], heat[2:], paf[:2], paf[2:], layout=0)
        dh, dp = _debug_maps(pe, 2, 12, 16)
        assert np.array_equal(dh, mh) and np.array_equal(dp, mp), (mode, k)
        _assert_same(got, _post(ref, mh, mp), "%s k=%d infer_u8_flip" % (mode, k))
        # infer_raw_u8, without and with flip (the RAW frame is mirrored before it is cropped)
        crops, crops_m = _crop(net, raw, 96), _crop(net, raw[:, :, ::-1], 96)
        ph, pw = crops.shape[1:3]
        pe.infer_raw_async_u8(raw.ctypes.data, False, 2, 90, 123, 96, 8)
        _assert_same(_fused(pe, 2), _post(ref, *_stage_maps(net, mode, crops, k)), "%s k=%d raw" % (mode, k))
        pe.infer_raw_async_u8(raw.ctypes.data, False, 2, 90, 123, 96, 8, flip=True)
        got = _fused(pe, 2)
        heat, paf = _stage_maps(net, mode, np.concatenate([crops, crops_m]), k)
        mp, mh = ref.flip_merge(heat[:2], heat[2:], paf[:2], paf[2:], layout=0)
        dh, dp = _debug_maps(pe, 2, ph // 8, pw // 8)
        assert np.array_equal(dh, mh) and np.array_equal(dp, mp), (mode, k)
        _assert_same(got, _post(ref, mh, mp), "%s k=%d raw flip" % (mode, k))
        # infer_raw_u8_ragged: each frame as it comes out alone
        packed = np.concatenate([f.ravel() for f in mixed])
        pe.infer_raw_ragged_async_u8(packed.ctypes.data, False, [f.shape[:2] for f in mixed], 96, 8)
        got = _fused(pe, 2)
        for i, f in enumerate(mixed):
            want = _post(ref, *_stage_maps(net, mode, _crop(net, f[None], 96), k))
            _assert_same(([got[0][i]], [got[1][i]]), want, "%s k=%d ragged frame %d" % (mode, k, i))
        # multi-scale with flip, uniform and ragged: stage k at every scale, composed as tests/test_gpu_tta.py does
        port = pafprocess_oracle.load_port()

        def averaged(frame):
            per_scale = []
            for s in SCALES:
                h, p = _stage_maps(net, mode, _crop(net, frame[None], int(96 * s)), k)
                hf, pf = _stage_maps(net, mode, _crop(net, np.ascontiguousarray(frame[:, ::-1])[None], int(96 * s)), k)
                per_scale.append(tuple(np.ascontiguousarray(a[0].transpose(1, 2, 0)) for a in (h, p, hf, pf)))
            base = _crop(net, frame[None], 96)
            return glue_port.multi_scale_maps(per_scale, (base.shape[1] // 8, base.shape[2] // 8))

        for name, imgs in (("multiscale", list(raw)), ("multiscale_ragged", mixed)):
            if name == "multiscale":
                pe.infer_raw_multiscale_async_u8(raw.ctypes.data, False, 2, 90, 123, SCALES, 96, 8, flip=True)
            else:
                pe.infer_raw_multiscale_ragged_async_u8(packed.ctypes.data, False, [f.shape[:2] for f in mixed], SCALES,
                                                        96, 8, flip=True)
            got = pe.fetch()
            pads = [_nat().crop_geometry(f.shape[0], f.shape[1], 96, 8)[2] for f in imgs]
            dh, dp = _debug_maps(pe, 2, max(p[0] for p in pads) // 8, max(p[1] for p in pads) // 8)
            for i, f in enumerate(imgs):
                ah, ap = averaged(f)
                h, w = ah.shape[:2]
                np.testing.assert_allclose(dh[i, :, :h, :w], ah.transpose(2, 0, 1), rtol=0, atol=1e-6,
                                           err_msg="%s k=%d %s frame %d" % (mode, k, name, i))
                np.testing.assert_allclose(dp[i, :, :h, :w], ap.transpose(2, 0, 1), rtol=0, atol=1e-6,
                                           err_msg="%s k=%d %s frame %d" % (mode, k, name, i))
                _, want = glue_port.paf_to_pose(ah, ap, port)
                assert_humans_equal(got[i], want, score_tol=0.0)
    assert peaks > 0
    net.set_stages(6)


# ------------------------------------------------------------------------------------------------ default, switching
@pytest.mark.parametrize("mode", MODES)
def test_explicit_six_equals_the_default_and_switching_reproduces(arrays, net, mode):
    fresh = pkg_module("engine").NativeNet(0)      # the setter never called
    fresh.load_state_dict_arrays(arrays)
    frames, _ = _plan_input("small")
    side = torch.cuda.Stream()
    nat = _nat()
    default = []
    for _ in range(2):
        outs = [torch.empty((2, 38 if i % 2 == 0 else 19, 8, 9), device="cuda") for i in range(12)]
        torch.cuda.synchronize()
        l0 = nat.launch_count()
        fresh.forward_u8_ptr(frames.data_ptr(), True, 2, 64, 72, nat.MODES[mode], [o.data_ptr() for o in outs], True,
                             side.cuda_stream)
        side.synchronize()
        default.append((outs, nat.launch_count() - l0))
    for (outs, launches), (want, want_launches) in zip([_forward(net, mode, frames, 6, side) for _ in range(2)], default):
        assert launches == want_launches
        assert all(torch.equal(a, b) for a, b in zip(outs, want))
    first = {k: _forward(net, mode, frames, k, side)[0] for k in (2, 4)}
    for k in (2, 4):
        _forward(net, mode, frames, 6, side)
        again, _ = _forward(net, mode, frames, k, side)
        assert all(torch.equal(a, b) for a, b in zip(again, first[k])), (mode, k)
    net.set_stages(6)


def test_two_runs_in_flight_with_different_stage_counts(net):
    eng = pkg_module("engine")
    pe = eng.PoseEngine.from_net(net, mode="bf16", batch_cap=4, peak_cap=1024, human_cap=2048)
    rs = np.random.RandomState(71)
    a = rs.randint(0, 256, (2, 90, 123, 3)).astype(np.uint8)
    b = rs.randint(0, 256, (3, 100, 80, 3)).astype(np.uint8)
    alone = {}
    for k, fr in ((2, a), (6, b)):
        pe.stages = k
        pe.infer_raw_async_u8(fr.ctypes.data, False, len(fr), fr.shape[1], fr.shape[2], 96, 8, flip=True)
        alone[k] = ([r.copy() for r in pe.fetch_arrays()], pe.fetch())
    pe.stages = 2
    t2 = pe.infer_raw_async_u8(a.ctypes.data, False, 2, 90, 123, 96, 8, flip=True)
    pe.stages = 6
    t6 = pe.infer_raw_async_u8(b.ctypes.data, False, 3, 100, 80, 96, 8, flip=True)
    for k, t in ((2, t2), (6, t6)):
        rows = [r.copy() for r in pe.fetch_arrays(ticket=t)]
        for g, w in zip(rows, alone[k][0]):
            np.testing.assert_array_equal(g, w)
        assert pe.fetch(ticket=t) == alone[k][1]
    assert sum(len(r) for r in alone[6][0]) + sum(len(r) for r in alone[2][0]) > 0
    net.set_stages(6)


def test_bad_stage_counts_and_outputs_are_refused(net):
    nat = _nat()
    frames, _ = _plan_input("small")
    net.set_stages(3)
    for bad in (0, 7, -1):
        with pytest.raises(nat.B200PoseError, match="stages must be 1 .. 6"):
            net.set_stages(bad)
    outs = [torch.empty((2, 38 if i % 2 == 0 else 19, 8, 9), device="cuda") for i in range(12)]
    ptrs = [o.data_ptr() for o in outs]
    for i in (6, 11):      # the setting is still 3: outputs[6 ..] belong to stages that do not run
        with pytest.raises(nat.B200PoseError, match=r"outputs\[%d\]" % i):
            net.forward_u8_ptr(frames.data_ptr(), True, 2, 64, 72, nat.MODE_BF16, ptrs[:6] + [0] * (i - 6) + [ptrs[i]] +
                               [0] * (11 - i), True, 0)
    with pytest.raises(nat.B200PoseError, match=r"outputs\[6\]"):
        net.forward_ragged_u8_ptr(frames.data_ptr(), True, [(64, 72), (64, 72)], nat.MODE_BF16, ptrs, True, 0)
    net.forward_u8_ptr(frames.data_ptr(), True, 2, 64, 72, nat.MODE_BF16, ptrs[:6] + [0] * 6, True, 0)
    torch.cuda.synchronize()
    full, _ = _forward(net, "bf16", frames, 6, torch.cuda.current_stream())
    assert all(torch.equal(a, b) for a, b in zip(outs[:6], full))
    with pytest.raises(nat.B200PoseError):
        pkg_module("engine").PoseEngine.from_net(net, stages=0)
    net.set_stages(6)


# ------------------------------------------------------------------------------------------------ Python surface
@pytest.fixture(scope="module")
def model(he_sd, built):
    m = pkg_module("lib.network.rtpose_vgg").get_model("vgg19")
    m.load_state_dict(he_sd)
    return m.cuda().eval()


@pytest.mark.parametrize("mode", MODES)
def test_module_stages(model, mode):
    model.precision = mode
    x = (torch.rand((2, 3, 64, 72), generator=torch.Generator().manual_seed(81)) - 0.5).cuda()
    model.stages = 6
    (paf6, heat6), full = model(x)
    for k in (1, 2, 5):
        model.stages = k
        (paf, heat), saved = model(x)
        assert len(saved) == 2 * k
        assert all(torch.equal(a, b) for a, b in zip(saved, full[:2 * k]))
        assert torch.equal(paf, full[2 * k - 2]) and torch.equal(heat, full[2 * k - 1])
    model.stages = 6
    model.precision = "bf16x3"


def test_get_outputs_and_pose_engine_use_stage_k(model, net):
    from evaluate.coco_eval import get_outputs
    img = np.random.RandomState(91).randint(0, 256, (90, 123, 3)).astype(np.uint8)
    model.precision = "bf16"
    crop = _crop(net, img[None], 368)
    try:
        for k in (1, 3):
            model.stages = k
            paf, heat, _ = get_outputs(img, model, "rtpose")
            sh, sp = _stage_maps(net, "bf16", crop, k)
            assert np.array_equal(paf, sp[0].transpose(1, 2, 0)) and np.array_equal(heat, sh[0].transpose(1, 2, 0))
            assert model.pose_engine(batch_cap=4).stages == k
    finally:
        model.stages = 6
        model.precision = "bf16x3"


def test_pose_engine_infer_images_on_mixed_sizes(net):
    eng = pkg_module("engine")
    ref = eng.NativePost(0, batch_cap=4, peak_cap=1024, human_cap=2048)
    rs = np.random.RandomState(93)
    imgs = [rs.randint(0, 256, s + (3,)).astype(np.uint8) for s in ((150, 211), (120, 100), (150, 211), (96, 120))]
    for k in (1, 3):
        pe = eng.PoseEngine.from_net(net, mode="bf16", batch_cap=4, peak_cap=1024, human_cap=2048, stages=k)
        got = pe.infer_images_arrays(imgs, dest_size=184, factor=8)
        for i, im in enumerate(imgs):
            rows, _ = _post(ref, *_stage_maps(net, "bf16", _crop(net, im[None], 184), k))
            np.testing.assert_array_equal(got[i], rows[0], err_msg="k=%d image %d" % (k, i))
    net.set_stages(6)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_data_parallel_honours_stages(model):
    x = (torch.rand((4, 3, 64, 72), generator=torch.Generator().manual_seed(95)) - 0.5).cuda()
    model.precision = "bf16"
    try:
        model.stages = 6
        _, full = model(x)
        model.stages = 2
        dp = torch.nn.DataParallel(model, device_ids=[0, 1])
        (paf, heat), saved = dp(x)
        assert len(saved) == 4
        assert all(torch.equal(a.cpu(), b.cpu()) for a, b in zip(saved, full[:4]))
    finally:
        model.stages = 6
        model.precision = "bf16x3"


def test_environment_sets_the_default(built, monkeypatch):
    monkeypatch.setitem(os.environ, "B200POSE_STAGES", "4")
    assert pkg_module("lib.network.rtpose_vgg").get_model("vgg19").stages == 4
