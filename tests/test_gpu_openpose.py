"""GPU (-m gpu): the reference's OpenPose_Model(l2, l1, 38, 19) on the device (b200pose_net_create_openpose,
NativeNet.openpose, engine.openpose_engine).  fp32 mode bit for bit against the CPU oracle of the same graph
(tests/openpose_port.forward_exact), fp32 / bf16x3 / bf16 against the unmodified reference module's goldens, pad lanes,
ragged batches, every fused entry point against the composed path, an rtpose and an OpenPose engine in flight on one
device, and the refusals."""
import ctypes

import numpy as np
import pytest
import torch

import openpose_port
from conftest import assert_humans_equal, golden, pkg_module
from oracle import glue_port, pafprocess_oracle

pytestmark = pytest.mark.gpu

MODES = ["bf16", "bf16x3", "fp32"]
SCALES = (0.5, 1.0, 1.5, 2.0)
L2, L1 = 4, 2


def _nat():
    return pkg_module("_native")


@pytest.fixture(scope="module")
def sd(built):
    return openpose_port.he_state_dict(L2, L1)


@pytest.fixture(scope="module")
def pe(sd):
    return pkg_module("engine").openpose_engine(sd, L2, L1, batch_cap=8, peak_cap=1024, human_cap=2048)


@pytest.fixture(scope="module")
def net(pe):
    return pe.net


def _maps(net, mode, x=None, frames=None, shapes=None):
    """The l2 + l1 maps (device tensors) of a forward of fp32 NCHW x, uint8 frames [n,H,W,3] or a ragged batch."""
    nat = _nat()
    l2, l1 = net.openpose_stages
    if x is not None:
        n, _, H, W = x.shape
    elif shapes is None:
        n, H, W = frames.shape[:3]
    else:
        n, H, W = len(shapes), max(s[0] for s in shapes), max(s[1] for s in shapes)
    outs = [torch.empty((n, 38 if i < l2 else 19, H // 8, W // 8), device="cuda") for i in range(l2 + l1)]
    ptrs = [o.data_ptr() for o in outs] + [0] * (12 - l2 - l1)
    st = torch.cuda.current_stream().cuda_stream
    if x is not None:
        net.forward_ptr(x.data_ptr(), True, n, H, W, nat.MODES[mode], ptrs, True, st)
    elif shapes is None:
        net.forward_u8_ptr(frames.data_ptr(), True, n, H, W, nat.MODES[mode], ptrs, True, st)
    else:
        net.forward_ragged_u8_ptr(frames.data_ptr(), True, shapes, nat.MODES[mode], ptrs, True, st)
    torch.cuda.synchronize()
    return outs


def _input(n, hw, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand((n, 3) + hw, generator=g) - 0.5


# ------------------------------------------------------------------------------------------------ maps
@pytest.mark.parametrize("n,hw", [(2, (64, 64)), (1, (368, 368))])
def test_fp32_is_bit_identical_to_the_exact_oracle(net, sd, n, hw):
    x = _input(n, hw, 5)
    got = _maps(net, "fp32", x=x.cuda())
    want = openpose_port.forward_exact(sd, x.numpy(), L2, L1)
    for i, (g, w) in enumerate(zip(got, want)):
        np.testing.assert_array_equal(g.cpu().numpy(), w, err_msg="map %d" % i)


def test_fp32_ragged_batch_is_bit_identical_to_the_exact_oracle(net, sd):
    """Each frame of a ragged fp32 batch: inside its extent the oracle's maps of that frame alone (rtpose_preprocess,
    then forward_exact), outside +0."""
    rs = np.random.RandomState(13)
    shapes = [(64, 72), (48, 80), (72, 56)]
    frames = [rs.randint(0, 256, s + (3,)).astype(np.uint8) for s in shapes]
    packed = torch.from_numpy(np.concatenate([f.ravel() for f in frames])).cuda()
    got = _maps(net, "fp32", frames=packed, shapes=shapes)
    for i, f in enumerate(frames):
        want = openpose_port.forward_exact(sd, glue_port.rtpose_preprocess(f)[None].astype(np.float32), L2, L1)
        h, w = f.shape[0] // 8, f.shape[1] // 8
        for m, (g, wm) in enumerate(zip(got, want)):
            g = g[i].cpu().numpy()
            np.testing.assert_array_equal(g[:, :h, :w], wm[0], err_msg="frame %d map %d" % (i, m))
            assert not g[:, h:, :].any() and not g[:, :, w:].any(), (i, m)


@pytest.mark.parametrize("mode,tol", [("fp32", 1e-3), ("bf16x3", 1e-3), ("bf16", 0.25)])
def test_368_against_the_reference_golden(net, mode, tol):
    g = golden("openpose_368")
    gen = torch.Generator().manual_seed(int(g["seed"]))
    x = torch.rand((1, 3, 368, 368), generator=gen) - 0.5
    outs = _maps(net, mode, x=x.cuda())
    e_paf = float(np.abs(outs[L2 - 1].cpu().numpy() - g["paf"]).max())
    e_heat = float(np.abs(outs[-1].cpu().numpy() - g["heat"]).max())
    print("OpenPose_Model(4, 2) %s @368: max|paf err| %.2e  max|heat err| %.2e (maps up to %.1f)"
          % (mode, e_paf, e_heat, float(np.max(g["stage_absmax"]))))
    assert e_paf < tol and e_heat < tol
    for i, o in enumerate(outs):
        np.testing.assert_allclose(o.cpu().numpy().reshape(-1)[::13][:64], g["stage_sample"][i], rtol=0, atol=tol)


@pytest.mark.parametrize("mode", ["bf16", "bf16x3"])
def test_pad_lanes_are_zero(net, mode):
    """After a forward: the concat buffer's pad lanes (38, 39, 59..63) and lanes 96..127 of the first stages' dense
    slots (bra / brb channels 384..767) hold +0, in both planes of bf16x3."""
    nat = _nat()
    frames = torch.from_numpy(np.random.RandomState(3).randint(0, 256, (2, 64, 72, 3)).astype(np.uint8)).cuda()
    _maps(net, mode, frames=frames)
    cat_id, bra, brb = 10, 11, 12
    for lo in ((0, 1) if mode == "bf16x3" else (0,)):
        for buf, c in ((cat_id, 192), (bra, 768), (brb, 768)):
            a = np.empty((2, 8, 9, c), np.uint16)
            nat.check(nat.lib().b200pose_net_debug_read(net._h, buf, lo, 0, 2, a.ctypes.data, a.nbytes), "debug_read")
            if buf == cat_id:
                lanes = [38, 39] + list(range(59, 64))
            else:
                lanes = [s * 128 + k for s in (3, 4, 5) for k in range(96, 128)]
            assert not a[..., lanes].any(), (mode, buf, lo)


@pytest.mark.parametrize("mode", MODES)
def test_ragged_frames_equal_each_frame_alone(net, mode):
    rs = np.random.RandomState(9)
    shapes = [(64, 72), (48, 80), (72, 56)]
    frames = [rs.randint(0, 256, s + (3,)).astype(np.uint8) for s in shapes]
    packed = torch.from_numpy(np.concatenate([f.ravel() for f in frames])).cuda()
    rag = _maps(net, mode, frames=packed, shapes=shapes)
    for i, f in enumerate(frames):
        alone = _maps(net, mode, frames=torch.from_numpy(f[None]).cuda())
        h, w = f.shape[0] // 8, f.shape[1] // 8
        for m, (a, b) in enumerate(zip(rag, alone)):
            assert torch.equal(a[i, :, :h, :w], b[0]), (mode, i, m)
            assert not a[i, :, h:, :].any() and not a[i, :, :, w:].any(), (mode, i, m)


# ------------------------------------------------------------------------------------------------ fused entry points
def _post(ref, heat, paf):
    n, _, h, w = heat.shape
    heat, paf = np.ascontiguousarray(heat), np.ascontiguousarray(paf)
    ref.run(heat.ctypes.data, paf.ctypes.data, False, 0, n, h, w, 0.1)
    ref.sync()
    return [ref.humans(i).copy() for i in range(n)], [ref.peaks(i) for i in range(n)]


def _fused(pe, n):
    rows = [r.copy() for r in pe.fetch_arrays()]
    return rows, [pe.post.peaks(i) for i in range(n)]


def _assert_same(got, want, what):
    for i, (g, w) in enumerate(zip(got[0], want[0])):
        np.testing.assert_array_equal(g, w, err_msg="%s rows of image %d" % (what, i))
    for i, (g, w) in enumerate(zip(got[1], want[1])):
        np.testing.assert_array_equal(g, w, err_msg="%s peaks of image %d" % (what, i))


def _final(net, mode, crops):
    """(heat_l1, paf_l2) of padded uint8 frames [n,H,W,3], NCHW host float32."""
    outs = _maps(net, mode, frames=torch.from_numpy(np.ascontiguousarray(crops)).cuda())
    return outs[-1].cpu().numpy(), outs[net.openpose_stages[0] - 1].cpu().numpy()


def _engine(net, mode):
    """An engine of its own per test, so that no test changes what another runs."""
    return pkg_module("engine").PoseEngine.from_net(net, mode=mode, batch_cap=8, peak_cap=1024, human_cap=2048)


def _crop(net, frames, dest):
    return net.crop_with_factor(np.ascontiguousarray(frames), dest, 8)[0]


def _check_u8_flip_and_ragged(pe, ref, net, mode, frames, mixed):
    """infer_u8, infer_u8_flip and infer_images on mixed sizes (one ragged batch) against the composed path: forward,
    flip merge, post-processing; each ragged frame as it comes out alone.  Returns the peaks of infer_u8."""
    label = "OpenPose_Model(%d, %d) %s" % (net.openpose_stages + (mode,))
    n, H, W = frames.shape[:3]
    pe.infer_async_u8(frames.ctypes.data, False, n, H, W)
    want = _post(ref, *_final(net, mode, frames))
    _assert_same(_fused(pe, n), want, "%s infer_u8" % label)
    peaks = sum(len(p) for p in want[1])
    pe.infer_flip_async_u8(frames.ctypes.data, False, n, H, W)
    got = _fused(pe, n)
    heat, paf = _final(net, mode, np.concatenate([frames, frames[:, :, ::-1]]))
    mp, mh = ref.flip_merge(heat[:n], heat[n:], paf[:n], paf[n:], layout=0)
    _assert_same(got, _post(ref, mh, mp), "%s infer_u8_flip" % label)
    got = pe.infer_images_arrays(mixed, 96, 8)
    for i, f in enumerate(mixed):
        want = _post(ref, *_final(net, mode, _crop(net, f[None], 96)))
        np.testing.assert_array_equal(got[i], want[0][0], err_msg="%s infer_images frame %d" % (label, i))
    return peaks


@pytest.mark.parametrize("mode", MODES)
def test_fused_entry_points_equal_the_composed_path(net, mode):
    eng = pkg_module("engine")
    pe = _engine(net, mode)
    ref = eng.NativePost(0, batch_cap=8, peak_cap=1024, human_cap=2048)
    rs = np.random.RandomState(61)
    frames = rs.randint(0, 256, (2, 96, 128, 3)).astype(np.uint8)
    raw = rs.randint(0, 256, (2, 90, 123, 3)).astype(np.uint8)
    mixed = [rs.randint(0, 256, s + (3,)).astype(np.uint8) for s in ((90, 123), (120, 100))]
    peaks = _check_u8_flip_and_ragged(pe, ref, net, mode, frames, mixed)
    # infer_frames, NV12: the same persons as BGR frames converted on the device and cropped
    nv12 = [rs.randint(0, 256, (144, 128)).astype(np.uint8) for _ in range(2)]
    bgr = net.convert_frames(nv12, "nv12")
    got = pe.infer_frames_arrays(nv12, "nv12", 0, 96, 8)
    want = _post(ref, *_final(net, mode, _crop(net, np.stack(bgr), 96)))
    for i in range(2):
        np.testing.assert_array_equal(got[i], want[0][i], err_msg="%s infer_frames nv12 frame %d" % (mode, i))
    # four scales with flip: the final maps at every scale, composed as tests/test_gpu_tta.py does
    port = pafprocess_oracle.load_port()
    got = pe.infer_images(list(raw), 96, 8, flip=True, scales=SCALES)
    for i, f in enumerate(raw):
        per_scale = []
        for s in SCALES:
            h, p = _final(net, mode, _crop(net, f[None], int(96 * s)))
            hf, pf = _final(net, mode, _crop(net, np.ascontiguousarray(f[:, ::-1])[None], int(96 * s)))
            per_scale.append(tuple(np.ascontiguousarray(a[0].transpose(1, 2, 0)) for a in (h, p, hf, pf)))
        base = _crop(net, f[None], 96)
        ah, ap = glue_port.multi_scale_maps(per_scale, (base.shape[1] // 8, base.shape[2] // 8))
        _, want = glue_port.paf_to_pose(ah, ap, port)
        assert_humans_equal(got[i], want, score_tol=0.0)
    assert peaks > 0


def test_fp32_image_to_persons_equals_the_cpu_oracle_pipeline(net, sd):
    """fp32: the fused path's persons on an image equal the CPU pipeline's - exact oracle forward, then the oracle's
    post-processing - since the maps are bit for bit the oracle's."""
    pe = _engine(net, "fp32")
    img = np.random.RandomState(77).randint(0, 256, (96, 112, 3)).astype(np.uint8)
    got = pe.infer_batch(img[None])
    x = glue_port.rtpose_preprocess(img)[None].astype(np.float32)
    maps = openpose_port.forward_exact(sd, x, L2, L1)
    heat, paf = maps[-1][0].transpose(1, 2, 0), maps[L2 - 1][0].transpose(1, 2, 0)
    _, want = glue_port.paf_to_pose(np.ascontiguousarray(heat), np.ascontiguousarray(paf), pafprocess_oracle.load_port())
    assert_humans_equal(got[0], want, score_tol=0.0)


# ------------------------------------------------------------------------------------------------ two nets, refusals
def test_rtpose_and_openpose_engines_in_flight_on_one_device(pe, he_sd):
    eng = pkg_module("engine")
    rt = eng.NativeNet(0)
    rt.load_state_dict_arrays([v.numpy() for v in he_sd.values()])
    rpe = eng.PoseEngine.from_net(rt, batch_cap=8, peak_cap=1024, human_cap=2048)
    rs = np.random.RandomState(71)
    a = rs.randint(0, 256, (2, 90, 123, 3)).astype(np.uint8)
    b = rs.randint(0, 256, (3, 100, 80, 3)).astype(np.uint8)
    alone = {}
    for name, e, fr in (("rt", rpe, a), ("op", pe, b)):
        e.infer_raw_async_u8(fr.ctypes.data, False, len(fr), fr.shape[1], fr.shape[2], 96, 8, flip=True)
        alone[name] = [r.copy() for r in e.fetch_arrays()]
    for rep in range(2):
        tr = rpe.infer_raw_async_u8(a.ctypes.data, False, 2, 90, 123, 96, 8, flip=True)
        to = pe.infer_raw_async_u8(b.ctypes.data, False, 3, 100, 80, 96, 8, flip=True)
        tr2 = rpe.infer_raw_async_u8(a.ctypes.data, False, 2, 90, 123, 96, 8, flip=True)
        for name, e, t in (("rt", rpe, tr), ("op", pe, to), ("rt", rpe, tr2)):
            for g, w in zip(e.fetch_arrays(ticket=t), alone[name]):
                np.testing.assert_array_equal(g, w, err_msg="%s rep %d" % (name, rep))
    assert sum(len(r) for r in alone["op"]) + sum(len(r) for r in alone["rt"]) > 0


def test_refusals_name_the_architecture_and_leave_the_net_usable(pe, net):
    nat = _nat()
    eng = pkg_module("engine")
    frames = torch.from_numpy(np.random.RandomState(5).randint(0, 256, (1, 64, 64, 3)).astype(np.uint8)).cuda()
    before = _maps(net, "bf16", frames=frames)
    for mode in ("fp8", "fp16"):
        l0 = nat.launch_count()
        with pytest.raises(nat.B200PoseError, match=r"OpenPose_Model\(4, 2\).*%s" % mode):
            _maps(net, mode, frames=frames)
        assert nat.launch_count() == l0
        with pytest.raises(nat.B200PoseError, match=r"OpenPose_Model\(4, 2\).*%s" % mode):
            eng.PoseEngine.from_net(net, mode=mode)
        u8 = np.zeros((1, 64, 64, 3), np.uint8)      # the fused C entry points refuse too, before staging anything
        with pytest.raises(nat.B200PoseError, match=r"OpenPose_Model\(4, 2\).*%s" % mode):
            nat.check(nat.lib().b200pose_infer_u8(net._h, pe.post._h, u8.ctypes.data, 0, 1, 64, 64, nat.MODES[mode],
                                                  ctypes.c_float(0.1), None), "b200pose_infer_u8")
        assert nat.launch_count() == l0
    with pytest.raises(nat.B200PoseError, match=r"OpenPose_Model\(4, 2\)"):
        nat.check(nat.lib().b200pose_net_set_stages(net._h, 3), "b200pose_net_set_stages")
    with pytest.raises(nat.B200PoseError, match=r"OpenPose_Model\(4, 2\).*expected 36864"):
        nat.check(nat.lib().b200pose_net_set_tensor(net._h, 2, np.zeros(5, np.float32).ctypes.data, 5), "set_tensor")
    with pytest.raises(nat.B200PoseError, match="outputs\\[6\\] must be NULL"):
        outs = [torch.empty(1, device="cuda") for _ in range(7)]
        net.forward_u8_ptr(frames.data_ptr(), True, 1, 64, 64, 0, [o.data_ptr() for o in outs], True, 0)
    with pytest.raises(nat.B200PoseError, match="stages"):
        eng.PoseEngine.from_net(net, stages=3)
    after = _maps(net, "bf16", frames=frames)
    assert all(torch.equal(x, y) for x, y in zip(before, after))


# ------------------------------------------------------------------------------------------------ other layouts
# (l2, l1) beyond (4, 2): a PAF stage that is first and last (l2 = 1), a one-stage L1 branch that never reads
# cat[features, heat, paf] (l1 = 1), a heat map that feeds several L1 stages (l1 >= 3), all twelve outputs (l2 + l1 = 12)
LAYOUTS = [(1, 1), (1, 11), (11, 1), (2, 3), (6, 6)]
LAYOUT_IDS = ["%d-%d" % lay for lay in LAYOUTS]


@pytest.fixture(scope="module")
def layout_engines(built):
    """openpose_engine(sd, l2, l1) per layout, made when a test first asks for it; one layout at a time."""
    made = {}

    def get(layout):
        if layout not in made:
            made.clear()
            sd = openpose_port.he_state_dict(*layout)
            made[layout] = sd, pkg_module("engine").openpose_engine(sd, *layout, batch_cap=8, peak_cap=1024,
                                                                    human_cap=2048)
        return made[layout]
    return get


@pytest.mark.parametrize("layout", LAYOUTS, ids=LAYOUT_IDS)
def test_layout_fp32_is_bit_identical_to_the_exact_oracle_uniform_and_ragged(layout_engines, layout):
    """Every map the layout returns (at (1, 11) and (11, 1) all twelve output pointers) equals forward_exact; in a ragged
    batch, each frame's maps inside its extent equal the oracle's of that frame alone, and +0 beyond it."""
    sd, pe = layout_engines(layout)
    l2, l1 = layout
    x = _input(2, (64, 64), 5)
    got = _maps(pe.net, "fp32", x=x.cuda())
    want = openpose_port.forward_exact(sd, x.numpy(), l2, l1)
    assert len(got) == len(want) == l2 + l1
    for i, (g, w) in enumerate(zip(got, want)):
        np.testing.assert_array_equal(g.cpu().numpy(), w, err_msg="%s map %d" % (layout, i))
    rs = np.random.RandomState(13)
    shapes = [(64, 72), (48, 80), (72, 56)]
    frames = [rs.randint(0, 256, s + (3,)).astype(np.uint8) for s in shapes]
    packed = torch.from_numpy(np.concatenate([f.ravel() for f in frames])).cuda()
    got = _maps(pe.net, "fp32", frames=packed, shapes=shapes)
    for i, f in enumerate(frames):
        want = openpose_port.forward_exact(sd, glue_port.rtpose_preprocess(f)[None].astype(np.float32), l2, l1)
        h, w = f.shape[0] // 8, f.shape[1] // 8
        for m, (g, wm) in enumerate(zip(got, want)):
            g = g[i].cpu().numpy()
            np.testing.assert_array_equal(g[:, :h, :w], wm[0], err_msg="%s frame %d map %d" % (layout, i, m))
            assert not g[:, h:, :].any() and not g[:, :, w:].any(), (layout, i, m)


@pytest.mark.parametrize("mode,tol", [("bf16x3", 1e-3), ("bf16", 0.25)])
@pytest.mark.parametrize("layout", LAYOUTS, ids=LAYOUT_IDS)
def test_layout_against_the_reference_golden(layout_engines, layout, mode, tol):
    """Every saved map against the unmodified module's (tests/golden/openpose_<l2>_<l1>_64.npz), at the tolerances of
    test_368_against_the_reference_golden."""
    _, pe = layout_engines(layout)
    g = golden("openpose_%d_%d_64" % layout)
    x = torch.rand((1, 3, 64, 64), generator=torch.Generator().manual_seed(int(g["seed"]))) - 0.5
    outs = _maps(pe.net, mode, x=x.cuda())
    errs = [float(np.abs(o.cpu().numpy() - g["maps_%d" % i]).max()) for i, o in enumerate(outs)]
    print("OpenPose_Model(%d, %d) %s @64: max|err| per map %s (maps up to %.1f)"
          % (layout + (mode, " ".join("%.1e" % e for e in errs), float(np.max(g["stage_absmax"])))))
    assert len(outs) == sum(layout) and max(errs) < tol, errs


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("layout", LAYOUTS, ids=LAYOUT_IDS)
def test_layout_ragged_frames_equal_each_frame_alone(layout_engines, layout, mode):
    _, pe = layout_engines(layout)
    rs = np.random.RandomState(9)
    shapes = [(64, 72), (48, 80), (72, 56)]
    frames = [rs.randint(0, 256, s + (3,)).astype(np.uint8) for s in shapes]
    packed = torch.from_numpy(np.concatenate([f.ravel() for f in frames])).cuda()
    rag = _maps(pe.net, mode, frames=packed, shapes=shapes)
    for i, f in enumerate(frames):
        alone = _maps(pe.net, mode, frames=torch.from_numpy(f[None]).cuda())
        h, w = f.shape[0] // 8, f.shape[1] // 8
        for m, (a, b) in enumerate(zip(rag, alone)):
            assert torch.equal(a[i, :, :h, :w], b[0]), (layout, mode, i, m)
            assert not a[i, :, h:, :].any() and not a[i, :, :, w:].any(), (layout, mode, i, m)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("layout", [(1, 1), (6, 6)], ids=["1-1", "6-6"])
def test_layout_fused_entry_points_equal_the_composed_path(layout_engines, layout, mode):
    _, pe0 = layout_engines(layout)
    pe = _engine(pe0.net, mode)
    ref = pkg_module("engine").NativePost(0, batch_cap=8, peak_cap=1024, human_cap=2048)
    rs = np.random.RandomState(62)
    frames = rs.randint(0, 256, (2, 96, 128, 3)).astype(np.uint8)
    mixed = [rs.randint(0, 256, s + (3,)).astype(np.uint8) for s in ((90, 123), (120, 100))]
    assert _check_u8_flip_and_ragged(pe, ref, pe.net, mode, frames, mixed) > 0
