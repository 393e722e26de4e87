"""GPU (-m gpu): COCO training targets and stage losses on the device (DESIGN.md 2.19; engine.ground_truth,
NativeNet.stage_losses, PoseEngine.validation_loss).  Targets bit for bit the host build of csrc/gt_core.h (itself bit
for bit the reference's goldens) on every golden and on seeded uniform and ragged batches; the loss sums against numpy
and torch.nn.MSELoss, independent of the canvas and of the batch's other frames; stage counts 1 .. 6, bf16 / fp32 and
OpenPose_Model(4, 2); validation_loss against the composed path; refusals; launch counts."""
import numpy as np
import pytest
import torch

import gt_check as gc
import gt_port
import openpose_port
from conftest import pkg_module

pytestmark = pytest.mark.gpu


def _eng():
    return pkg_module("engine")


def _nat():
    return pkg_module("_native")


@pytest.fixture(scope="module")
def core(built, tmp_path_factory):
    return gc.compile_core(str(tmp_path_factory.mktemp("gt") / "libgtcore.so"))


@pytest.fixture(scope="module")
def net(built, he_sd):
    n = _eng().NativeNet(0)
    n.load_state_dict_arrays([v.numpy() for v in he_sd.values()])
    return n


def _bits_equal(a, b):
    return np.array_equal(gc.bits(np.ascontiguousarray(a)), gc.bits(np.ascontiguousarray(b)))


def _gt(kps, sizes, canvas=None):
    heat, paf = _eng().ground_truth(kps, sizes, 0, canvas)
    torch.cuda.synchronize()
    return heat.cpu().numpy(), paf.cpu().numpy()


@pytest.mark.parametrize("name", sorted(gc.goldens()))
def test_kernels_equal_core_and_golden(core, name):
    g = gc.goldens()[name]
    heat, paf = _gt([g["kp"]], [tuple(g["size"])])
    ch, cp = gc.core_gt(core, [g["kp"]], [tuple(g["size"])])
    assert _bits_equal(heat, ch) and _bits_equal(paf, cp)
    assert _bits_equal(heat[0], g["heat"]) and _bits_equal(paf[0], g["paf"])


@pytest.mark.parametrize("seed,n,sizes", [(1, 32, ((368, 368),)), (2, 7, ((368, 368), (368, 656), (656, 368))),
                                          (3, 12, ((64, 128), (100, 36), (368, 248), (8, 8), (17, 23)))])
def test_random_batches_equal_core_and_each_frame_alone(core, seed, n, sizes):
    kps, hw = gc.random_scenario(seed, n, sizes, max_persons=9)
    heat, paf = _gt(kps, hw)
    ch, cp = gc.core_gt(core, kps, hw)
    assert _bits_equal(heat, ch) and _bits_equal(paf, cp)
    ph, pp = gt_port.ground_truth_batch(kps, hw)
    assert _bits_equal(heat, ph) and _bits_equal(paf, pp)
    for i, (h, w) in enumerate(hw):
        gh, gw = h // 8, w // 8
        ah, ap = _gt([kps[i]], [(h, w)])
        assert _bits_equal(heat[i, :, :gh, :gw], ah[0]) and _bits_equal(paf[i, :, :gh, :gw], ap[0])
        for m in (heat[i], paf[i]):
            assert not np.any(gc.bits(m[:, gh:])) and not np.any(gc.bits(m[:, :, gw:]))      # +0, not -0


def test_no_persons_and_a_larger_canvas(core):
    heat, paf = _gt([np.zeros((0, 17, 3), np.float32)], [(64, 64)], canvas=(10, 12))
    assert heat.shape == (1, 19, 10, 12) and np.all(heat[0, 18, :8, :8] == 1) and not np.any(gc.bits(paf))
    assert not np.any(gc.bits(heat[0, :18])) and not np.any(gc.bits(heat[0, 18, 8:])) and not np.any(gc.bits(heat[0, 18, :, 8:]))


def test_ground_truth_launches_two_kernels():
    nat = _nat()
    kps, hw = gc.random_scenario(4, 5, ((368, 368), (256, 368)))
    _gt(kps, hw)
    l0 = nat.launch_count()
    _gt(kps, hw)
    assert nat.launch_count() - l0 == 2


def _frames(n, hw, seed):
    return np.random.RandomState(seed).randint(0, 256, (n,) + hw + (3,), dtype=np.uint8)


def _forward(net, mode, frames, shapes=None):
    """The stage maps (device tensors) of a uniform ([n,H,W,3]) or ragged (list of [h,w,3]) forward of uint8 frames."""
    nat = _nat()
    names, is_paf = net.stage_map_names()
    if shapes is None:
        n, H, W = frames.shape[:3]
    else:
        n, H, W = len(shapes), max(s[0] for s in shapes), max(s[1] for s in shapes)
    outs = [torch.empty((n, 38 if p else 19, H // 8, W // 8), device="cuda") for p in is_paf]
    ptrs = [o.data_ptr() for o in outs] + [0] * (12 - len(outs))
    stream = torch.cuda.current_stream().cuda_stream
    if shapes is None:
        net.forward_u8_ptr(frames.ctypes.data, False, n, H, W, nat.MODES[mode], ptrs, True, stream)
    else:
        packed = np.concatenate([f.ravel() for f in frames])
        net.forward_ragged_u8_ptr(packed.ctypes.data, False, shapes, nat.MODES[mode], ptrs, True, stream)
    torch.cuda.synchronize()
    return outs


def _targets(shapes, seed, canvas=None):
    kps, _ = gc.random_scenario(seed, len(shapes), ((368, 368),), max_persons=5)
    kps = [k * np.array([s[1] / 368, s[0] / 368, 1], np.float32) for k, s in zip(kps, shapes)]
    return kps, _eng().ground_truth(kps, shapes, 0, canvas)


def _check_sums(net, outs, heat, paf, shapes):
    names, is_paf = net.stage_map_names()
    sums, ext, cells, got_names = net.stage_loss_sums(heat, paf)
    assert got_names == (names, is_paf) and cells == [(h // 8) * (w // 8) for h, w in shapes]
    th, tp = heat.cpu().numpy(), paf.cpu().numpy()
    for m, (o, p) in enumerate(zip(outs, is_paf)):
        pred, tgt = o.cpu().numpy(), tp if p else th
        for i, (h, w) in enumerate(shapes):
            d = pred[i, :, :h // 8, :w // 8] - tgt[i, :, :h // 8, :w // 8]
            want = np.sum((d * d).astype(np.float64))
            assert abs(sums[i, m] - want) <= 1e-12 * abs(want), (names[m], i, sums[i, m], want)
        if m == len(outs) - 1 or m == max(k for k, q in enumerate(is_paf) if q):
            sel = [pred[i, :(18 if not p else 38), :h // 8, :w // 8] for i, (h, w) in enumerate(shapes)]
            got = ext[:, 2:] if p else ext[:, :2]
            assert np.array_equal(got[:, 0], [s.max() for s in sel]) and np.array_equal(got[:, 1], [s.min() for s in sel])
    return sums


@pytest.mark.parametrize("mode", ["bf16", "fp32"])
@pytest.mark.parametrize("k", [1, 2, 3, 4, 5, 6])
def test_stage_losses_match_numpy_and_mse_loss(net, mode, k):
    net.set_stages(k)
    try:
        frames = _frames(3, (128, 96), 10 + k)
        outs = _forward(net, mode, frames)
        shapes = [(128, 96)] * 3
        _, (heat, paf) = _targets(shapes, k)
        _check_sums(net, outs, heat, paf, shapes)
        got = net.stage_losses(heat, paf)
        names, is_paf = net.stage_map_names()
        assert list(got)[:len(names)] == names and len(names) == 2 * k
        assert list(got)[len(names):] == ["total_loss", "max_ht", "min_ht", "max_paf", "min_paf"]
        mse = torch.nn.MSELoss(reduction="mean").cuda()
        for name, o, p in zip(names, outs, is_paf):
            want = mse(o, paf if p else heat).item()
            assert abs(got[name] - want) <= 1e-5 * abs(want), (name, got[name], want)
        assert got["max_ht"] == outs[-1][:, :18].max().item() and got["min_ht"] == outs[-1][:, :18].min().item()
        assert got["max_paf"] == outs[-2].max().item() and got["min_paf"] == outs[-2].min().item()
        assert got["total_loss"] == sum(got[n] for n in names)
    finally:
        net.set_stages(6)


def test_stage_losses_of_openpose_model(built):
    sd = openpose_port.he_state_dict(4, 2)
    pe = _eng().openpose_engine(sd, 4, 2, batch_cap=4)
    net = pe.net
    frames = _frames(2, (96, 128), 5)
    outs = _forward(net, "bf16", frames)
    shapes = [(96, 128)] * 2
    _, (heat, paf) = _targets(shapes, 6)
    _check_sums(net, outs, heat, paf, shapes)
    got = net.stage_losses(heat, paf)
    assert list(got)[:6] == ["loss_paf_1", "loss_paf_2", "loss_paf_3", "loss_paf_4", "loss_heat_1", "loss_heat_2"]
    mse = torch.nn.MSELoss().cuda()
    assert abs(got["loss_heat_2"] - mse(outs[5], heat).item()) <= 1e-5 * got["loss_heat_2"]
    assert got["max_paf"] == outs[3].max().item() and got["min_ht"] == outs[5][:, :18].min().item()


@pytest.mark.parametrize("mode", ["bf16", "fp32"])
def test_sums_do_not_depend_on_canvas_or_companions(net, mode):
    shapes = [(128, 96), (64, 128), (200, 64)]
    frames = [_frames(1, s, 20 + i)[0] for i, s in enumerate(shapes)]
    kps, _ = _targets(shapes, 7)
    per_image = {}
    # each frame alone, the three as one ragged batch, and two other compositions (other canvases, other neighbours)
    for batch in ([0], [1], [2], [0, 1, 2], [2, 0], [1, 2, 1]):
        sh = [shapes[i] for i in batch]
        if len(batch) == 1:
            _forward(net, mode, frames[batch[0]][None])
        else:
            _forward(net, mode, [frames[i] for i in batch], sh)
        heat, paf = _eng().ground_truth([kps[i] for i in batch], sh, 0,
                                        (max(h for h, _ in sh) // 8, max(w for _, w in sh) // 8))
        sums, ext, _, _ = net.stage_loss_sums(heat, paf)
        for j, i in enumerate(batch):
            got = (gc.bits(sums[j]).tobytes(), gc.bits(ext[j]).tobytes())
            assert per_image.setdefault(i, got) == got, (batch, i)


def test_validation_loss_equals_the_composed_path(net, he_sd):
    eng = _eng()
    pe = eng.PoseEngine.from_net(net, mode="bf16", batch_cap=3)
    rs = np.random.RandomState(3)
    srcs = [(240, 320), (300, 200), (240, 320), (480, 640), (123, 77)]
    images = [rs.randint(0, 256, s + (3,), dtype=np.uint8) for s in srcs]
    kps = [gc.random_scenario(30 + i, 1, (s,), max_persons=4)[0][0] for i, s in enumerate(srcs)]
    got = pe.validation_loss(images, kps)
    # composed: device crop -> forward -> ground_truth -> stage_losses, batch by batch
    geo = [_nat().crop_geometry(s[0], s[1], 368, 8) for s in srcs]
    names = net.stage_map_names()
    sums, ext, cells = 0.0, [], 0
    for part in eng.plan_ragged_batches([g[2] for g in geo], 3):
        crops = [net.crop_with_factor(images[i])[0] for i in part]
        sh = [c.shape[:2] for c in crops]
        outs = _forward(net, "bf16", np.stack(crops) if len(set(sh)) == 1 else crops, None if len(set(sh)) == 1 else sh)
        mapped = []
        for i in part:
            (rh, rw), k = geo[i][1], kps[i].astype(np.float32).copy()
            k[:, :, 0] = (k[:, :, 0] + np.float32(0.5)) * np.float32(rw / srcs[i][1]) - np.float32(0.5)
            k[:, :, 1] = (k[:, :, 1] + np.float32(0.5)) * np.float32(rh / srcs[i][0]) - np.float32(0.5)
            mapped.append(k)
        heat, paf = eng.ground_truth(mapped, sh, 0, tuple(outs[0].shape[2:]))
        s, e, c, _ = net.stage_loss_sums(heat, paf)
        sums = sums + s.sum(0)
        ext.append(e)
        cells += sum(c)
    want = eng._loss_dict(names, sums, np.concatenate(ext), cells)
    assert list(got) == list(want)
    for k in want:
        assert np.float64(got[k]).tobytes() == np.float64(want[k]).tobytes(), k


def test_refusals_name_their_argument_and_leave_the_net_usable(built, he_sd):
    eng, nat = _eng(), _nat()
    fresh = eng.NativeNet(0)
    fresh.load_state_dict_arrays([v.numpy() for v in he_sd.values()])
    shapes = [(64, 64)]
    heat, paf = eng.ground_truth([np.zeros((0, 17, 3), np.float32)], shapes)
    with pytest.raises(nat.B200PoseError, match="stage_losses: no forward has run"):
        fresh.stage_losses(heat, paf)
    outs = _forward(fresh, "bf16", _frames(1, (64, 64), 1))
    with pytest.raises(nat.B200PoseError, match="paf must be"):
        fresh.stage_losses(heat, paf[:, :19])
    with pytest.raises(nat.B200PoseError, match="keypoints"):
        eng.ground_truth([np.full((2, 17, 3), np.inf, np.float32)], shapes)
    with pytest.raises(nat.B200PoseError, match="sizes of image 1"):
        eng.ground_truth([np.zeros((0, 17, 3))] * 2, [(64, 64), (64, 7)])
    with pytest.raises(nat.B200PoseError, match="persons of image 0 = 257"):
        eng.ground_truth([np.zeros((257, 17, 3))], shapes)
    with pytest.raises(nat.B200PoseError, match="canvas"):
        eng.ground_truth([np.zeros((0, 17, 3))], shapes, 0, (4, 8))
    l0 = nat.launch_count()
    got = fresh.stage_losses(heat, paf)
    assert nat.launch_count() - l0 == 1
    assert got["loss_stage6_L2"] == torch.nn.MSELoss()(outs[11], heat).item() or \
        abs(got["loss_stage6_L2"] - torch.nn.MSELoss()(outs[11], heat).item()) <= 1e-5 * got["loss_stage6_L2"]


def test_losses_follow_the_last_forward_not_the_stage_setting(net):
    """The map count comes from the forward that ran: a set_stages after it changes neither the keys nor the sums."""
    nat = _nat()
    frames = _frames(2, (96, 96), 40)
    shapes = [(96, 96)] * 2
    _, (heat, paf) = _targets(shapes, 41)
    try:
        for ran, later in ((6, 3), (3, 6)):
            net.set_stages(ran)
            outs = _forward(net, "bf16", frames)
            want = net.stage_losses(heat, paf)
            net.set_stages(later)
            got = net.stage_losses(heat, paf)
            assert list(got) == list(want) and len([k for k in got if k.startswith("loss_stage")]) == 2 * ran
            assert all(np.float64(got[k]).tobytes() == np.float64(want[k]).tobytes() for k in want)
            mse = torch.nn.MSELoss()
            assert abs(got["loss_stage%d_L2" % ran] - mse(outs[-1], heat).item()) <= 1e-5 * got["loss_stage%d_L2" % ran]
            assert net.last_forward()[3] == 2 * ran
        # a C caller whose sums row does not match the forward's map count is refused before anything runs
        sums = torch.zeros((2, 6), dtype=torch.float64, device="cuda")
        ext = torch.zeros((2, 4), device="cuda")
        rc = nat.lib().b200pose_net_stage_losses(net._h, heat.data_ptr(), paf.data_ptr(), sums.data_ptr(), 12,
                                                 ext.data_ptr(), None)
        assert rc != 0 and "maps = 12, but the last forward wrote 6" in nat.lib().b200pose_last_error().decode()
        torch.cuda.synchronize()
        assert not sums.any()
    finally:
        net.set_stages(6)


def test_losses_after_a_fused_ragged_run_use_its_extents(net, he_sd):
    """A ragged forward run by the engine's fused entry point: the cell counts are that forward's frames' own."""
    eng = _eng()
    pe = eng.PoseEngine.from_net(net, mode="bf16", batch_cap=4)
    rs = np.random.RandomState(8)
    srcs = [(200, 300), (300, 200), (150, 150)]
    images = [rs.randint(0, 256, s + (3,), dtype=np.uint8) for s in srcs]
    _forward(net, "bf16", _frames(1, (64, 64), 1))      # a uniform forward first: its extents must not be reused
    packed = np.concatenate([im.ravel() for im in images])
    pe.infer_raw_ragged_async_u8(packed.ctypes.data, False, srcs)
    pe.fetch()
    n, H, W, maps, extents = net.last_forward()
    pads = [_nat().crop_geometry(h, w, 368, 8)[2] for h, w in srcs]
    assert n == 3 and extents == pads and (H, W) == (max(p[0] for p in pads), max(p[1] for p in pads))
    assert len(set(pads)) == 3 and maps == 12
    kps, _ = gc.random_scenario(9, n, ((368, 368),), max_persons=3)
    heat, paf = eng.ground_truth(kps, extents, 0, (H // 8, W // 8))
    sums, ext, cells, (names, is_paf) = net.stage_loss_sums(heat, paf)
    assert cells == [(h // 8) * (w // 8) for h, w in extents]
    got = net.stage_losses(heat, paf)
    for m, (name, p) in enumerate(zip(names, is_paf)):
        assert got[name] == float(sums[:, m].sum()) / ((38 if p else 19) * sum(cells))


def test_validation_loss_refuses_an_empty_list(net):
    eng, nat = _eng(), _nat()
    pe = eng.PoseEngine.from_net(net, mode="bf16", batch_cap=4)
    with pytest.raises(nat.B200PoseError, match="images is empty"):
        pe.validation_loss([], [])
