"""GPU (-m gpu): peak refinement modes and up-sampling factors (b200pose_post_set_refine, b200pose_post_run_scaled).
For every factor and mode the device's peaks equal the oracle's NMS (tests/nms_modes_port.py) bit for bit and its persons
the C port of pafprocess on the xf nearest maps, from host maps in either layout and from device tensors, and agree
with what the reference itself made of the same maps (tests/golden/nms_modes.npz); the drop-in NMS / paf_to_pose_cpp
give the reference's results; fused runs refine with their post object's mode; two runs in flight keep their own mode;
a run above the coordinate bound is refused by name and the object stays usable."""
import numpy as np
import pytest
import torch

import nms_modes_port as nmp
from conftest import assert_humans_equal, golden, humans_rows_to_dicts, pkg_module
from oracle import nms_port, pafprocess_oracle

pytestmark = pytest.mark.gpu

FACTORS = (1, 2, 3, 4, 5, 7, 8, 16)
GOLDEN_SCORE_TOL = 1e-6      # see tests/test_refine_host.py: IPP's cubic arithmetic on the stick-figure fixtures
THRESH = nmp.GOLDEN_THRESH


@pytest.fixture(scope="module")
def eng(built):
    return pkg_module("engine")


@pytest.fixture(scope="module")
def maps():
    return nmp.scenarios()


@pytest.fixture(scope="module")
def port():
    return pafprocess_oracle.load_port()


def _want(port, heat, paf, f, mode):
    refine, gauss = nmp.MODES[mode]
    jl, humans = nmp.paf_to_pose(heat, paf, port, thresh=THRESH, upsample=f, refine=refine, gauss=gauss)
    return nmp.device_joint_list(jl), humans


def _check(eng, post, i, heat, f, want, what):
    jl, humans = want
    h, w = heat.shape[:2]
    assert post.status(i) == 0, what
    np.testing.assert_array_equal(post.peaks(i), jl, err_msg=str(what))
    assert_humans_equal(eng.humans_to_dicts(post.humans(i), w * f, h * f), humans, score_tol=0.0)
    return len(humans)


def _check_golden(peaks, name, f, mode, g):
    """The device's peaks against the reference's NMS: positions identical (as pafprocess reads them), scores within
    GOLDEN_SCORE_TOL."""
    ref = nmp.device_joint_list(g[nmp.golden_key(name, f, mode) + "_joint_list"])
    assert peaks.shape == ref.shape, (name, f, mode)
    np.testing.assert_array_equal(peaks[:, [0, 1, 3, 4]], ref[:, [0, 1, 3, 4]], err_msg=str((name, f, mode)))
    np.testing.assert_allclose(peaks[:, 2], ref[:, 2], rtol=0, atol=GOLDEN_SCORE_TOL, err_msg=str((name, f, mode)))


@pytest.mark.parametrize("mode", list(nmp.MODES))
@pytest.mark.parametrize("f", FACTORS)
def test_factor_and_mode_equal_the_oracle(f, mode, eng, maps, port):
    want = {k: _want(port, heat, paf, f, mode) for k, (heat, paf) in maps.items()}
    g = golden("nms_modes")
    gold = set(nmp.golden_scenarios()) if f in nmp.GOLDEN_FACTORS else set()
    post = eng.NativePost(0, batch_cap=4, peak_cap=2048, human_cap=2048)
    post.set_refine(mode)
    assert post.refine() == mode
    persons = 0
    for k, (heat, paf) in maps.items():             # layout 1 from the host
        h, w = heat.shape[:2]
        post.run(np.ascontiguousarray(heat).ctypes.data, np.ascontiguousarray(paf).ctypes.data, False, 1, 1, h, w,
                 THRESH, upsample=f)
        post.sync()
        persons += _check(eng, post, 0, heat, f, want[k], (f, mode, k, "layout 1"))
        if k in gold:
            _check_golden(post.peaks(0), k, f, mode, g)
    shapes = {}
    for k, (heat, _) in maps.items():
        shapes.setdefault(heat.shape[:2], []).append(k)
    for (h, w), keys in sorted(shapes.items()):     # layout 0 as batches of one shape
        for b in range(0, len(keys), 4):
            ks = keys[b:b + 4]
            heats = np.ascontiguousarray(np.stack([maps[k][0] for k in ks]).transpose(0, 3, 1, 2))
            pafs = np.ascontiguousarray(np.stack([maps[k][1] for k in ks]).transpose(0, 3, 1, 2))
            post.run(heats.ctypes.data, pafs.ctypes.data, False, 0, len(ks), h, w, THRESH, upsample=f)
            post.sync()
            for i, k in enumerate(ks):
                _check(eng, post, i, maps[k][0], f, want[k], (f, mode, k, "layout 0"))
    keys = shapes[(46, 46)][:4]                     # device tensors, layout 1
    heat = torch.from_numpy(np.stack([maps[k][0] for k in keys])).cuda().contiguous()
    paf = torch.from_numpy(np.stack([maps[k][1] for k in keys])).cuda().contiguous()
    torch.cuda.synchronize()
    post.run(heat.data_ptr(), paf.data_ptr(), True, 1, len(keys), 46, 46, THRESH, torch.cuda.current_stream().cuda_stream,
             upsample=f)
    post.sync()
    for i, k in enumerate(keys):
        _check(eng, post, i, maps[k][0], f, want[k], (f, mode, k, "on device"))
    print(f, mode, "persons", persons)
    assert persons > 0


# ------------------------------------------------------------------------------------------------ the drop-in
class _Cfg:
    class MODEL:
        DOWNSAMPLE = 8
        NUM_KEYPOINTS = 18

    class TEST:
        THRESH_HEATMAP = THRESH


@pytest.mark.parametrize("f", nmp.GOLDEN_FACTORS)
def test_dropin_equals_the_reference(f, built):
    """paf_to_pose_cpp with MODEL.DOWNSAMPLE = f and NMS with each flag combination against the reference's results."""
    p2p = pkg_module("lib.utils.paf_to_pose")
    g = golden("nms_modes")
    _Cfg.MODEL.DOWNSAMPLE = f
    try:
        for name, (heat, paf) in nmp.golden_scenarios().items():
            for mode, (refine, gauss) in nmp.MODES.items():
                key = nmp.golden_key(name, f, mode)
                got = nms_port.joint_list_from_nms(p2p.NMS(heat, upsampFactor=f, bool_refine_center=refine,
                                                           bool_gaussian_filt=gauss, config=_Cfg))
                ref = g[key + "_joint_list"]
                np.testing.assert_array_equal(got[:, [0, 1, 3, 4]], ref[:, [0, 1, 3, 4]], err_msg=key)
                np.testing.assert_allclose(got[:, 2], ref[:, 2], rtol=0, atol=GOLDEN_SCORE_TOL, err_msg=key)
            # refine=False ignores the Gaussian flag, as in the reference
            a = p2p.NMS(heat, upsampFactor=f, bool_refine_center=False, bool_gaussian_filt=True, config=_Cfg)
            b = p2p.NMS(heat, upsampFactor=f, bool_refine_center=False, bool_gaussian_filt=False, config=_Cfg)
            assert all(np.array_equal(x, y) for x, y in zip(a, b))
            humans = p2p.paf_to_pose_cpp(heat, paf, _Cfg)
            got = [(h.score, {p: (bp.x, bp.y, bp.score) for p, bp in h.body_parts.items()}) for h in humans]
            assert_humans_equal(got, humans_rows_to_dicts(g[nmp.golden_key(name, f, "cubic") + "_humans"]),
                                score_tol=GOLDEN_SCORE_TOL)
    finally:
        _Cfg.MODEL.DOWNSAMPLE = 8


# ------------------------------------------------------------------------------------------------ fused runs
@pytest.fixture(scope="module")
def net(built, he_sd):
    n = pkg_module("engine").NativeNet(0)
    n.load_state_dict_arrays([v.numpy() for v in he_sd.values()])
    return n


def _debug_maps(pe, n, h, w):
    nat = pkg_module("_native")
    heat = np.empty((n, 19, h, w), np.float32)
    paf = np.empty((n, 38, h, w), np.float32)
    nat.check(nat.lib().b200pose_post_debug_maps(pe.post._h, heat.ctypes.data, heat.size, paf.ctypes.data, paf.size),
              "b200pose_post_debug_maps")
    return heat, paf


@pytest.mark.parametrize("mode", ["gauss", "none"])
def test_fused_runs_refine_with_the_mode(mode, eng, net, port):
    """A ragged batch with flip, and four scales with flip: each frame's peaks and persons equal the oracle applied to the
    maps the fused run post-processed (b200pose_post_debug_maps, the frame's own extent of the canvas)."""
    nat = pkg_module("_native")
    pe = eng.PoseEngine.from_net(net, mode="bf16", batch_cap=4, peak_cap=1024, human_cap=2048, refine=mode)
    assert pe.post.refine() == mode
    rs = np.random.RandomState(7)
    frames = [rs.randint(0, 256, s + (3,)).astype(np.uint8) for s in ((90, 123), (70, 150), (96, 97))]
    packed = np.concatenate([f.ravel() for f in frames])
    shapes = [f.shape[:2] for f in frames]
    calls = [(96, lambda: pe.infer_raw_ragged_async_u8(packed.ctypes.data, False, shapes, 96, 8, 0.05, flip=True)),
             (64, lambda: pe.infer_raw_multiscale_ragged_async_u8(packed.ctypes.data, False, shapes, (0.5, 1.0, 1.5, 2.0),
                                                                  64, 8, 0.05, flip=True))]
    refine, gauss = nmp.MODES[mode]
    peaks_total = 0
    for dest, call in calls:
        call()
        rows = [r.copy() for r in pe.fetch_arrays()]
        pads = [nat.crop_geometry(h, w, dest, 8)[2] for h, w in shapes]
        heat, paf = _debug_maps(pe, len(frames), max(p[0] for p in pads) // 8, max(p[1] for p in pads) // 8)
        for i, (ph, pw) in enumerate(pads):
            h, w = ph // 8, pw // 8
            hh = np.ascontiguousarray(heat[i, :, :h, :w].transpose(1, 2, 0))
            pp = np.ascontiguousarray(paf[i, :, :h, :w].transpose(1, 2, 0))
            jl, humans = nmp.paf_to_pose(hh, pp, port, thresh=0.05, upsample=8, refine=refine, gauss=gauss)
            np.testing.assert_array_equal(pe.post.peaks(i), nmp.device_joint_list(jl), err_msg="%s %d %d" % (mode, dest, i))
            assert_humans_equal(eng.humans_to_dicts(rows[i], pw, ph), humans, score_tol=0.0)
            peaks_total += len(jl)
    print(mode, "fused peaks", peaks_total)
    assert peaks_total > 0


# ------------------------------------------------------------------------------------------------ runs in flight, refusals
def test_two_runs_in_flight_keep_their_mode(eng, maps, port):
    keys = ["p3", "p30"]
    heats = np.ascontiguousarray(np.stack([maps[k][0] for k in keys]))
    pafs = np.ascontiguousarray(np.stack([maps[k][1] for k in keys]))
    post = eng.NativePost(0, batch_cap=2, peak_cap=2048, human_cap=2048)
    tickets = {}
    for mode in ("gauss", "none"):
        post.set_refine(mode)
        post.run(heats.ctypes.data, pafs.ctypes.data, False, 1, len(keys), 46, 46, THRESH, upsample=4)
        tickets[mode] = post.last_ticket()
    for mode, t in tickets.items():
        post.select(t)
        for i, k in enumerate(keys):
            want = _want(port, maps[k][0], maps[k][1], 4, mode)
            h, w = maps[k][0].shape[:2]
            jl, humans = want
            assert_humans_equal(eng.humans_to_dicts(post.humans(i), w * 4, h * 4), humans, score_tol=0.0)
    np.testing.assert_array_equal(post.peaks(1), _want(port, maps["p30"][0], maps["p30"][1], 4, "none")[0])


def test_refusals_leave_the_object_usable(eng, maps, port):
    nat = pkg_module("_native")
    post = eng.NativePost(0, batch_cap=1, peak_cap=2048, human_cap=2048)
    with pytest.raises(nat.B200PoseError, match="7"):
        nat.check(nat.lib().b200pose_post_set_refine(post._h, 7), "b200pose_post_set_refine")
    assert post.refine() == "cubic"
    with pytest.raises(nat.B200PoseError):
        post.set_refine("bilinear")
    heat = np.zeros((16, 1025, 19), np.float32)
    paf = np.zeros((16, 1025, 38), np.float32)
    with pytest.raises(nat.B200PoseError, match="16400"):      # 1025 x 16 > 16384
        post.run(heat.ctypes.data, paf.ctypes.data, False, 1, 1, 16, 1025, THRESH, upsample=16)
    heat, paf = maps["p30"]
    post.set_refine("gauss")
    post.run(np.ascontiguousarray(heat).ctypes.data, np.ascontiguousarray(paf).ctypes.data, False, 1, 1, 46, 46, THRESH,
             upsample=16)
    post.sync()
    _check(eng, post, 0, heat, 16, _want(port, heat, paf, 16, "gauss"), "after a refusal")
