"""GPU (-m gpu): multi-scale (+ flip) test-time averaging on ragged batches (DESIGN.md 2.7) - frames of different sizes
averaged over four scales in one device batch per scale.  Every frame must come out bit for bit as
b200pose_infer_raw_u8_multiscale gives it for that frame alone, and the averaged maps must be +0 outside each frame."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import assert_humans_equal, pkg_module
from oracle import glue_port, pafprocess_oracle

pytestmark = pytest.mark.gpu

SCALES = (0.5, 1.0, 1.5, 2.0)
BASE = 96
# raw sizes: both orientations; (70, 150) alone sets the canvas width and (150, 70) its height at every scale; (96, 97)
# and (96, 104) pad to 48 x 48 and 48 x 56 at 0.5x but both to 96 x 104 at 1.0x; (64, 64) sits far inside the canvas
RAW = [(96, 97), (96, 104), (70, 150), (150, 70), (90, 123), (123, 90), (64, 64), (100, 110), (61, 88)]
LARGE = [(70, 150), (150, 70), (60, 180), (180, 64)]
SMALL = [(96, 97), (96, 104), (90, 123)]      # landscape only: (90, 123) is the whole canvas at every scale


def _nat():
    return pkg_module("_native")


def _pads(shapes, dest):
    return [_nat().crop_geometry(h, w, dest, 8)[2] for h, w in shapes]


def _frames(shapes, seed):
    rs = np.random.RandomState(seed)
    return [rs.randint(0, 256, s + (3,)).astype(np.uint8) for s in shapes]


@pytest.fixture(scope="module")
def net(built, he_sd):
    eng = pkg_module("engine")
    n = eng.NativeNet(0)
    n.load_state_dict_arrays([v.numpy() for v in he_sd.values()])
    return n


def _engine(net, mode="bf16", batch_cap=16):
    return pkg_module("engine").PoseEngine.from_net(net, mode=mode, batch_cap=batch_cap, peak_cap=1024, human_cap=2048)


def _debug_maps(pe, n, h, w):
    nat = _nat()
    heat = np.empty((n, 19, h, w), np.float32)
    paf = np.empty((n, 38, h, w), np.float32)
    nat.check(nat.lib().b200pose_post_debug_maps(pe.post._h, heat.ctypes.data, heat.size, paf.ctypes.data, paf.size),
              "b200pose_post_debug_maps")
    return heat, paf


def _ragged(pe, frames, flip, thresh=0.1):
    """Rows, peaks and averaged maps (base canvas) of one ragged multi-scale call."""
    shapes = [f.shape[:2] for f in frames]
    packed = np.concatenate([f.ravel() for f in frames])
    pe.infer_raw_multiscale_ragged_async_u8(packed.ctypes.data, False, shapes, SCALES, BASE, 8, thresh, flip)
    rows = [r.copy() for r in pe.fetch_arrays()]
    peaks = [pe.post.peaks(i) for i in range(len(frames))]
    pads = _pads(shapes, BASE)
    heat, paf = _debug_maps(pe, len(frames), max(p[0] for p in pads) // 8, max(p[1] for p in pads) // 8)
    return rows, peaks, heat, paf


def _alone(pe, frame, flip, thresh=0.1):
    """The same of b200pose_infer_raw_u8_multiscale on one frame."""
    h, w = frame.shape[:2]
    buf = np.ascontiguousarray(frame[None])
    pe.infer_raw_multiscale_async_u8(buf.ctypes.data, False, 1, h, w, SCALES, BASE, 8, thresh, flip)
    rows = pe.fetch_arrays()[0].copy()
    peaks = pe.post.peaks(0)
    (ph, pw), = _pads([(h, w)], BASE)
    heat, paf = _debug_maps(pe, 1, ph // 8, pw // 8)
    return rows, peaks, heat[0], paf[0]


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _assert_frames_equal(got, want, shapes, what=""):
    rows, peaks, heat, paf = got
    for i, (ph, pw) in enumerate(_pads(shapes, BASE)):
        msg = "%s frame %d %s" % (what, i, shapes[i])
        np.testing.assert_array_equal(rows[i], want[i][0], err_msg=msg)
        np.testing.assert_array_equal(peaks[i], want[i][1], err_msg=msg)
        h, w = ph // 8, pw // 8
        for m, ref in ((heat, want[i][2]), (paf, want[i][3])):
            assert np.array_equal(_bits(m[i, :, :h, :w]), _bits(ref)), msg
            assert not _bits(m[i, :, h:, :]).any() and not _bits(m[i, :, :h, w:]).any(), msg     # +0 outside


def test_frame_set_covers_the_ragged_edge_cases(built):
    for s in SCALES:
        pads = _pads(RAW, int(BASE * s))
        hs, ws = [p[0] for p in pads], [p[1] for p in pads]
        assert hs.count(max(hs)) == 1 and ws.count(max(ws)) == 1, s           # one frame alone sets each canvas edge
        assert len({h > w for h, w in RAW}) == 2
        small = _pads([(64, 64)], int(BASE * s))[0]
        assert 2 * small[0] <= max(hs) and 2 * small[1] <= max(ws)            # far inside the canvas
        sp = _pads(SMALL, int(BASE * s))
        assert max(sp) == (max(p[0] for p in sp), max(p[1] for p in sp))     # one SMALL frame is the whole canvas
    assert _pads(RAW[:2], BASE // 2) == [(48, 48), (48, 56)] and _pads(RAW[:2], BASE) == [(96, 104)] * 2


@pytest.mark.parametrize("flip", [False, True])
@pytest.mark.parametrize("mode", ["bf16", "bf16x3", "fp32"])
def test_ragged_multiscale_equals_each_frame_alone(net, mode, flip):
    pe = _engine(net, mode)
    frames = _frames(RAW, 31)
    want = [_alone(pe, f, flip) for f in frames]
    assert sum(len(w[0]) for w in want) > 0
    _assert_frames_equal(_ragged(pe, frames, flip), want, RAW, "%s flip=%s" % (mode, flip))


def test_small_group_after_large_group_leaves_no_stale_data(net):
    for mode in ("bf16", "bf16x3"):
        small = _frames(SMALL, 43)
        first = _ragged(_engine(net, mode), small, True)
        pe = _engine(net, mode)
        _ragged(pe, _frames(LARGE, 44), True)
        again = _ragged(pe, small, True)
        want = [(first[0][i], first[1][i], first[2][i, :, :ph // 8, :pw // 8], first[3][i, :, :ph // 8, :pw // 8])
                for i, (ph, pw) in enumerate(_pads(SMALL, BASE))]
        _assert_frames_equal(again, want, SMALL, mode)
        for a, b in zip(again[2:], first[2:]):       # the whole canvas, +0 outside each frame included
            assert np.array_equal(_bits(a), _bits(b)), mode


def test_two_ragged_multiscale_runs_in_flight_return_their_own_results(net):
    pe = _engine(net)
    mix_a, mix_b = _frames(RAW[:5], 47), _frames([(123, 90), (100, 110), (61, 88)], 48)
    packed = [np.concatenate([f.ravel() for f in mix]) for mix in (mix_a, mix_b)]
    want = []
    for mix, p in zip((mix_a, mix_b), packed):
        pe.infer_raw_multiscale_ragged_async_u8(p.ctypes.data, False, [f.shape[:2] for f in mix], SCALES, BASE, 8, 0.1, True)
        want.append(([r.copy() for r in pe.fetch_arrays()], pe.fetch()))
    tickets = [pe.infer_raw_multiscale_ragged_async_u8(p.ctypes.data, False, [f.shape[:2] for f in mix], SCALES, BASE, 8,
                                                       0.1, True)
               for mix, p in zip((mix_a, mix_b), packed)]
    for t, mix, (w_rows, w_dicts) in zip(tickets, (mix_a, mix_b), want):
        rows = [r.copy() for r in pe.fetch_arrays(ticket=t)]
        dicts = pe.fetch(ticket=t)
        assert len(rows) == len(mix) and sum(len(r) for r in rows) > 0
        for g, w in zip(rows, w_rows):
            np.testing.assert_array_equal(g, w)
        assert dicts == w_dicts        # each frame normalised by its own padded base size


def test_ragged_multiscale_launches_no_more_than_one_uniform_call(net):
    nat = _nat()
    pe = _engine(net)
    for shapes in (RAW, SMALL):
        frames = _frames(shapes, 53)
        packed = np.concatenate([f.ravel() for f in frames])
        same = np.ascontiguousarray(np.stack([frames[0]] * len(frames)))
        for flip in (False, True):
            l0 = nat.launch_count()
            pe.infer_raw_multiscale_ragged_async_u8(packed.ctypes.data, False, shapes, SCALES, BASE, 8, 0.1, flip)
            pe.fetch_arrays()
            ragged = nat.launch_count() - l0
            l0 = nat.launch_count()
            pe.infer_raw_multiscale_async_u8(same.ctypes.data, False, len(frames), shapes[0][0], shapes[0][1], SCALES, BASE,
                                             8, 0.1, flip)
            pe.fetch_arrays()
            uniform = nat.launch_count() - l0
            assert ragged <= uniform, (shapes, flip, ragged, uniform)


def test_ragged_multiscale_rejects_bad_arguments(net):
    nat = _nat()
    pe = _engine(net, batch_cap=2)
    frames = _frames([(64, 80), (80, 64)], 59)
    packed = np.concatenate([f.ravel() for f in frames])
    hw = (ctypes.c_int * 6)(64, 80, 80, 64, 64, 64)
    sc = (ctypes.c_double * 17)(*([1.0] * 17))

    def call(images=packed.ctypes.data, n=2, src_hw=hw, scales=sc, n_scales=4):
        return nat.lib().b200pose_infer_raw_u8_multiscale_ragged(pe.net._h, pe.post._h, images, 0, n, src_hw, BASE, 8,
                                                                 scales, n_scales, pe.mode, ctypes.c_float(0.1), 1, None)
    for kwargs in ({"n_scales": 0}, {"n_scales": 17}, {"n": 3}, {"n": 0}, {"images": None}, {"src_hw": None},
                   {"scales": None}):
        with pytest.raises(nat.B200PoseError):
            nat.check(call(**kwargs), "multiscale_ragged %s" % kwargs)
    nat.check(call(), "multiscale_ragged")      # the same call with valid arguments runs
    pe.post.sync()
    pe.post.check_status(2)


def test_infer_images_multiscale_flip_on_mixed_sizes_matches_composed_oracle(net):
    """BASELINE.json configs[4] on two frames of different sizes that form one ragged group: infer_images(scales=...,
    flip=True) == per frame the composition of tests/test_gpu_tta.py's multi-scale oracle test."""
    eng = pkg_module("engine")
    pe = _engine(net, batch_cap=2)
    rs = np.random.RandomState(41)
    imgs = [rs.randint(0, 256, s + (3,)).astype(np.uint8) for s in ((90, 123), (90, 130))]
    assert len(eng.plan_ragged_batches(_pads([im.shape[:2] for im in imgs], BASE), 2)) == 1
    got = pe.infer_images(imgs, dest_size=BASE, factor=8, flip=True, scales=SCALES)
    port = pafprocess_oracle.load_port()

    def maps(frame, dest):
        crop, _, _ = glue_port.crop_with_factor(frame, dest, 8)
        H, W = crop.shape[:2]
        outs = [torch.empty((1, 38 if k % 2 == 0 else 19, H // 8, W // 8), device="cuda") for k in range(12)]
        xd = torch.from_numpy(np.ascontiguousarray(crop[None])).cuda()
        pe.net.forward_u8_ptr(xd.data_ptr(), True, 1, H, W, pe.mode, [o.data_ptr() for o in outs], True,
                              torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        return (outs[11][0].permute(1, 2, 0).contiguous().cpu().numpy(), outs[10][0].permute(1, 2, 0).contiguous().cpu().numpy())
    total = 0
    for i, im in enumerate(imgs):
        base_crop, _, _ = glue_port.crop_with_factor(im, BASE, 8)
        per_scale = []
        for s in SCALES:
            heat, paf = maps(im, int(BASE * s))
            heat_f, paf_f = maps(np.ascontiguousarray(im[:, ::-1]), int(BASE * s))
            per_scale.append((heat, paf, heat_f, paf_f))
        ah, ap = glue_port.multi_scale_maps(per_scale, (base_crop.shape[0] // 8, base_crop.shape[1] // 8))
        _, want = glue_port.paf_to_pose(ah, ap, port)
        assert_humans_equal(got[i], want, score_tol=0.0)
        total += len(want)
    assert total > 0
