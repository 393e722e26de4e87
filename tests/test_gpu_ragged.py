"""GPU (-m gpu): ragged batches (DESIGN.md 1) - frames of different sizes as one device batch on the canvas of the
largest.  Every frame must come out exactly as it does when it runs alone, and the canvas outside it must be +0."""
import numpy as np
import pytest
import torch

from conftest import pkg_module

pytestmark = pytest.mark.gpu

# padded sizes: portrait and landscape; at stride 8 h = 25, 17, 7, 31 are not multiples of the 16-row conv tile and
# w = 17, 25, 9, 5, 33 not multiples of the 8-column one; (248, 264) is the canvas itself; (8, 8) a one-pixel map
SHAPES = [(8, 8), (200, 136), (136, 200), (96, 72), (248, 264), (56, 40)]
ACT_C = [64, 64, 128, 128, 256, 256, 256, 512, 512, 256, 192, 256, 256, 1024]
ACT_DIV = [1, 2, 2, 4, 4, 4, 8, 8, 8, 8, 8, 8, 8, 8]


@pytest.fixture(scope="module")
def net(built, he_sd):
    eng = pkg_module("engine")
    n = eng.NativeNet(0)
    n.load_state_dict_arrays([v.numpy() for v in he_sd.values()])
    return n


def _frames(shapes, seed):
    rs = np.random.RandomState(seed)
    return [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in shapes]


def _maps(n, H, W):
    return [torch.empty((n, 38 if k % 2 == 0 else 19, H // 8, W // 8), device="cuda") for k in range(12)]


def _alone(net, frame, mode):
    H, W = frame.shape[:2]
    outs = _maps(1, H, W)
    xd = torch.from_numpy(np.ascontiguousarray(frame[None])).cuda()
    net.forward_u8_ptr(xd.data_ptr(), True, 1, H, W, mode, [o.data_ptr() for o in outs], True,
                       torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return outs


def _ragged(net, frames, mode, stream=None):
    shapes = [f.shape[:2] for f in frames]
    Hc, Wc = max(s[0] for s in shapes), max(s[1] for s in shapes)
    outs = _maps(len(frames), Hc, Wc)
    packed = torch.from_numpy(np.concatenate([f.ravel() for f in frames])).cuda()
    torch.cuda.synchronize()
    s = stream if stream is not None else torch.cuda.current_stream()
    net.forward_ragged_u8_ptr(packed.data_ptr(), True, shapes, mode, [o.data_ptr() for o in outs], True, s.cuda_stream)
    torch.cuda.synchronize()
    return outs


def _positive_zero(t):
    return bool((t.contiguous().view(torch.int32) == 0).all())


def _check_maps(net, frames, got, mode, alone_cache=None):
    for i, f in enumerate(frames):
        h, w = f.shape[0] // 8, f.shape[1] // 8
        want = alone_cache[i] if alone_cache is not None else _alone(net, f, mode)
        for k in range(12):
            assert torch.equal(got[k][i, :, :h, :w], want[k][0]), (i, k)
            plane = got[k][i]
            assert _positive_zero(plane[:, h:, :]) and _positive_zero(plane[:, :h, w:]), (i, k)


@pytest.mark.parametrize("mode", ["bf16", "bf16x3", "fp32"])
@pytest.mark.parametrize("pre", ["rtpose", "vgg"])
def test_ragged_maps_equal_each_frame_alone(net, mode, pre):
    nat = pkg_module("_native")
    net.set_preprocess(pre)
    try:
        frames = _frames(SHAPES, 11)
        got = _ragged(net, frames, nat.MODES[mode])
        _check_maps(net, frames, got, nat.MODES[mode])
    finally:
        net.set_preprocess("rtpose")


def _read(net, buf, lo, n, H, W):
    per = (H // ACT_DIV[buf]) * (W // ACT_DIV[buf]) * ACT_C[buf]
    out = np.empty(n * per, np.uint16)
    nat = pkg_module("_native")
    nat.check(nat.lib().b200pose_net_debug_read(net._h, buf, lo, 0, n, out.ctypes.data, out.nbytes), "debug_read")
    return out.reshape(n, H // ACT_DIV[buf], W // ACT_DIV[buf], ACT_C[buf])


def test_ragged_batch_after_larger_frames_leaves_no_stale_data(net):
    """A batch of canvas-size frames, then a mix on the same canvas: the maps still equal each frame alone and every
    activation buffer and residual plane is exactly 0 outside each frame's extent at its resolution."""
    nat = pkg_module("_native")
    Hc, Wc = 248, 264
    for mode in ("bf16x3", "bf16"):
        m = nat.MODES[mode]
        big = _frames([(Hc, Wc)] * len(SHAPES), 5)
        _ragged(net, big, m)
        frames = _frames(SHAPES, 12)
        got = _ragged(net, frames, m)
        for buf in range(len(ACT_C)):
            for lo in ((0, 1) if mode == "bf16x3" else (0,)):
                a = _read(net, buf, lo, len(frames), Hc, Wc)
                for i, (h, w) in enumerate(SHAPES):
                    hh, ww = h // ACT_DIV[buf], w // ACT_DIV[buf]
                    assert not a[i, hh:].any() and not a[i, :hh, ww:].any(), (mode, buf, lo, i)
        _check_maps(net, frames, got, m)


def _engine(he_sd, batch_cap=8):
    eng = pkg_module("engine")
    return eng.PoseEngine([v.numpy() for v in he_sd.values()], 0, mode="bf16", batch_cap=batch_cap, peak_cap=1024,
                          human_cap=2048)


RAW = [(150, 211), (120, 100), (97, 64), (184, 184), (130, 260), (300, 190)]


def _alone_persons(pe, frame, flip, thresh):
    h, w = frame.shape[:2]
    buf = np.ascontiguousarray(frame[None])
    pe.infer_raw_async_u8(buf.ctypes.data, False, 1, h, w, 184, 8, thresh, flip)
    rows = pe.fetch_arrays()[0].copy()
    return rows, pe.post.peaks(0)


def test_ragged_inference_gives_each_frames_persons_and_peaks(built, he_sd):
    pe = _engine(he_sd)
    rs = np.random.RandomState(23)
    frames = [rs.randint(0, 256, s + (3,)).astype(np.uint8) for s in RAW]
    # a frame without persons: a grey frame, with the peak threshold at the top of its own heat maps (its mirror is
    # itself, so the flip-averaged maps stay below it as well)
    grey = np.full((140, 170, 3), 128, np.uint8)
    crop, _, _ = pe.net.crop_with_factor(grey, 184, 8)
    thresh = float(_alone(pe.net, crop, pe.mode)[11][0, :18].max())
    frames.insert(2, grey)
    for flip in (False, True):
        want = [_alone_persons(pe, f, flip, thresh) for f in frames]
        assert sum(len(r) for r, _ in want) > 0 and len(want[2][0]) == 0 and len(want[2][1]) == 0
        packed = np.concatenate([f.ravel() for f in frames])
        pe.infer_raw_ragged_async_u8(packed.ctypes.data, False, [f.shape[:2] for f in frames], 184, 8, thresh, flip)
        got = pe.fetch_arrays()
        for i in range(len(frames)):
            np.testing.assert_array_equal(got[i], want[i][0], err_msg="flip=%s frame %d" % (flip, i))
            np.testing.assert_array_equal(pe.post.peaks(i), want[i][1], err_msg="flip=%s frame %d" % (flip, i))


def test_two_ragged_runs_in_flight_return_their_own_results(built, he_sd):
    pe = _engine(he_sd)
    rs = np.random.RandomState(29)
    mix_a = [rs.randint(0, 256, s + (3,)).astype(np.uint8) for s in RAW[:4]]
    mix_b = [rs.randint(0, 256, s + (3,)).astype(np.uint8) for s in ((160, 230), (110, 200), (200, 120))]
    want = []
    for mix in (mix_a, mix_b):
        p = np.concatenate([f.ravel() for f in mix])
        pe.infer_raw_ragged_async_u8(p.ctypes.data, False, [f.shape[:2] for f in mix], 184, 8, 0.1, False)
        want.append([r.copy() for r in pe.fetch_arrays()])
    pa = np.concatenate([f.ravel() for f in mix_a])
    pb = np.concatenate([f.ravel() for f in mix_b])
    ta = pe.infer_raw_ragged_async_u8(pa.ctypes.data, False, [f.shape[:2] for f in mix_a], 184, 8, 0.1, False)
    tb = pe.infer_raw_ragged_async_u8(pb.ctypes.data, False, [f.shape[:2] for f in mix_b], 184, 8, 0.1, False)
    got_a = [r.copy() for r in pe.fetch_arrays(ticket=ta)]
    got_b = [r.copy() for r in pe.fetch_arrays(ticket=tb)]
    assert len(got_a) == 4 and len(got_b) == 3
    for g, w in zip(got_a + got_b, want[0] + want[1]):
        np.testing.assert_array_equal(g, w)


def test_graph_replay_of_a_small_ragged_batch_equals_plain_launches(built, he_sd, monkeypatch):
    eng = pkg_module("engine")
    nat = pkg_module("_native")
    arrays = [v.numpy() for v in he_sd.values()]
    monkeypatch.setenv("B200POSE_GRAPH", "0")
    plain = eng.NativeNet(0)
    plain.load_state_dict_arrays(arrays)
    monkeypatch.setenv("B200POSE_GRAPH", "1")
    graphed = eng.NativeNet(0)
    graphed.load_state_dict_arrays(arrays)
    stream = torch.cuda.Stream()             # a real stream: small plans are captured at their second use
    mix_a = _frames([(64, 64), (32, 48)], 3)
    mix_b = _frames([(48, 64), (64, 40)], 4)     # same 64 x 64 canvas, another mix
    for mode in ("bf16", "bf16x3"):
        m = nat.MODES[mode]
        for mix in (mix_a, mix_a, mix_a, mix_b, mix_b, mix_a):
            want = _ragged(plain, mix, m, stream)
            got = _ragged(graphed, mix, m, stream)
            for a, b in zip(got, want):
                assert torch.equal(a, b), mode
            _check_maps(graphed, mix, got, m)


def test_mixed_shapes_in_one_ragged_batch_issue_one_forward(built, he_sd):
    """32 landscape frames in 8 padded shapes that the grouping rule puts into one batch: infer_images issues the
    launches of one pass (crop, 52 network launches, post-processing), the same count as one uniform batch of 32."""
    nat = pkg_module("_native")
    eng = pkg_module("engine")
    pe = _engine(he_sd, batch_cap=32)
    rs = np.random.RandomState(37)
    frames = [rs.randint(0, 256, (184, 240 + 8 * (i % 8), 3)).astype(np.uint8) for i in range(32)]
    pads = [nat.crop_geometry(184, f.shape[1], 184, 8)[2] for f in frames]
    assert len(set(pads)) == 8 and len(eng.plan_ragged_batches(pads, 32)) == 1
    pe.infer_images(frames, dest_size=184)
    l0 = nat.launch_count()
    pe.infer_images(frames, dest_size=184)
    ragged = nat.launch_count() - l0
    same = np.ascontiguousarray(np.stack([f[:, :240] for f in frames]))
    pe.infer_raw_async_u8(same.ctypes.data, False, 32, 184, 240, 184, 8, 0.1, False)
    pe.fetch()
    l0 = nat.launch_count()
    pe.infer_raw_async_u8(same.ctypes.data, False, 32, 184, 240, 184, 8, 0.1, False)
    pe.fetch()
    uniform = nat.launch_count() - l0
    assert ragged == uniform and ragged < 2 * 52, (ragged, uniform)
