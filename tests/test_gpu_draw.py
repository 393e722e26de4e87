"""GPU (-m gpu): drawing of detected persons on the device (DESIGN.md 2.12).  b200pose_post_draw must equal the host
build of csrc/draw_core.h (tests/test_draw_host.py ties that to cv2 and draw_humans) bit for bit on host and device
frames, ragged, without touching a byte around the frames; and PoseStream(draw='device' / 'cuda') must yield exactly
what PoseStream(draw=True) yields."""
import numpy as np
import pytest
import torch

from conftest import pkg_module
import draw_check as dc

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu

SIZES = [(1080, 1920), (200, 150), (480, 640)]
NET = (368, 368)
SENTINEL = 4096


@pytest.fixture(scope="module")
def core(built, tmp_path_factory):
    return dc.compile_core(str(tmp_path_factory.mktemp("draw") / "libdrawcore.so"))


def _post(batch_cap=4):
    return pkg_module("engine").NativePost(0, batch_cap=batch_cap, peak_cap=1024, human_cap=512)


def _run(post, persons, seed):
    """post-processing of synthetic stick-figure maps (46 x 46, a 368 x 368 network input) for len(persons) images."""
    synth = pytest.importorskip("oracle.synth")
    maps = [synth.stick_figures(p, seed + i)[:2] if p else (np.zeros((46, 46, 19), np.float32),
                                                           np.zeros((46, 46, 38), np.float32))
            for i, p in enumerate(persons)]
    heat = np.ascontiguousarray(np.stack([m[0] for m in maps]))
    paf = np.ascontiguousarray(np.stack([m[1] for m in maps]))
    post.run(heat.ctypes.data, paf.ctypes.data, False, 1, len(persons), 46, 46, 0.1)
    post.__dict__.setdefault("_keep", []).append((heat, paf))


def _frames(seed):
    rs = np.random.RandomState(seed)
    return [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in SIZES]


def _packed(frames, seed):
    """frames back to back with seeded 4 KB sentinels before and after them"""
    rs = np.random.RandomState(seed)
    body = np.concatenate([f.reshape(-1) for f in frames])
    return np.concatenate([rs.randint(0, 256, SENTINEL).astype(np.uint8), body,
                           rs.randint(0, 256, SENTINEL).astype(np.uint8)])


def _unpack(buf, shapes):
    out, at = [], SENTINEL
    for h, w in shapes:
        out.append(buf[at:at + h * w * 3].reshape(h, w, 3))
        at += h * w * 3
    return out


def _want(core, post, frames):
    return [dc.core_draw(core, f.copy(), post.humans(i), *NET) for i, f in enumerate(frames)]


@pytest.mark.parametrize("on_device", [False, True])
def test_ragged_draw_equals_the_host_core(core, on_device):
    post = _post()
    _run(post, [8, 3, 5], 21)
    post.sync()
    assert all(len(post.humans(i)) for i in range(3))
    frames = _frames(4)
    want = _want(core, post, frames)
    common, p2p = pkg_module("lib.utils.common"), pkg_module("lib.utils.paf_to_pose")
    np.testing.assert_array_equal(want[0], common.draw_humans(frames[0].copy(), p2p.humans_from_rows(post.humans(0), 368, 368)))
    buf = _packed(frames, 9)
    ref = buf.copy()
    hw = [s for s in SIZES]
    if on_device:
        d = torch.from_numpy(buf).cuda()
        post.draw(d.data_ptr() + SENTINEL, True, 3, hw, [NET] * 3, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        buf = d.cpu().numpy()
    else:
        post.draw(buf.ctypes.data + SENTINEL, False, 3, hw, [NET] * 3)
    np.testing.assert_array_equal(buf[:SENTINEL], ref[:SENTINEL])
    np.testing.assert_array_equal(buf[-SENTINEL:], ref[-SENTINEL:])
    for i, (g, w) in enumerate(zip(_unpack(buf, SIZES), want)):
        np.testing.assert_array_equal(g, w, err_msg="frame %d" % i)
        assert (g != frames[i]).any()


def test_a_run_without_persons_leaves_the_frames_unchanged():
    post = _post()
    _run(post, [0, 0], 3)
    post.sync()
    frames = _frames(5)[:2]
    buf = _packed(frames, 1)
    ref = buf.copy()
    post.draw(buf.ctypes.data + SENTINEL, False, 2, SIZES[:2], [NET] * 2)
    np.testing.assert_array_equal(buf, ref)


def test_a_later_run_does_not_change_what_a_draw_call_drew(core):
    post = _post()
    _run(post, [6, 6, 6], 40)
    post.sync()
    frames = _frames(6)
    want = _want(core, post, frames)
    d = torch.from_numpy(_packed(frames, 2)).cuda()
    post.draw(d.data_ptr() + SENTINEL, True, 3, SIZES, [NET] * 3, torch.cuda.current_stream().cuda_stream)
    _run(post, [9, 2, 4], 77)        # run i+1 writes the other pinned slot, then the one after it this slot
    _run(post, [1, 7, 3], 78)
    torch.cuda.synchronize()
    post.sync()
    for g, w in zip(_unpack(d.cpu().numpy(), SIZES), want):
        np.testing.assert_array_equal(g, w)


def test_refusals_name_their_field_and_a_clean_call_follows(core):
    nat = pkg_module("_native")
    post = _post(batch_cap=2)
    frames = _frames(8)[1:3]
    buf = _packed(frames, 3)
    ptr = buf.ctypes.data + SENTINEL
    with pytest.raises(nat.B200PoseError, match="no run selected"):
        post.draw(ptr, False, 2, SIZES[1:], [NET] * 2)
    _run(post, [4, 4], 50)
    post.sync()
    with pytest.raises(nat.B200PoseError, match="batch_cap"):
        post.draw(ptr, False, 3, SIZES, [NET] * 3)
    with pytest.raises(nat.B200PoseError, match="frame_hw of image 1"):
        post.draw(ptr, False, 2, [SIZES[1], (0, 5)], [NET] * 2)
    with pytest.raises(nat.B200PoseError, match="net_hw of image 0"):
        post.draw(ptr, False, 2, SIZES[1:], [(368, 0), NET])
    ref = buf.copy()
    post.draw(ptr, False, 2, SIZES[1:], [NET] * 2)
    np.testing.assert_array_equal(buf[:SENTINEL], ref[:SENTINEL])
    for i, (g, f) in enumerate(zip(_unpack(buf, SIZES[1:]), frames)):
        np.testing.assert_array_equal(g, dc.core_draw(core, f.copy(), post.humans(i), *NET))


def _yuv_nv12(bgr):
    h, w = bgr.shape[:2]
    i420 = cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420)
    flat, q = i420.reshape(-1), (h // 2) * (w // 2)
    u, v = flat[h * w:h * w + q].reshape(h // 2, w // 2), flat[h * w + q:].reshape(h // 2, w // 2)
    return np.concatenate([i420[:h], np.stack([u, v], -1).reshape(h // 2, w)])


def _streams_agree(make, frames, **kw):
    streaming = pkg_module("streaming")
    want = list(streaming.PoseStream(make(), frames, batch=3, **kw))
    assert sum(len(h) for _, h, _ in want) > 0
    for mode in ("device", "cuda"):
        got = list(streaming.PoseStream(make(), frames, batch=3, draw=mode, **kw))
        assert len(got) == len(want)
        for (gf, gh, gd), (wf, wh, wd) in zip(got, want):
            assert len(gh) == len(wh)
            if mode == "cuda":
                assert isinstance(gd, torch.Tensor) and gd.is_cuda
                gd = gd.cpu().numpy()
                gf = gf.cpu().numpy() if isinstance(gf, torch.Tensor) else gf
            np.testing.assert_array_equal(gf, wf)
            np.testing.assert_array_equal(gd, wd)


@pytest.fixture(scope="module")
def model(built, he_sd):
    from lib.network.rtpose_vgg import get_model
    m = get_model("vgg19")
    m.load_state_dict(he_sd)
    return m.cuda().float().eval()


def test_pose_stream_device_drawing_on_bgr_frames(model):
    frames = [np.random.RandomState(s).randint(0, 256, (240, 320, 3)).astype(np.uint8) for s in range(7)]
    _streams_agree(lambda: model, frames)


def test_pose_stream_device_drawing_on_rotated_nv12_frames(model):
    nat = pkg_module("_native")
    frames = [_yuv_nv12(np.random.RandomState(11 + s).randint(0, 256, (240, 320, 3)).astype(np.uint8)) for s in range(7)]
    _streams_agree(lambda: model, frames, format="nv12", rotate=nat.rotation_of(cv2.ROTATE_90_CLOCKWISE))


def test_pose_stream_device_drawing_on_an_openpose_engine(built):
    import openpose_port
    pe = pkg_module("engine").openpose_engine(openpose_port.he_state_dict(4, 2), 4, 2, batch_cap=8, peak_cap=1024,
                                              human_cap=2048)
    frames = [np.random.RandomState(30 + s).randint(0, 256, (240, 320, 3)).astype(np.uint8) for s in range(5)]
    _streams_agree(lambda: pe, frames)
