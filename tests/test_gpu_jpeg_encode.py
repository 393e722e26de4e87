"""GPU: JPEG encoding on the device (b200pose_net_encode_jpegs, DESIGN.md 2.14) equals the host core and
cv2.imencode byte for byte - host and device frames and outputs, uniform and ragged batches from 1 frame to the call's
limit of 1024, every sampling and several qualities - leaves the bytes around its output alone, decodes back to
cv2.imdecode's frame on the device, encodes frames drawn on the device as cv2 encodes draw_humans' frames, adds five
launches per call, and refuses bad arguments before anything is enqueued."""
import ctypes

import numpy as np
import pytest

import jpeg_enc_check as je
from conftest import pkg_module

cv2 = pytest.importorskip("cv2")
torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def net(built):
    return pkg_module("engine").NativeNet(0)


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    return je.compile_core(str(tmp_path_factory.mktemp("jpeg_enc_gpu") / "libjpegenccore.so"))


def _frames(sizes, seed=0, kinds=("photo", "checker", "noise", "flat", "saturated")):
    return [je.frame(h, w, seed + k, kinds[k % len(kinds)]) for k, (h, w) in enumerate(sizes)]


@pytest.mark.parametrize("sampling", sorted(je.SAMPLING))
@pytest.mark.parametrize("quality", [1, 50, 95, 100])
def test_ragged_host_frames_host_output(net, core, sampling, quality):
    frames = _frames([(1, 1), (17, 23), (33, 47), (480, 640), (37, 16), (64, 80)], quality)
    got = net.encode_jpegs(frames, quality, sampling)
    for k, f in enumerate(frames):
        want = je.cv2_encode(f, quality, sampling)
        assert got[k] == want, (k, f.shape)
        assert je.core_encode(core, f, quality, sampling) == want


@pytest.mark.parametrize("sampling", sorted(je.SAMPLING))
def test_device_frames_and_device_output(net, sampling):
    frames = _frames([(368, 368)] * 4, 3)
    dev = torch.from_numpy(np.stack(frames)).cuda()
    got = net.encode_jpegs(dev, 90, sampling, device=True)
    torch.cuda.synchronize()
    assert all(g.is_cuda for g in got)
    assert [g.cpu().numpy().tobytes() for g in got] == [je.cv2_encode(f, 90, sampling) for f in frames]
    ragged = _frames([(100, 31), (7, 250), (1080, 1920)], 5)
    got = net.encode_jpegs([torch.from_numpy(f).cuda() for f in ragged], 75, sampling)
    assert got == [je.cv2_encode(f, 75, sampling) for f in ragged]


@pytest.mark.parametrize("n", [1, 2, 33, 1024])
def test_batch_sizes_up_to_the_limit(net, n):
    rs = np.random.RandomState(n)
    sizes = [(int(rs.randint(1, 70)), int(rs.randint(1, 70))) for _ in range(n)]
    frames = _frames(sizes, n)
    got = net.encode_jpegs(frames, 85, "420")
    assert got == [je.cv2_encode(f, 85, "420") for f in frames]


def test_sentinels_around_the_output(net):
    frames = _frames([(45, 61), (120, 90)], 9)
    L = pkg_module("_native").lib()
    fl = np.concatenate([f.reshape(-1) for f in frames])
    hw = (ctypes.c_int * 4)(45, 61, 120, 90)
    cap = sum(L.b200pose_jpeg_encode_bound(h, w, 0x221111) for h, w in ((45, 61), (120, 90)))
    pad = 4096
    for dev in (False, True):
        if dev:
            buf = torch.full((cap + 2 * pad,), 0xA5, dtype=torch.uint8, device="cuda")
            ptr, stream = buf.data_ptr() + pad, torch.cuda.current_stream().cuda_stream
        else:
            buf = np.full(cap + 2 * pad, 0xA5, np.uint8)
            ptr, stream = buf.ctypes.data + pad, 0
        lens = (ctypes.c_longlong * 2)()
        assert L.b200pose_net_encode_jpegs(net._h, ctypes.c_void_p(fl.ctypes.data), 0, hw, 2, 95, 0x221111,
                                           ctypes.c_void_p(ptr), cap, int(dev), lens, ctypes.c_void_p(stream)) == 0
        b = buf.cpu().numpy() if dev else buf
        total = lens[0] + lens[1]
        assert (b[:pad] == 0xA5).all() and (b[pad + cap:] == 0xA5).all()
        assert b[pad:pad + total].tobytes() == b"".join(je.cv2_encode(f, 95, "420") for f in frames)


def test_device_decoder_reads_the_streams_back(net):
    frames = _frames([(240, 320), (33, 47), (1, 1)], 11, ("photo",))
    for s in sorted(je.SAMPLING):
        blobs = net.encode_jpegs(frames, 90, s)
        dec = net.decode_jpegs(blobs)
        for b, d in zip(blobs, dec):
            assert np.array_equal(d, cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR)), s


def test_encoding_device_drawn_frames(net):
    """Frames drawn on the device (b200pose_post_draw, what PoseEngine.draw_humans runs) and encoded from the same
    buffer give cv2.imencode(draw_humans(frame, humans)) byte for byte."""
    synth = pytest.importorskip("oracle.synth")
    common, p2p = pkg_module("lib.utils.common"), pkg_module("lib.utils.paf_to_pose")
    post = pkg_module("engine").NativePost(0, batch_cap=4, peak_cap=512, human_cap=256)
    maps = [synth.stick_figures(p, 30 + p)[:2] for p in (3, 5)]
    heat = np.ascontiguousarray(np.stack([m[0] for m in maps]))
    paf = np.ascontiguousarray(np.stack([m[1] for m in maps]))
    post.run(heat.ctypes.data, paf.ctypes.data, False, 1, 2, 46, 46, 0.1)
    post.sync()
    sizes = [(368, 368), (300, 420)]
    frames = _frames(sizes, 13, ("photo",))
    dev = torch.from_numpy(np.concatenate([f.reshape(-1) for f in frames])).cuda()
    post.draw(dev.data_ptr(), True, 2, sizes, [(368, 368)] * 2, torch.cuda.current_stream().cuda_stream)
    at, views = 0, []
    for h, w in sizes:
        views.append(dev[at:at + h * w * 3].view(h, w, 3))
        at += h * w * 3
    got = net.encode_jpegs(views, 95, "420")
    for i, f in enumerate(frames):
        drawn = common.draw_humans(f.copy(), p2p.humans_from_rows(post.humans(i), 368, 368))
        assert got[i] == je.cv2_encode(drawn, 95, "420"), i


def test_refusals_leave_the_net_usable(net):
    nat = pkg_module("_native")
    L = nat.lib()
    f = je.frame(16, 16, 1)
    hw = (ctypes.c_int * 2)(16, 16)
    cap = L.b200pose_jpeg_encode_bound(16, 16, 0x221111)
    out = np.empty(cap, np.uint8)
    lens = (ctypes.c_longlong * 1)()
    before = nat.launch_count()
    cases = [((0, 95, 0x221111, cap, hw), "n = 0"), ((1025, 95, 0x221111, cap, hw), "n = 1025"),
             ((1, 0, 0x221111, cap, hw), "quality 0"), ((1, 101, 0x221111, cap, hw), "quality 101"),
             ((1, 95, 0x222222, cap, hw), "sampling"), ((1, 95, 0x221111, cap - 1, hw), "out_cap"),
             ((1, 95, 0x221111, cap, (ctypes.c_int * 2)(0, 16)), "size"),
             ((1, 95, 0x221111, cap, (ctypes.c_int * 2)(16, 65536)), "size")]
    for (n, q, s, c, h), what in cases:
        rc = L.b200pose_net_encode_jpegs(net._h, ctypes.c_void_p(f.ctypes.data), 0, h, n, q, s,
                                         ctypes.c_void_p(out.ctypes.data), c, 0, lens, None)
        assert rc != 0 and what in L.b200pose_last_error().decode(), what
    assert nat.launch_count() == before
    assert net.encode_jpegs([f], 95, "420") == [je.cv2_encode(f, 95, "420")]
    assert nat.launch_count() == before + 5
    assert L.b200pose_jpeg_encode_bound(0, 5, 0x221111) == -1 and L.b200pose_jpeg_encode_bound(5, 5, 7) == -1
