"""GPU: PNG encoding on the device (b200pose_net_encode_pngs, DESIGN.md 2.15) equals the host core and
cv2.imencode('.png') byte for byte - host and device frames and outputs, uniform and ragged batches from 1 frame to the
call's limit of 1024, 1080p and 3000 x 4000 - leaves the bytes around its output alone, encodes frames drawn on the
device as cv2 encodes draw_humans' frames, adds nine launches per call, and refuses bad arguments before anything is
enqueued."""
import ctypes

import numpy as np
import pytest

import png_enc_check as pe
from conftest import pkg_module

cv2 = pytest.importorskip("cv2")
torch = pytest.importorskip("torch")

pytestmark = pytest.mark.gpu

KINDS = ("photo", "noise", "flat", "stripes", "norun", "drawn")


@pytest.fixture(scope="module")
def net(built):
    return pkg_module("engine").NativeNet(0)


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    return pe.compile_core(str(tmp_path_factory.mktemp("png_enc_gpu") / "libpngenccore.so"))


def _frames(sizes, seed=0, kinds=KINDS):
    return [pe.frame(h, w, seed + k, kinds[k % len(kinds)]) for k, (h, w) in enumerate(sizes)]


def test_ragged_host_frames_host_output(net, core):
    sizes = [(1, 1), (1, 300), (300, 1), (17, 23), (129, 42), (258, 42), (64, 85), (480, 640), (37, 16), (100, 300),
             (5, 1000)]
    for seed in range(len(KINDS)):
        frames = _frames(sizes, seed)
        got = net.encode_pngs(frames)
        for k, f in enumerate(frames):
            want = pe.cv2_encode(f)
            assert got[k] == want, (seed, k, f.shape)
            assert pe.core_encode(core, f) == want


def test_device_frames_and_device_output(net):
    frames = _frames([(368, 368)] * 4, 3)
    dev = torch.from_numpy(np.stack(frames)).cuda()
    got = net.encode_pngs(dev, device=True)
    torch.cuda.synchronize()
    assert all(g.is_cuda for g in got)
    assert [g.cpu().numpy().tobytes() for g in got] == [pe.cv2_encode(f) for f in frames]
    ragged = _frames([(100, 31), (7, 250), (1080, 1920)], 5)
    got = net.encode_pngs([torch.from_numpy(f).cuda() for f in ragged])
    assert got == [pe.cv2_encode(f) for f in ragged]


def test_large_frames(net):
    frames = [pe.frame(1080, 1920, 1, k) for k in ("photo", "noise", "flat", "drawn")] + [pe.frame(3000, 4000, 2)]
    assert net.encode_pngs(frames) == [pe.cv2_encode(f) for f in frames]


@pytest.mark.parametrize("n", [1, 2, 33, 1024])
def test_batch_sizes_up_to_the_limit(net, n):
    rs = np.random.RandomState(n)
    sizes = [(int(rs.randint(1, 70)), int(rs.randint(1, 70))) for _ in range(n)]
    frames = _frames(sizes, n)
    assert net.encode_pngs(frames) == [pe.cv2_encode(f) for f in frames]


def test_sentinels_around_the_output(net):
    frames = _frames([(45, 61), (120, 90)], 9, ("photo", "noise"))
    L = pkg_module("_native").lib()
    fl = np.concatenate([f.reshape(-1) for f in frames])
    hw = (ctypes.c_int * 4)(45, 61, 120, 90)
    cap = sum(L.b200pose_png_encode_bound(h, w) for h, w in ((45, 61), (120, 90)))
    pad = 4096
    for dev in (False, True):
        if dev:
            buf = torch.full((cap + 2 * pad,), 0xA5, dtype=torch.uint8, device="cuda")
            ptr, stream = buf.data_ptr() + pad, torch.cuda.current_stream().cuda_stream
        else:
            buf = np.full(cap + 2 * pad, 0xA5, np.uint8)
            ptr, stream = buf.ctypes.data + pad, 0
        lens = (ctypes.c_longlong * 2)()
        assert L.b200pose_net_encode_pngs(net._h, ctypes.c_void_p(fl.ctypes.data), 0, hw, 2, ctypes.c_void_p(ptr), cap,
                                          int(dev), lens, ctypes.c_void_p(stream)) == 0
        b = buf.cpu().numpy() if dev else buf
        total = lens[0] + lens[1]
        assert (b[:pad] == 0xA5).all() and (b[pad + cap:] == 0xA5).all()
        assert b[pad:pad + total].tobytes() == b"".join(pe.cv2_encode(f) for f in frames)


def test_encoding_device_drawn_frames(net):
    """Frames drawn on the device (b200pose_post_draw, what PoseEngine.draw_humans runs) and encoded from the same
    buffer give cv2.imencode('.png', draw_humans(frame, humans)) byte for byte."""
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
    got = net.encode_pngs(views)
    for i, f in enumerate(frames):
        drawn = common.draw_humans(f.copy(), p2p.humans_from_rows(post.humans(i), 368, 368))
        assert got[i] == pe.cv2_encode(drawn), i


def test_refusals_leave_the_net_usable(net):
    nat = pkg_module("_native")
    L = nat.lib()
    f = pe.frame(16, 16, 1)
    hw = (ctypes.c_int * 2)(16, 16)
    cap = L.b200pose_png_encode_bound(16, 16)
    out = np.empty(cap, np.uint8)
    lens = (ctypes.c_longlong * 1)()
    before = nat.launch_count()
    cases = [((0, cap, hw), "n = 0"), ((1025, cap, hw), "n = 1025"), ((1, cap - 1, hw), "out_cap"),
             ((1, cap, (ctypes.c_int * 2)(0, 16)), "size"), ((1, cap, (ctypes.c_int * 2)(16, 65536)), "size")]
    for (n, c, h), what in cases:
        rc = L.b200pose_net_encode_pngs(net._h, ctypes.c_void_p(f.ctypes.data), 0, h, n, ctypes.c_void_p(out.ctypes.data),
                                        c, 0, lens, None)
        assert rc != 0 and what in L.b200pose_last_error().decode(), what
    assert nat.launch_count() == before
    assert net.encode_pngs([f]) == [pe.cv2_encode(f)]
    assert nat.launch_count() == before + 9
    assert L.b200pose_png_encode_bound(0, 5) == -1 and L.b200pose_png_encode_bound(5, 65536) == -1
