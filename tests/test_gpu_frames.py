"""GPU (-m gpu): video-frame ingestion (DESIGN.md 2.10) - NV12 / I420 / pitched BGR frames, host or device, converted and
rotated on the device.  The conversion must equal the host build of csrc/frame_core.h (tests/test_frames_host.py ties
that to cv2.cvtColor + cv2.rotate), and b200pose_infer_frames must give, bit for bit, what the b200pose_infer_raw_u8*
entry points give on the frames converted and rotated with cv2 on the host."""
import ctypes
import os
import subprocess

import numpy as np
import pytest
import torch

from conftest import ROOT, pkg_module

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu

CV_ROTATE = {0: None, 90: cv2.ROTATE_90_CLOCKWISE, 180: cv2.ROTATE_180, 270: cv2.ROTATE_90_COUNTERCLOCKWISE}
FORMATS = {"bgr": 0, "nv12": 1, "i420": 2}
DEST = 96
SCALES = (0.5, 1.0, 1.5, 2.0)
MIXED = [(120, 160), (96, 130), (160, 120), (100, 100), (88, 150), (120, 160), (132, 96), (110, 140)]


def _nat():
    return pkg_module("_native")


@pytest.fixture(scope="module")
def net(built, he_sd):
    n = pkg_module("engine").NativeNet(0)
    n.load_state_dict_arrays([v.numpy() for v in he_sd.values()])
    return n


@pytest.fixture(scope="module")
def host_core(built, tmp_path_factory):
    so = str(tmp_path_factory.mktemp("frames") / "libframecore.so")
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-o", so,
                    os.path.join(ROOT, "tests", "cuda", "frame_core_host.cpp")], check=True)
    lib = ctypes.CDLL(so)
    lib.core_convert_frame.argtypes = [ctypes.c_void_p] * 2 + [ctypes.c_int] * 5 + [ctypes.c_void_p]
    return lib


def _engine(net, mode="bf16", batch_cap=8):
    return pkg_module("engine").PoseEngine.from_net(net, mode=mode, batch_cap=batch_cap, peak_cap=1024, human_cap=2048)


def _bgr_frames(shapes, seed):
    """Seeded uint8 BGR frames, as tests/test_gpu_ragged.py makes them."""
    rs = np.random.RandomState(seed)
    return [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in shapes]


def _yuv(bgr, fmt):
    """A BGR frame as a packed cv2 4:2:0 array (3h/2, w): I420 from cv2, NV12 with U and V interleaved."""
    if fmt == "bgr":
        return bgr
    h, w = bgr.shape[:2]
    i420 = cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420)
    if fmt == "i420":
        return i420
    flat, q = i420.reshape(-1), (h // 2) * (w // 2)
    uv = np.stack([flat[h * w:h * w + q], flat[h * w + q:]], -1).reshape(h // 2, w)
    return np.concatenate([i420[:h], uv])


def _cv2_bgr(frame, fmt, rot):
    """What a host pipeline does today: cv2.cvtColor, then cv2.rotate."""
    code = {"nv12": cv2.COLOR_YUV2BGR_NV12, "i420": cv2.COLOR_YUV2BGR_I420}
    bgr = frame if fmt == "bgr" else cv2.cvtColor(frame, code[fmt])
    return bgr if CV_ROTATE[rot] is None else cv2.rotate(bgr, CV_ROTATE[rot])


def _planes(frame, fmt):
    h = frame.shape[0] * 2 // 3
    w = frame.shape[1]
    if fmt == "nv12":
        return [frame[:h], frame[h:]]
    flat, q = frame.reshape(-1), (h // 2) * (w // 2)
    return [frame[:h], flat[h * w:h * w + q].reshape(h // 2, w // 2), flat[h * w + q:].reshape(h // 2, w // 2)]


def _padded_cuda(plane, extra):
    """A CUDA view of `plane` whose rows are `extra` bytes longer than the plane (a pitched decoder surface)."""
    h = plane.shape[0]
    row = int(np.prod(plane.shape[1:]))
    buf = torch.randint(0, 256, (h, row + extra), dtype=torch.uint8, device="cuda")
    buf[:, :row] = torch.from_numpy(np.ascontiguousarray(plane).reshape(h, row)).cuda()
    return buf[:, :row].view(*plane.shape) if plane.ndim == 2 else buf[:, :row].view(h, plane.shape[1], 3)


def _host_core(lib, frame, fmt, rot):
    planes = [frame] if fmt == "bgr" else [np.ascontiguousarray(p) for p in _planes(frame, fmt)]
    h, w = (frame.shape[0], frame.shape[1]) if fmt == "bgr" else (frame.shape[0] * 2 // 3, frame.shape[1])
    ptrs = (ctypes.c_void_p * 3)(*([p.ctypes.data for p in planes] + [None] * (3 - len(planes))))
    pit = (ctypes.c_int * 3)(*([p.strides[0] for p in planes] + [0] * (3 - len(planes))))
    oh, ow = (w, h) if rot in (90, 270) else (h, w)
    out = np.empty((oh, ow, 3), np.uint8)
    lib.core_convert_frame(ptrs, pit, h, w, FORMATS[fmt], rot, 0, out.ctypes.data)
    return out


@pytest.mark.parametrize("fmt", ["bgr", "nv12", "i420"])
@pytest.mark.parametrize("rot", [0, 90, 180, 270])
def test_convert_frames_equals_the_host_core(net, host_core, fmt, rot):
    bgr = _bgr_frames(MIXED, 3 + rot + FORMATS[fmt])
    frames = [_yuv(f, fmt) for f in bgr]
    want = [_host_core(host_core, f, fmt, rot) for f in frames]
    for f, w in zip(frames, want):
        np.testing.assert_array_equal(w, _cv2_bgr(f, fmt, rot))
    for batch in (frames[:1], frames):
        n = len(batch)
        # host input: packed cv2 arrays, and planes given separately
        got = net.convert_frames(batch, fmt, rot)
        for g, w in zip(got, want[:n]):
            np.testing.assert_array_equal(g, w)
        if fmt != "bgr":
            got = net.convert_frames([tuple(_planes(f, fmt)) for f in batch], fmt, rot)
            for g, w in zip(got, want[:n]):
                np.testing.assert_array_equal(g, w)
        # device input: pitched torch views, read in place
        dev = [tuple(_padded_cuda(p, 13 + 3 * k) for k, p in enumerate(_planes(f, fmt))) if fmt != "bgr"
               else _padded_cuda(f, 13) for f in batch]
        torch.cuda.synchronize()
        got = net.convert_frames(dev, fmt, rot)
        for g, w in zip(got, want[:n]):
            np.testing.assert_array_equal(g, w)


def test_convert_frames_to_device_memory(net, host_core):
    nat, eng = _nat(), pkg_module("engine")
    frames = [_yuv(f, "nv12") for f in _bgr_frames(MIXED[:3], 9)]
    want = np.concatenate([_host_core(host_core, f, "nv12", 270).ravel() for f in frames])
    out = torch.empty(want.size, dtype=torch.uint8, device="cuda")
    table, keep, on_dev, _ = eng.frame_table(frames, "nv12")
    s = torch.cuda.current_stream()
    nat.check(nat.lib().b200pose_net_convert_frames(net._h, table, 3, 1, int(on_dev), 270, ctypes.c_void_p(out.data_ptr()),
                                                    1, ctypes.c_void_p(s.cuda_stream)), "convert_frames")
    torch.cuda.synchronize()
    np.testing.assert_array_equal(out.cpu().numpy(), want)


def _results(pe, n):
    rows = pe.fetch_arrays()
    return [(r.copy(), pe.post.peaks(i)) for i, r in enumerate(rows)]


def _reference(pe, bgr, flip, scales):
    """The verified BGR path: b200pose_infer_raw_u8 / _ragged / _multiscale / _multiscale_ragged on host BGR frames."""
    shapes = [f.shape[:2] for f in bgr]
    if len(set(shapes)) == 1:
        batch = np.ascontiguousarray(np.stack(bgr))
        (h, w), n = shapes[0], len(bgr)
        if scales is None:
            pe.infer_raw_async_u8(batch.ctypes.data, False, n, h, w, DEST, 8, 0.1, flip)
        else:
            pe.infer_raw_multiscale_async_u8(batch.ctypes.data, False, n, h, w, scales, DEST, 8, 0.1, flip)
    else:
        batch = np.concatenate([f.ravel() for f in bgr])
        if scales is None:
            pe.infer_raw_ragged_async_u8(batch.ctypes.data, False, shapes, DEST, 8, 0.1, flip)
        else:
            pe.infer_raw_multiscale_ragged_async_u8(batch.ctypes.data, False, shapes, scales, DEST, 8, 0.1, flip)
    return _results(pe, len(bgr))


def _assert_same(got, want):
    assert len(got) == len(want)
    for i, ((gr, gp), (wr, wp)) in enumerate(zip(got, want)):
        assert gr.shape == wr.shape and np.array_equal(gr, wr), ("rows", i)        # score_tol = 0
        assert gp.shape == wp.shape and np.array_equal(gp, wp), ("peaks", i)


CASES = [("single", False, None), ("flip", True, None), ("scales_flip", True, SCALES)]


@pytest.mark.parametrize("mode", ["bf16", "fp32"])
@pytest.mark.parametrize("case,flip,scales", CASES, ids=[c[0] for c in CASES])
@pytest.mark.parametrize("sizes", ["one", "mixed"])
def test_infer_frames_equals_the_bgr_path(net, mode, case, flip, scales, sizes):
    pe = _engine(net, mode)
    shapes = [(120, 160)] * 4 if sizes == "one" else MIXED[:5]
    bgr = _bgr_frames(shapes, 21)
    for fmt, rot, on_dev in (("nv12", 90, False), ("i420", 0, True), ("nv12", 270, True), ("i420", 180, False)):
        frames = [_yuv(f, fmt) for f in bgr]
        want = _reference(pe, [_cv2_bgr(f, fmt, rot) for f in frames], flip, scales)
        src = [torch.from_numpy(f).cuda() for f in frames] if on_dev else frames
        torch.cuda.synchronize()
        pe.infer_frames_async(src, fmt, rot, DEST, 8, 0.1, flip, scales)
        _assert_same(_results(pe, len(frames)), want)
        assert sum(len(r) for r, _ in want) > 0


def test_infer_frames_groups_like_infer_images(net):
    pe = _engine(net, "bf16", batch_cap=3)
    bgr = _bgr_frames(MIXED, 31)
    frames = [_yuv(f, "i420") for f in bgr]
    got = pe.infer_frames_arrays(frames, "i420", 90, DEST)
    want = pe.infer_images_arrays([_cv2_bgr(f, "i420", 90) for f in frames], DEST)
    assert len(got) == len(want) == len(frames)
    for g, w in zip(got, want):
        assert np.array_equal(g, w)


def test_launch_count_adds_one_conversion(net):
    nat = _nat()
    pe = _engine(net)
    bgr = _bgr_frames([(120, 160)] * 4, 41)
    nv12 = [_yuv(f, "nv12") for f in bgr]
    rotated = [_cv2_bgr(f, "bgr", 90) for f in bgr]

    def count(fn):
        fn()            # warm: plans and graphs of the shape exist before the counted call
        pe.fetch_arrays()
        l0 = nat.launch_count()
        fn()
        pe.fetch_arrays()
        return nat.launch_count() - l0

    for flip in (False, True):
        base = count(lambda: _reference(pe, bgr, flip, None))
        base_rot = count(lambda: _reference(pe, rotated, flip, None))
        packed = np.ascontiguousarray(np.stack(bgr))
        assert count(lambda: pe.infer_frames_async(list(packed), "bgr", 0, DEST, 8, 0.1, flip)) == base
        assert count(lambda: pe.infer_frames_async(nv12, "nv12", 0, DEST, 8, 0.1, flip)) == base + 1
        assert count(lambda: pe.infer_frames_async(bgr, "bgr", 90, DEST, 8, 0.1, flip)) == base_rot + 1
        pitched = [_padded_cuda(f, 7) for f in bgr]
        assert count(lambda: pe.infer_frames_async(pitched, "bgr", 0, DEST, 8, 0.1, flip)) == base + 1


def test_pose_stream_of_rotated_nv12_equals_host_rotated_bgr(built, he_sd):
    from lib.network.rtpose_vgg import get_model
    streaming, nat = pkg_module("streaming"), _nat()
    model = get_model("vgg19")
    model.load_state_dict(he_sd)
    model = model.cuda().float().eval()
    nv12 = [_yuv(f, "nv12") for f in _bgr_frames([(240, 320)] * 7, 11)]
    rot = nat.rotation_of(cv2.ROTATE_90_CLOCKWISE)
    host = [_cv2_bgr(f, "nv12", rot) for f in nv12]
    got = list(streaming.PoseStream(model, nv12, batch=3, format="nv12", rotate=rot))
    want = list(streaming.PoseStream(model, host, batch=3))
    assert len(got) == len(want) == 7
    assert sum(len(h) for _, h, _ in want) > 0
    for (gf, gh, gd), (wf, wh, wd) in zip(got, want):
        np.testing.assert_array_equal(gf, wf)
        assert len(gh) == len(wh)
        for a, b in zip(gh, wh):
            assert a.score == b.score and a.body_parts.keys() == b.body_parts.keys()
            for k in a.body_parts:
                pa, pb = a.body_parts[k], b.body_parts[k]
                assert (pa.x, pa.y, pa.score, pa.uidx) == (pb.x, pb.y, pb.score, pb.uidx)
        np.testing.assert_array_equal(gd, wd)


def test_invalid_frames_are_refused_naming_frame_and_field(net):
    nat, eng = _nat(), pkg_module("engine")
    pe = _engine(net, batch_cap=4)
    bgr = _bgr_frames([(120, 160)] * 3, 51)
    frames = [_yuv(f, "nv12") for f in bgr]

    def call(table, n, fmt=1, rot=0, flip=0):
        return nat.lib().b200pose_infer_frames(pe._net_h(), pe.post._h, table, n, fmt, 0, rot, DEST, 8, None, 0, pe.mode,
                                               ctypes.c_float(0.1), flip, None)

    def refused(expect, **kw):
        table, keep, _, _ = eng.frame_table(frames, "nv12")
        mutate = kw.pop("mutate", None)
        if mutate:
            mutate(table)
        with pytest.raises(nat.B200PoseError) as e:
            nat.check(call(table, kw.pop("n", 3), **kw), "b200pose_infer_frames")
        for word in expect:
            assert word in str(e.value), (expect, str(e.value))

    refused(["frame 1", "h = 119"], mutate=lambda t: setattr(t[1], "h", 119))
    refused(["frame 2", "pitch[1]"], mutate=lambda t: t[2].pitch.__setitem__(1, 100))
    refused(["format 5"], fmt=5)
    refused(["rotate 45"], rot=45)
    many = frames * 2
    table, keep, _, _ = eng.frame_table(many, "nv12")
    with pytest.raises(nat.B200PoseError) as e:
        nat.check(call(table, 6), "b200pose_infer_frames")
    assert "6 frames" in str(e.value)
    # the same engine then runs a clean call as the BGR path does
    want = _reference(pe, [_cv2_bgr(f, "nv12", 0) for f in frames], False, None)
    pe.infer_frames_async(frames, "nv12", 0, DEST)
    _assert_same(_results(pe, 3), want)
