"""GPU (-m gpu): JPEG decoding on the device (DESIGN.md 2.13).  b200pose_net_decode_jpegs must equal the host build of
csrc/jpeg_core.h and cv2.imdecode bit for bit (tests/test_jpeg_host.py ties the core to cv2), to host and to device
output, in uniform and ragged calls, with 4 KB sentinels around the output untouched; b200pose_infer_jpegs must give
the person rows and peaks infer_images gives on the frames cv2.imdecode returns, progressive streams taking the cv2
fallback; a damaged stream raises naming its image; and the path adds kJpegLaunches launches to infer_raw_*."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import pkg_module
import jpeg_check as jc

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu

DEST = 96
SCALES = (0.5, 1.0, 1.5, 2.0)
SENT = 4096
JPEG_LAUNCHES = 5


def _eng():
    return pkg_module("engine")


@pytest.fixture(scope="module")
def net(built, he_sd):
    n = _eng().NativeNet(0)
    n.load_state_dict_arrays([v.numpy() for v in he_sd.values()])
    return n


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    return jc.compile_core(str(tmp_path_factory.mktemp("jpeg") / "libjpegcore.so"))


def _engine(net, mode="bf16", batch_cap=8):
    return _eng().PoseEngine.from_net(net, mode=mode, batch_cap=batch_cap, peak_cap=1024, human_cap=2048)


def _blob(h, w, seed, kind, **kw):
    img = jc.content(h, w, seed, kw.pop("content", "photo"))
    return jc.encode(jc.gray(img) if kind == "gray" else img, sampling="420" if kind == "gray" else kind, **kw)


def _set():
    """Every sampling factor and grayscale at three qualities and restart intervals, optimised tables, separate luma /
    chroma quality, checkerboards, EXIF orientations in both byte orders with extra segments, odd and larger sizes."""
    out = []
    for k, kind in enumerate(list(jc.SAMPLING) + ["gray"]):
        for q, rst, opt in ((1, 0, False), (50, 7, True), (100, 1, False), (95, 0, True)):
            out.append(_blob(33 + k, 47, q + k, kind, quality=q, restart=rst, optimize=opt))
        out.append(_blob(24, 40, k, kind, quality=100, content="checker"))
        out.append(_blob(1, 17, k, kind, quality=90))
        out.append(_blob(480, 640, k, kind, quality=85, restart=7 * (k % 2)))
        for o in range(1, 9):
            out.append(jc.with_exif(_blob(21, 38, o + k, kind, quality=90, restart=o % 3), o, "MM" if o % 2 else "II",
                                    extra=o % 3 == 0))
    for kind in jc.SAMPLING:
        out.append(_blob(37, 53, 5, kind, luma=90, chroma=10))
    out.append(_blob(1080, 1920, 2, "420", quality=95))
    return out


def _cv2(blob):
    return cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR)


def _decode_raw(net, blobs, on_device):
    """b200pose_net_decode_jpegs into a buffer with SENT sentinel bytes on both sides: (frames, sentinels intact)."""
    shapes = [_cv2(b).shape for b in blobs]
    total = sum(int(np.prod(s)) for s in shapes)
    ptrs, sizes, keep = _eng().jpeg_table(blobs)
    nat = pkg_module("_native")
    if on_device:
        buf = torch.full((total + 2 * SENT,), 0xA5, dtype=torch.uint8, device="cuda")
        nat.check(nat.lib().b200pose_net_decode_jpegs(net._h, ptrs, sizes, len(blobs), ctypes.c_void_p(buf.data_ptr() + SENT),
                                                      1, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "decode")
        torch.cuda.synchronize()
        buf = buf.cpu().numpy()
    else:
        buf = np.full(total + 2 * SENT, 0xA5, np.uint8)
        nat.check(nat.lib().b200pose_net_decode_jpegs(net._h, ptrs, sizes, len(blobs), ctypes.c_void_p(buf.ctypes.data + SENT),
                                                      0, None), "decode")
    ok = bool((buf[:SENT] == 0xA5).all() and (buf[SENT + total:] == 0xA5).all())
    frames, at = [], SENT
    for s in shapes:
        n = int(np.prod(s))
        frames.append(buf[at:at + n].reshape(s))
        at += n
    return frames, ok


@pytest.mark.parametrize("on_device", [False, True])
def test_decode_equals_host_core_and_cv2(net, core, on_device):
    blobs = _set()
    bad = []
    for start in range(0, len(blobs), 24):       # ragged calls of up to 24 streams
        part = blobs[start:start + 24]
        frames, ok = _decode_raw(net, part, on_device)
        assert ok, "sentinels around the output changed"
        for k, (b, f) in enumerate(zip(part, frames)):
            rc, st, host = jc.core_decode(core, b)
            assert rc == 0 and st == 0
            if not (np.array_equal(f, host) and np.array_equal(f, _cv2(b))):
                bad.append(start + k)
    assert not bad, "frames differ: %s" % bad


def test_decode_uniform_call_and_tensor_api(net):
    blobs = [_blob(120, 160, s, "420", quality=80 + s) for s in range(6)]
    frames, ok = _decode_raw(net, blobs, True)
    assert ok
    for b, f in zip(blobs, frames):
        assert np.array_equal(f, _cv2(b))
    for dev in (False, True):
        got = net.decode_jpegs(blobs, device=dev)
        for b, g in zip(blobs, got):
            assert np.array_equal(g.cpu().numpy() if dev else g, _cv2(b))


MIXED = [(120, 160, "420"), (96, 130, "444"), (160, 120, "422"), (100, 100, "gray"), (88, 150, "411"),
         (120, 160, "440"), (132, 96, "420"), (110, 140, "420")]


@pytest.mark.parametrize("mode", ["bf16", "fp32"])
@pytest.mark.parametrize("flip,scales", [(False, None), (True, None), (True, SCALES)], ids=["single", "flip", "ms_flip"])
@pytest.mark.parametrize("mixed", [False, True], ids=["uniform", "mixed"])
def test_infer_jpegs_equals_infer_images(net, mode, flip, scales, mixed):
    shapes = MIXED if mixed else [(120, 160, "420")] * 5
    # uniform: orientations that keep the frame's size; mixed: all eight
    blobs = [jc.with_exif(_blob(h, w, k, s, quality=90, restart=k % 2), 1 + k % (8 if mixed else 4))
             for k, (h, w, s) in enumerate(shapes)]
    if mixed:   # progressive streams take the cv2.imdecode fallback
        blobs.insert(2, jc.encode(jc.content(112, 150, 9), 90, "420", progressive=True))
        blobs.append(jc.encode(jc.content(120, 160, 8), 90, "420", progressive=True))
    pe = _engine(net, mode)
    got = pe.infer_jpegs_arrays(blobs, DEST, 8, 0.1, flip, scales)
    want = pe.infer_images_arrays([_cv2(b) for b in blobs], DEST, 8, 0.1, flip, scales)
    assert len(got) == len(want) == len(blobs)
    for k, (g, w) in enumerate(zip(got, want)):
        assert np.array_equal(g, w), k
    if mixed:
        return
    # one device batch: its peaks equal those of infer_images' one batch of the same frames
    dev = blobs
    pe.infer_jpegs_async(dev, DEST, 8, 0.1, flip, scales)
    pe.fetch_arrays()
    pk_got = [pe.post.peaks(i) for i in range(len(dev))]
    frames = [_cv2(b) for b in dev]
    pe.infer_images_arrays(frames, DEST, 8, 0.1, flip, scales)
    pk_want = [pe.post.peaks(i) for i in range(len(dev))]
    for g, w in zip(pk_got, pk_want):
        assert np.array_equal(g, w)


def test_damaged_stream_raises_and_the_engine_recovers(net):
    pe = _engine(net)
    good = [_blob(96, 128, k, "420", quality=85) for k in range(3)]
    for name, bad in jc.corrupt_set()[:8]:
        info = _eng().jpeg_info(bad)
        if not info[2]:
            continue
        with pytest.raises(pkg_module("_native").B200PoseError, match=r"image\(s\) \[\(1,"):
            pe.infer_jpegs_arrays([good[0], bad, good[1]], DEST)
        with pytest.raises(pkg_module("_native").B200PoseError, match="jpeg image 1"):
            net.decode_jpegs([good[0], bad])
        pe.infer_jpegs_async([good[0], bad], DEST)       # the asynchronous path raises at fetch
        with pytest.raises(pkg_module("_native").B200PoseError, match=r"image\(s\) \[\(1,"):
            pe.fetch_arrays(check=False)
        got = pe.infer_jpegs_arrays(good, DEST)
        want = pe.infer_images_arrays([_cv2(b) for b in good], DEST)
        for g, w in zip(got, want):
            assert np.array_equal(g, w), name
    with pytest.raises(pkg_module("_native").B200PoseError, match="image 1"):
        pe.infer_jpegs_arrays([good[0], b"\xff\xd8\xff\xc0\x00"], DEST)
    with pytest.raises(pkg_module("_native").B200PoseError, match="jpeg image 0: unsupported: progressive"):
        net.decode_jpegs([jc.encode(jc.content(40, 56, 2), 90, "420", progressive=True)])


def test_launch_count_adds_the_decoder(net):
    nat = pkg_module("_native")
    pe = _engine(net)
    blobs = [_blob(120, 160, k, "420", quality=90) for k in range(4)]
    frames = [_cv2(b) for b in blobs]
    batch = np.ascontiguousarray(np.stack(frames))

    def count(fn):
        fn()
        pe.fetch_arrays()
        l0 = nat.launch_count()
        fn()
        pe.fetch_arrays()
        return nat.launch_count() - l0

    for flip in (False, True):
        base = count(lambda: pe.infer_raw_async_u8(batch.ctypes.data, False, 4, 120, 160, DEST, 8, 0.1, flip))
        assert count(lambda: pe.infer_jpegs_async(blobs, DEST, 8, 0.1, flip)) == base + JPEG_LAUNCHES
