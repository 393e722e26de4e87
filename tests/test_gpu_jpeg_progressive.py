"""GPU (-m gpu): progressive JPEG decoding on the device (DESIGN.md 2.18).  With the net's switch on,
b200pose_net_decode_jpegs must equal the host build of the progressive path of csrc/jpeg_core.h and cv2.imdecode bit for
bit (tests/test_jpeg_progressive_host.py ties the core to cv2) on cv2's progressive output and the writer's scripts, to
host and to device output, uniform and ragged, baseline and progressive streams mixed in one call, with 4 KB sentinels
around the output untouched; infer_jpegs must give the person rows and peaks infer_images gives on cv2-decoded frames
without taking the cv2 fallback for any stream it accepts; damaged streams raise naming the image and the engine
recovers; a call makes the documented launches; and with the switch off the old refusal holds."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import pkg_module
import jpeg_check as jc
import jpeg_prog_check as pc

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu

DEST = 96
SCALES = (0.5, 1.0, 1.5, 2.0)
SENT = 4096
JPEG_LAUNCHES, PROG_LAUNCHES, PROG_ONLY_LAUNCHES = 5, 6, 4


def _eng():
    return pkg_module("engine")


@pytest.fixture(scope="module")
def net(built, he_sd):
    n = _eng().NativeNet(0)
    n.load_state_dict_arrays([v.numpy() for v in he_sd.values()])
    n.set_jpeg_progressive(True)
    yield n
    n.set_jpeg_progressive(False)


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    return pc.compile_core(str(tmp_path_factory.mktemp("jpegprog") / "libjpegprog.so"))


def _engine(net, mode="bf16", batch_cap=8, progressive=True):
    return _eng().PoseEngine.from_net(net, mode=mode, batch_cap=batch_cap, peak_cap=1024, human_cap=2048,
                                      jpeg_progressive=progressive)


def _img(h, w, seed, kind):
    img = jc.content(h, w, seed)
    return jc.gray(img) if kind == "gray" else img


def _prog(h, w, seed, kind, quality=90, restart=0):
    return pc.cv2_progressive(_img(h, w, seed, kind), quality, "420" if kind == "gray" else kind, restart)


def _base(h, w, seed, kind, quality=90, restart=0):
    return jc.encode(_img(h, w, seed, kind), quality, "420" if kind == "gray" else kind, restart)


def _writer_set():
    out = []
    for kind in ("420", "444", "gray"):
        samp = pc.SAMP[kind]
        nc = len(samp)
        qts = [np.random.RandomState(c).randint(1, 30, 64) for c in range(nc)]
        blocks = pc.random_blocks(37, 53, samp, 3)
        for script in (pc.spectral_only(nc), pc.successive(nc, 13)):
            for rst in (0, 3):
                out.append(pc.write(blocks, 37, 53, script, samp, qts, restart=rst))
        full = [((c,), 0, 0, 0, 0) for c in range(nc)] + [((c,), 1, 9, 0, 0) for c in range(nc)]
        out.append(pc.write(blocks, 37, 53, full + [((0,), 10, 63, 0, 1)], samp, qts))       # incomplete at >= 10
    return out


def _set():
    """cv2's progressive output for every sampling and grayscale at several qualities, restart intervals and sizes,
    EXIF orientations, the writer's scripts, and baseline streams among them."""
    out = []
    for k, kind in enumerate(list(jc.SAMPLING) + ["gray"]):
        for q, rst in ((1, 0), (50, 7), (100, 1), (95, 50)):
            out.append(_prog(33 + k, 47, q + k, kind, q, rst))
        out.append(_prog(1, 17, k, kind))
        out.append(_prog(480, 640, k, kind, 85, 7 * (k % 2)))
        out.append(_base(64, 80, k, kind, 85, k % 2))
        for o in range(1, 9, 3):
            out.append(jc.with_exif(_prog(21, 38, o + k, kind, 90, o % 3), o))
    out.append(_prog(1080, 1920, 2, "420", 95))
    return out + _writer_set()


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
    for start in range(0, len(blobs), 24):       # ragged calls of up to 24 streams, baseline and progressive mixed
        part = blobs[start:start + 24]
        frames, ok = _decode_raw(net, part, on_device)
        assert ok, "sentinels around the output changed"
        for k, (b, f) in enumerate(zip(part, frames)):
            rc, st, host = pc.decode(core, b)
            assert rc == 0 and st == 0
            if not (np.array_equal(f, host) and np.array_equal(f, _cv2(b))):
                bad.append(start + k)
    assert not bad, "frames differ: %s" % bad


def test_decode_uniform_call_and_tensor_api(net):
    blobs = [_prog(120, 160, s, "420", 80 + s, 3 * (s % 2)) for s in range(6)]
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
def test_infer_jpegs_equals_infer_images(net, mode, flip, scales, mixed, monkeypatch):
    shapes = MIXED if mixed else [(120, 160, "420")] * 5
    blobs = [jc.with_exif(_prog(h, w, k, s, 90, k % 2), 1 + k % (8 if mixed else 4)) for k, (h, w, s) in enumerate(shapes)]
    if mixed:   # baseline streams in the same device batches
        blobs.insert(2, _base(112, 150, 9, "420"))
        blobs.append(_base(120, 160, 8, "444", 90, 2))
    pe = _engine(net, mode)
    want = pe.infer_images_arrays([_cv2(b) for b in blobs], DEST, 8, 0.1, flip, scales)
    fallback = []
    real = pe.infer_images

    def spy(frames, *a, **kw):
        fallback.append(len(frames))
        return real(frames, *a, **kw)
    monkeypatch.setattr(pe, "infer_images", spy)
    got = pe.infer_jpegs_arrays(blobs, DEST, 8, 0.1, flip, scales)
    monkeypatch.undo()
    assert not fallback, "accepted streams took the cv2 fallback"
    assert len(got) == len(want) == len(blobs)
    for k, (g, w) in enumerate(zip(got, want)):
        assert np.array_equal(g, w), k
    if mixed:
        return
    pe.infer_jpegs_async(blobs, DEST, 8, 0.1, flip, scales)
    pe.fetch_arrays()
    pk_got = [pe.post.peaks(i) for i in range(len(blobs))]
    pe.infer_images_arrays([_cv2(b) for b in blobs], DEST, 8, 0.1, flip, scales)
    pk_want = [pe.post.peaks(i) for i in range(len(blobs))]
    for g, w in zip(pk_got, pk_want):
        assert np.array_equal(g, w)


def _damaged():
    rs = np.random.RandomState(5)
    out = []
    for k, (h, w, s, rst) in enumerate([(64, 80, "420", 0), (57, 43, "444", 3), (40, 72, "gray", 1)]):
        blob = _prog(h, w, k, s, 85, rst)
        b, e = blob.index(b"\xff\xda"), blob.rindex(b"\xff\xd9")
        for t in range(3):
            arr = bytearray(blob)
            for _ in range(24):
                p = rs.randint(b + 20, e)
                if arr[p] != 0xFF and arr[p - 1] != 0xFF:
                    arr[p] ^= 1 << rs.randint(8)
            out.append(("flipped_%d_%d" % (k, t), bytes(arr)))
        out.append(("truncated_%d" % k, blob[:b + int((e - b) * 0.97)]))
    return out


def test_damaged_stream_raises_and_the_engine_recovers(net, core):
    nat = pkg_module("_native")
    pe = _engine(net)
    good = [_prog(96, 128, k, "420", 85) for k in range(3)]
    tried = 0
    for name, bad in _damaged():
        rc, st, _ = pc.decode(core, bad)
        if rc != 0 or st == 0:      # refused on the host, or damage the decoder cannot see
            continue
        tried += 1
        with pytest.raises(nat.B200PoseError, match=r"image\(s\) \[\(1,"):
            pe.infer_jpegs_arrays([good[0], bad, good[1]], DEST)
        with pytest.raises(nat.B200PoseError, match="jpeg image 1"):
            net.decode_jpegs([good[0], bad])
        got = pe.infer_jpegs_arrays(good, DEST)
        want = pe.infer_images_arrays([_cv2(b) for b in good], DEST)
        for g, w in zip(got, want):
            assert np.array_equal(g, w), name
    assert tried >= 3
    invalid = pc.write(pc.random_blocks(16, 24, pc.SAMP["gray"], 1), 16, 24, [((0,), 0, 0, 0, 0), ((0,), 0, 5, 0, 0)])
    ptrs, sizes, keep = _eng().jpeg_table([good[0], invalid])
    out = np.empty(96 * 128 * 3 + 16 * 24 * 3, np.uint8)
    assert nat.lib().b200pose_net_decode_jpegs(net._h, ptrs, sizes, 2, ctypes.c_void_p(out.ctypes.data), 0, None) != 0
    assert "jpeg image 1: malformed scan 1" in nat.lib().b200pose_last_error().decode()
    with pytest.raises(nat.B200PoseError, match="malformed scan 1"):
        net.decode_jpegs([good[0], invalid])


def _count(pe, fn):
    nat = pkg_module("_native")
    fn()
    pe.fetch_arrays()
    l0 = nat.launch_count()
    fn()
    pe.fetch_arrays()
    return nat.launch_count() - l0


def test_launch_counts(net):
    pe = _engine(net)
    prog = [_prog(120, 160, k, "420", 90) for k in range(4)]
    base = [_base(120, 160, k, "420", 90) for k in range(4)]
    batch = np.ascontiguousarray(np.stack([_cv2(b) for b in prog]))
    for flip in (False, True):
        raw = _count(pe, lambda: pe.infer_raw_async_u8(batch.ctypes.data, False, 4, 120, 160, DEST, 8, 0.1, flip))
        assert _count(pe, lambda: pe.infer_jpegs_async(prog, DEST, 8, 0.1, flip)) == raw + PROG_ONLY_LAUNCHES
        mixed = prog[:2] + base[:2]
        assert _count(pe, lambda: pe.infer_jpegs_async(mixed, DEST, 8, 0.1, flip)) == raw + PROG_LAUNCHES
        # without progressive streams, today's launches even with the switch on
        assert _count(pe, lambda: pe.infer_jpegs_async(base, DEST, 8, 0.1, flip)) == raw + JPEG_LAUNCHES


def test_switch_off_keeps_the_refusal(net):
    nat = pkg_module("_native")
    blob = _prog(40, 56, 2, "420")
    assert net.jpeg_progressive
    net.set_jpeg_progressive(False)
    try:
        assert not net.jpeg_progressive
        with pytest.raises(nat.B200PoseError, match="jpeg image 0: unsupported: progressive"):
            net.decode_jpegs([blob])
        assert _eng().jpeg_info(blob)[2] is False and _eng().jpeg_info(blob, progressive=True)[2] is True
    finally:
        net.set_jpeg_progressive(True)
    assert np.array_equal(net.decode_jpegs([blob])[0], _cv2(blob))
    # an engine with the switch off decodes progressive streams by cv2.imdecode, and sets the net's switch per submission
    pe = _engine(net, progressive=False)
    got = pe.infer_jpegs_arrays([blob], DEST)
    assert not net.jpeg_progressive
    with pytest.raises(nat.B200PoseError, match="unsupported: progressive"):
        pe.infer_jpegs_async([blob], DEST)
    pe.set_jpeg_progressive(True)
    assert all(np.array_equal(g, w) for g, w in zip(pe.infer_jpegs_arrays([blob], DEST), got))
    assert net.jpeg_progressive
