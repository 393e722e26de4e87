"""GPU (-m gpu): PNG decoding on the device (DESIGN.md 2.17).  b200pose_net_decode_pngs must equal the host build of
csrc/png_core.h and cv2.imdecode bit for bit (tests/test_png_host.py ties the core to cv2), to host and to device
output, in uniform and ragged calls, with 4 KB sentinels around the output untouched; encode_pngs -> decode_pngs on the
device returns the frames; b200pose_infer_pngs must give the person rows and peaks infer_images gives on the frames
cv2.imdecode returns, APNG streams taking the cv2 fallback; a damaged stream raises naming its image and the engine
then runs the next batch correctly; and the path adds kPngLaunches launches to infer_raw_*."""
import ctypes
import struct

import numpy as np
import pytest
import torch

from conftest import pkg_module
import png_check as pc
import png_enc_check as pec

cv2 = pytest.importorskip("cv2")
pytestmark = pytest.mark.gpu

DEST = 96
SCALES = (0.5, 1.0, 1.5, 2.0)
SENT = 4096
PNG_LAUNCHES = 4


def _eng():
    return pkg_module("engine")


@pytest.fixture(scope="module")
def net(built, he_sd):
    n = _eng().NativeNet(0)
    n.load_state_dict_arrays([v.numpy() for v in he_sd.values()])
    return n


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    return pc.compile_core(str(tmp_path_factory.mktemp("png") / "libpngcore.so"))


def _engine(net, mode="bf16", batch_cap=8):
    return _eng().PoseEngine.from_net(net, mode=mode, batch_cap=batch_cap, peak_cap=1024, human_cap=2048)


def _photo(h, w, seed, orientation=None, interlace=0, level=6):
    """A photo-like BGR frame as an 8-bit RGB PNG with mixed filters, optionally with an eXIf orientation."""
    img = pec.frame(h, w, seed, "photo")
    s = img[..., ::-1].astype(np.int64)
    exif = None if orientation is None else pc.exif_payload(orientation, "MM" if seed % 2 else "II")
    return pc.build(s, 2, 8, interlace, "random", level=level, exif=exif, split=[4096], seed=seed)


def _set():
    """Every colour type and depth, interlaced and not, at odd sizes, zlib strategies and levels, split IDATs,
    orientations, cv2's own output and a larger frame."""
    out = []
    for k, (ct, d) in enumerate(pc.PAIRS):
        for il in (0, 1):
            s = pc.samples(17 + k, 29 + 2 * k, ct, d, k, "smooth" if il else "noise")
            out.append(pc.build(s, ct, d, il, "random", level=(k * 3 + il) % 10,
                                strategy=list(pc.STRATEGIES)[k % 5], split=[1, 0, 37], seed=k))
    for o in range(1, 9):
        out.append(_photo(21, 38, o, orientation=o, interlace=o % 2))
    for lvl in (0, 1, 9):
        out.append(cv2.imencode(".png", pec.frame(64, 80, lvl, "drawn"), [cv2.IMWRITE_PNG_COMPRESSION, lvl])[1].tobytes())
    out.append(_photo(480, 640, 3))
    out.append(_photo(1080, 1920, 4, interlace=1, level=1))
    return out


def _decode_raw(net, blobs, on_device):
    """b200pose_net_decode_pngs into a buffer with SENT sentinel bytes on both sides: (frames, sentinels intact)."""
    shapes = [pc.cv2_decode(b).shape for b in blobs]
    total = sum(int(np.prod(s)) for s in shapes)
    ptrs, sizes, keep = _eng().png_table(blobs)
    nat = pkg_module("_native")
    if on_device:
        buf = torch.full((total + 2 * SENT,), 0xA5, dtype=torch.uint8, device="cuda")
        nat.check(nat.lib().b200pose_net_decode_pngs(net._h, ptrs, sizes, len(blobs), ctypes.c_void_p(buf.data_ptr() + SENT),
                                                     1, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "decode")
        torch.cuda.synchronize()
        buf = buf.cpu().numpy()
    else:
        buf = np.full(total + 2 * SENT, 0xA5, np.uint8)
        nat.check(nat.lib().b200pose_net_decode_pngs(net._h, ptrs, sizes, len(blobs), ctypes.c_void_p(buf.ctypes.data + SENT),
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
    for start in range(0, len(blobs), 16):       # ragged calls of up to 16 streams
        part = blobs[start:start + 16]
        frames, ok = _decode_raw(net, part, on_device)
        assert ok, "sentinels around the output changed"
        for k, (b, f) in enumerate(zip(part, frames)):
            rc, st, host = pc.core_decode(core, b)
            assert rc == 0 and st == 0
            if not (np.array_equal(f, host) and np.array_equal(f, pc.cv2_decode(b))):
                bad.append(start + k)
    assert not bad, "frames differ: %s" % bad


def test_decode_uniform_call_and_tensor_api(net):
    blobs = [_photo(120, 160, s, interlace=s % 2) for s in range(6)]
    frames, ok = _decode_raw(net, blobs, True)
    assert ok
    for b, f in zip(blobs, frames):
        assert np.array_equal(f, pc.cv2_decode(b))
    for dev in (False, True):
        got = net.decode_pngs(blobs, device=dev)
        for b, g in zip(blobs, got):
            assert np.array_equal(g.cpu().numpy() if dev else g, pc.cv2_decode(b))


def test_encode_then_decode_on_the_device_returns_the_frames(net):
    frames = [pec.frame(h, w, k, kind) for k, (h, w, kind) in
              enumerate([(64, 80, "photo"), (33, 1, "noise"), (100, 120, "flat"), (57, 91, "stripes"), (240, 320, "drawn")])]
    files = net.encode_pngs(frames)
    got = net.decode_pngs([bytes(f) for f in files])
    for f, g in zip(frames, got):
        assert np.array_equal(f, g)


def _apng(h, w, seed):
    """An APNG whose IDAT is its first frame (acTL, then fcTL ahead of the IDAT)."""
    s = pec.frame(h, w, seed, "photo")[..., ::-1].astype(np.int64)
    fctl = pc.chunk(b"fcTL", struct.pack(">IIIIIHHBB", 0, w, h, 0, 0, 1, 10, 0, 0))
    return pc.build(s, 2, 8, before=[pc.chunk(b"acTL", struct.pack(">II", 1, 0)), fctl], seed=seed)


MIXED = [(120, 160), (96, 130), (160, 120), (100, 100), (88, 150), (120, 160), (132, 96), (110, 140)]


@pytest.mark.parametrize("mode", ["bf16", "fp32"])
@pytest.mark.parametrize("flip,scales", [(False, None), (True, None), (True, SCALES)], ids=["single", "flip", "ms_flip"])
@pytest.mark.parametrize("mixed", [False, True], ids=["uniform", "mixed"])
def test_infer_pngs_equals_infer_images(net, mode, flip, scales, mixed):
    shapes = MIXED if mixed else [(120, 160)] * 5
    # uniform: orientations that keep the frame's size; mixed: all eight
    blobs = [_photo(h, w, k, orientation=1 + k % (8 if mixed else 4), interlace=k % 2) for k, (h, w) in enumerate(shapes)]
    if mixed:   # APNG streams take the cv2.imdecode fallback
        blobs.insert(2, _apng(112, 150, 9))
        blobs.append(_apng(120, 160, 8))
    pe = _engine(net, mode)
    got = pe.infer_pngs_arrays(blobs, DEST, 8, 0.1, flip, scales)
    want = pe.infer_images_arrays([pc.cv2_decode(b) for b in blobs], DEST, 8, 0.1, flip, scales)
    assert len(got) == len(want) == len(blobs)
    for k, (g, w) in enumerate(zip(got, want)):
        assert np.array_equal(g, w), k
    if mixed:
        return
    # one device batch: its peaks equal those of infer_images' one batch of the same frames
    pe.infer_pngs_async(blobs, DEST, 8, 0.1, flip, scales)
    pe.fetch_arrays()
    pk_got = [pe.post.peaks(i) for i in range(len(blobs))]
    pe.infer_images_arrays([pc.cv2_decode(b) for b in blobs], DEST, 8, 0.1, flip, scales)
    pk_want = [pe.post.peaks(i) for i in range(len(blobs))]
    for g, w in zip(pk_got, pk_want):
        assert np.array_equal(g, w)


def _damaged(good):
    """Streams whose damage the device finds, each with the status bit it must set."""
    z = pc.zlib_of(good)
    adler = z[:-1] + bytes([z[-1] ^ 1])
    return [("idat_crc", pc.bad_crc(good, b"IDAT"), 8),
            ("adler", pc.with_zlib(good, adler), 4),
            ("short", pc.with_zlib(good, z[:len(z) // 2]), 2),
            ("btype3", pc.with_zlib(good, z[:2] + bytes([z[2] | 6]) + z[3:]), 1)]


def test_damaged_stream_raises_and_the_engine_recovers(net):
    nat = pkg_module("_native")
    pe = _engine(net)
    good = [_photo(96, 128, k) for k in range(3)]
    for name, bad, bit in _damaged(good[2]):
        assert cv2.imdecode(np.frombuffer(bad, np.uint8), cv2.IMREAD_COLOR) is None, name
        with pytest.raises(nat.B200PoseError, match=r"image\(s\) \[\(1, %d\)" % bit):
            pe.infer_pngs_arrays([good[0], bad, good[1]], DEST)
        with pytest.raises(nat.B200PoseError, match="png image 1"):
            net.decode_pngs([good[0], bad])
        pe.infer_pngs_async([good[0], bad], DEST)       # the asynchronous path raises at fetch
        with pytest.raises(nat.B200PoseError, match=r"image\(s\) \[\(1,"):
            pe.fetch_arrays(check=False)
        assert pe.post.jpeg_status(1) == 0
        got = pe.infer_pngs_arrays(good, DEST)
        want = pe.infer_images_arrays([pc.cv2_decode(b) for b in good], DEST)
        for g, w in zip(got, want):
            assert np.array_equal(g, w), name
    with pytest.raises(nat.B200PoseError, match="image 1"):
        pe.infer_pngs_arrays([good[0], good[1][:40]], DEST)
    with pytest.raises(nat.B200PoseError, match="png image 0: unsupported: APNG"):
        net.decode_pngs([_apng(40, 56, 2)])


def test_launch_count_adds_the_decoder(net):
    nat = pkg_module("_native")
    pe = _engine(net)
    blobs = [_photo(120, 160, k) for k in range(4)]
    frames = [pc.cv2_decode(b) for b in blobs]
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
        assert count(lambda: pe.infer_pngs_async(blobs, DEST, 8, 0.1, flip)) == base + PNG_LAUNCHES
    l0 = nat.launch_count()
    net.decode_pngs(blobs)
    assert nat.launch_count() - l0 == PNG_LAUNCHES
