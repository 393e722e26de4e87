"""Shared by tests/test_jpeg_host.py and tests/test_gpu_jpeg.py: seeded JPEG streams made with cv2.imencode (sampling
factors, qualities, restart intervals, optimised tables, EXIF orientations, extra APPn / COM segments) and the host
build of csrc/jpeg_core.h (tests/cuda/jpeg_core_host.cpp)."""
import ctypes
import os
import struct
import subprocess

import numpy as np

from conftest import ROOT

HOST_SRC = os.path.join(ROOT, "tests", "cuda", "jpeg_core_host.cpp")
CSRC = os.path.join(ROOT, "pytorch_realtime_multi-person_pose_estimation_b200", "csrc")
SAMPLING = {"444": 0x111111, "422": 0x211111, "420": 0x221111, "440": 0x121111, "411": 0x411111}


def compile_core(so, core=None):
    """The host decoding core as a ctypes library; `core` replaces jpeg_core.h (a copy with a planted mistake)."""
    cmd = ["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-I", CSRC, "-o", so, HOST_SRC]
    if core:
        cmd.insert(1, '-DJPEG_CORE="%s"' % core)
    subprocess.run(cmd, check=True)
    lib = ctypes.CDLL(so)
    lib.core_decode.argtypes = [ctypes.c_char_p, ctypes.c_longlong, ctypes.c_void_p, ctypes.c_longlong,
                                ctypes.POINTER(ctypes.c_uint)]
    lib.core_info.argtypes = [ctypes.c_char_p, ctypes.c_longlong, ctypes.c_void_p, ctypes.c_char_p, ctypes.c_int]
    return lib


def core_info(lib, blob):
    """(rc, h, w, oriented h, oriented w, supported, reason) of the host parse."""
    out = np.zeros(5, np.int32)
    reason = ctypes.create_string_buffer(256)
    rc = lib.core_info(blob, len(blob), out.ctypes.data, reason, 256)
    return (rc,) + tuple(int(v) for v in out) + (reason.value.decode(),)


def core_decode(lib, blob, cap=None):
    """(rc, status, frame) of the host decoder; frame [oh, ow, 3] when rc == 0."""
    rc, _, _, oh, ow, _, _ = core_info(lib, blob)
    cap = cap if cap is not None else max(3, 3 * oh * ow)
    out = np.zeros(cap, np.uint8)
    st = ctypes.c_uint(0)
    rc = lib.core_decode(blob, len(blob), out.ctypes.data, cap, ctypes.byref(st))
    return rc, st.value, (out[:3 * oh * ow].reshape(oh, ow, 3) if rc == 0 else None)


def content(h, w, seed, kind="photo"):
    """Seeded BGR content: smooth noise with edges ('photo'), or a 0 / 255 checkerboard ('checker': large AC
    coefficients at the edges of the sample range)."""
    rs = np.random.RandomState(seed)
    if kind == "checker":
        y, x = np.mgrid[0:h, 0:w]
        c = (((y // (1 + seed % 3)) + (x // (1 + seed % 2))) % 2 * 255).astype(np.uint8)
        return np.dstack([c, 255 - c, c])
    import cv2
    img = rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
    if h > 2 and w > 2:
        img = cv2.GaussianBlur(img, (5, 5), 1.5)
    yy, xx = np.mgrid[0:h, 0:w]
    img[(yy * 7 + xx * 3) % 41 < 4] = rs.randint(0, 256, 3)
    return img


def encode(img, quality=90, sampling="420", restart=0, optimize=False, luma=None, chroma=None, progressive=False):
    import cv2
    p = [cv2.IMWRITE_JPEG_QUALITY, int(quality), cv2.IMWRITE_JPEG_RST_INTERVAL, int(restart),
         cv2.IMWRITE_JPEG_OPTIMIZE, int(optimize), cv2.IMWRITE_JPEG_PROGRESSIVE, int(progressive)]
    if img.ndim == 3:
        p += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SAMPLING[sampling]]
    if luma is not None:
        p += [cv2.IMWRITE_JPEG_LUMA_QUALITY, int(luma), cv2.IMWRITE_JPEG_CHROMA_QUALITY, int(chroma)]
    ok, buf = cv2.imencode(".jpg", img, p)
    assert ok
    return buf.tobytes()


def gray(img):
    import cv2
    return cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)


def with_exif(blob, orientation, order="II", extra=False):
    """blob with an EXIF APP1 segment (IFD0: one SHORT orientation entry) right after SOI; extra: an APP2 and a COM
    segment before it and an APP13 after it."""
    e = "<" if order == "II" else ">"
    tiff = order.encode() + struct.pack(e + "HI", 42, 8) + struct.pack(e + "H", 1) + \
        struct.pack(e + "HHIHH", 0x0112, 3, 1, orientation, 0) + struct.pack(e + "I", 0)
    app1 = b"Exif\0\0" + tiff
    seg = b"\xff\xe1" + struct.pack(">H", len(app1) + 2) + app1
    if extra:
        junk = bytes(range(200)) * 3
        seg = b"\xff\xe2" + struct.pack(">H", len(junk) + 2) + junk + b"\xff\xfe\x00\x0bcomment" + \
            b"\xff\xff" + seg + b"\xff\xed\x00\x06abcd"
    return blob[:2] + seg + blob[2:]


def app1(payload):
    return b"\xff\xe1" + struct.pack(">H", len(payload) + 2) + payload


def exif_payload(orientation, order="II", ident=b"Exif\0\0", tag=0x0112):
    """An APP1 payload: `ident`, then a TIFF header whose IFD0 holds one SHORT entry `tag` = orientation."""
    e = "<" if order == "II" else ">"
    return ident + order.encode() + struct.pack(e + "HI", 42, 8) + struct.pack(e + "H", 1) + \
        struct.pack(e + "HHIHH", tag, 3, 1, orientation, 0) + struct.pack(e + "I", 0)


XMP = b"http://ns.adobe.com/xap/1.0/\0<x:xmpmeta xmlns:x='adobe:ns:meta/'/>"


def with_segments(blob, segments):
    """blob with the given marker segments inserted right after SOI."""
    return blob[:2] + b"".join(segments) + blob[2:]


def set_sof(blob, marker):
    """blob with its SOF0 marker byte replaced (e.g. 0xC9: an arithmetic-coded header)."""
    i = blob.index(b"\xff\xc0")
    return blob[:i + 1] + bytes([marker]) + blob[i + 2:]


def cmyk_header(blob):
    """A grayscale stream whose SOF declares four components (the header of a CMYK / YCCK stream)."""
    i = blob.index(b"\xff\xc0")
    n = struct.unpack(">H", blob[i + 2:i + 4])[0]
    sof = blob[i + 4:i + 2 + n]
    comps = b"".join(bytes([k + 1, 0x11, 0]) for k in range(4))
    new = sof[:5] + bytes([4]) + comps
    return blob[:i] + b"\xff\xc0" + struct.pack(">H", len(new) + 2) + new + blob[i + 2 + n:]


def scan_range(blob):
    """[begin, end) of the entropy-coded data: after the SOS header, up to EOI."""
    i = blob.index(b"\xff\xda")
    n = struct.unpack(">H", blob[i + 2:i + 4])[0]
    return i + 2 + n, blob.rindex(b"\xff\xd9")


def corrupt_set(seed=11):
    """Streams with damaged entropy data: truncated in the scan, bit-flipped, and over-long (junk before EOI)."""
    rs = np.random.RandomState(seed)
    out = []
    for k, (h, w, s, rst) in enumerate([(64, 80, "420", 0), (57, 43, "444", 3), (96, 96, "422", 1), (40, 72, "411", 0)]):
        blob = encode(content(h, w, seed + k), 85, s, rst)
        b, e = scan_range(blob)
        for frac in (0.2, 0.6, 0.97):
            out.append(("truncated_%d_%g" % (k, frac), blob[:b + int((e - b) * frac)]))
        for t in range(3):
            arr = bytearray(blob)
            for _ in range(24):
                p = rs.randint(b, e)
                if arr[p] != 0xFF and (p == 0 or arr[p - 1] != 0xFF):
                    arr[p] ^= 1 << rs.randint(8)
            out.append(("flipped_%d_%d" % (k, t), bytes(arr)))
        out.append(("overlong_%d" % k, blob[:e] + bytes(rs.randint(0, 255, 700).astype(np.uint8)) + blob[e:]))
    return out


_ZIGZAG = [0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
           21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60,
           61, 54, 47, 55, 62, 63]


def coef_stream(blocks, qt):
    """A baseline grayscale stream whose 8 x 8 blocks carry exactly the given quantised coefficients: blocks
    [by, bx, 64] int (natural order, DC absolute, |DC differences| < 32768, |AC| < 32768), qt 64 values 1 .. 255
    (natural order).  Its Huffman tables code every DC size 0 .. 15 and every AC run / size, so any coefficient reaches
    the IDCT - the sums past the sample range that encoded photos do not reach."""
    blocks = np.asarray(blocks, np.int64)
    bh, bw = blocks.shape[:2]
    dc_syms = list(range(16))
    ac_syms = [0x00, 0xF0] + [(r << 4) | s for r in range(16) for s in range(1, 16)]

    def table(syms, length):
        counts = [0] * 16
        counts[length - 1] = len(syms)
        return bytes(counts) + bytes(syms), {s: (i, length) for i, s in enumerate(syms)}

    dc_spec, dc_code = table(dc_syms, 5)
    ac_spec, ac_code = table(ac_syms, 8)
    bits = []

    def put(v, n):
        bits.extend((v >> (n - 1 - i)) & 1 for i in range(n))

    def value(v):
        size = int(abs(v)).bit_length()
        return size, (v if v >= 0 else v + (1 << size) - 1)

    pred = 0
    for by in range(bh):
        for bx in range(bw):
            b = blocks[by, bx]
            size, v = value(int(b[0]) - pred)
            pred = int(b[0])
            put(*dc_code[size])
            if size:
                put(v, size)
            run = 0
            zz = [int(b[_ZIGZAG[k]]) for k in range(64)]
            last = max([k for k in range(1, 64) if zz[k]] or [0])
            for k in range(1, last + 1):
                if zz[k] == 0:
                    run += 1
                    continue
                while run > 15:
                    put(*ac_code[0xF0])
                    run -= 16
                size, v = value(zz[k])
                put(*ac_code[(run << 4) | size])
                put(v, size)
                run = 0
            if last < 63:
                put(*ac_code[0x00])
    bits.extend([1] * (-len(bits) % 8))
    data = bytearray()
    for i in range(0, len(bits), 8):
        byte = int("".join(map(str, bits[i:i + 8])), 2)
        data.append(byte)
        if byte == 0xFF:
            data.append(0)

    def seg(marker, payload):
        return bytes([0xFF, marker]) + struct.pack(">H", len(payload) + 2) + payload

    dqt = bytes([0]) + bytes(int(qt[_ZIGZAG[k]]) for k in range(64))
    sof = struct.pack(">BHHB", 8, bh * 8, bw * 8, 1) + bytes([1, 0x11, 0])
    dht = bytes([0x00]) + dc_spec + bytes([0x10]) + ac_spec
    sos = bytes([1, 1, 0x00, 0, 63, 0])
    return b"\xff\xd8" + seg(0xDB, dqt) + seg(0xC0, sof) + seg(0xC4, dht) + seg(0xDA, sos) + bytes(data) + b"\xff\xd9"


def idct_range_set(seed=5):
    """Crafted streams whose IDCT sums leave the sample range in every way: DC-only blocks (the SIMD pass-1 shortcut,
    whose 16-bit shift wraps), large sparse and dense AC (16-bit dequantised products and word sums that wrap, pass 1
    saturating), and one-block streams whose DC alone, at quantisation 255, lies past the sample range."""
    rs = np.random.RandomState(seed)
    out = []
    q255 = np.full(64, 255)
    for dc in (17, 20, 30, 40, -17, -20, -30, -40, 127, -128, 300, 8191, -8192):
        b = np.zeros((1, 1, 64), np.int64)
        b[0, 0, 0] = dc
        out.append(("dc%d" % dc, coef_stream(b, q255)))
    for k in range(24):
        bh, bw = 2 + k % 3, 3 + k % 2
        b = np.zeros((bh, bw, 64), np.int64)
        mode = k % 4
        for y in range(bh):
            for x in range(bw):
                if mode == 0:      # DC and row 0 only: the pass-1 shortcut with large values
                    b[y, x, :8] = rs.randint(-3000, 3000, 8) * (rs.rand(8) < 0.6)
                elif mode == 1:    # sparse, huge
                    idx = rs.choice(64, 4, replace=False)
                    b[y, x, idx] = rs.randint(-32767, 32768, 4)
                elif mode == 2:    # dense, moderate
                    b[y, x] = rs.randint(-400, 400, 64)
                else:              # a few large AC next to a large DC
                    b[y, x, 0] = rs.randint(-2000, 2000)
                    b[y, x, rs.randint(1, 64)] = rs.randint(-6000, 6000)
        b[..., 0] = np.clip(b[..., 0], -16000, 16000)
        qt = rs.randint(1, 256, 64) if k % 3 else q255
        out.append(("random%d_mode%d" % (k, mode), coef_stream(b, qt)))
    return out
