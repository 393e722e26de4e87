"""Shared by tests/test_png_host.py and tests/test_gpu_png.py: a PNG writer in numpy + zlib with control over every
part of a stream (colour type, depth, PLTE / tRNS, Adam7, eXIf, the filter of each row, zlib level, strategy and
window, IDAT split sizes, extra chunks), damage helpers, and the host build of csrc/png_core.h
(tests/cuda/png_core_host.cpp)."""
import ctypes
import os
import struct
import subprocess
import zlib

import numpy as np

from conftest import ROOT

HOST_SRC = os.path.join(ROOT, "tests", "cuda", "png_core_host.cpp")
CSRC = os.path.join(ROOT, "pytorch_realtime_multi-person_pose_estimation_b200", "csrc")
SIG = b"\x89PNG\r\n\x1a\n"
# every legal (colour type, bit depth) pair
PAIRS = [(0, 1), (0, 2), (0, 4), (0, 8), (0, 16), (2, 8), (2, 16), (3, 1), (3, 2), (3, 4), (3, 8), (4, 8), (4, 16),
         (6, 8), (6, 16)]
CHANNELS = {0: 1, 2: 3, 3: 1, 4: 2, 6: 4}
STRATEGIES = {"default": zlib.Z_DEFAULT_STRATEGY, "filtered": zlib.Z_FILTERED, "huffman": zlib.Z_HUFFMAN_ONLY,
              "rle": zlib.Z_RLE, "fixed": zlib.Z_FIXED}
ADAM7 = [(0, 0, 8, 8), (4, 0, 8, 8), (0, 4, 4, 8), (2, 0, 4, 4), (0, 2, 2, 4), (1, 0, 2, 2), (0, 1, 1, 2)]   # x0 y0 dx dy


def compile_core(so, core=None, extra=()):
    """The host decoding core as a ctypes library; `core` replaces png_core.h (a copy with a planted mistake)."""
    cmd = ["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-I", CSRC, "-o", so, HOST_SRC]
    if core:
        cmd.insert(1, '-DPNG_CORE="%s"' % core)
    subprocess.run(cmd + list(extra), check=True)
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


def core_decode(lib, blob):
    """(rc, status, frame) of the host decoder; frame [oh, ow, 3] when rc == 0."""
    rc, _, _, oh, ow, _, _ = core_info(lib, blob)
    cap = max(3, 3 * oh * ow)
    out = np.zeros(cap, np.uint8)
    st = ctypes.c_uint(0)
    rc = lib.core_decode(blob, len(blob), out.ctypes.data, cap, ctypes.byref(st))
    return rc, st.value, (out[:3 * oh * ow].reshape(oh, ow, 3) if rc == 0 else None)


def cv2_decode(blob):
    """cv2.imdecode(blob, cv2.IMREAD_COLOR); None for an empty stream too (cv2 asserts on one)."""
    import cv2
    if not len(blob):
        return None
    return cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR)


# ------------------------------------------------------------------------------------------------ writing
def chunk(kind, data, crc=None):
    c = zlib.crc32(kind + data) & 0xFFFFFFFF if crc is None else crc
    return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", c)


def samples(h, w, ctype, depth, seed, kind="noise"):
    """Seeded samples [h, w, channels] in 0 .. 2^depth - 1: 'noise' or 'smooth' (gradients: long matches)."""
    rs = np.random.RandomState(seed)
    c, top = CHANNELS[ctype], (1 << depth) - 1
    if kind == "smooth":
        y, x = np.mgrid[0:h, 0:w]
        base = (y[..., None] * (3 + np.arange(c)) + x[..., None] * (1 + 2 * np.arange(c))) // 4
        return (base % (top + 1)).astype(np.int64)
    return rs.randint(0, top + 1, (h, w, c)).astype(np.int64)


def pack_rows(s, depth):
    """Rows of samples [h, w, c] as bytes [h, rowbytes] (big-endian 16-bit, MSB-first packing below 8 bits)."""
    h, w, c = s.shape
    flat = s.reshape(h, w * c)
    if depth == 16:
        return np.stack([flat >> 8, flat & 255], -1).reshape(h, 2 * w * c).astype(np.uint8)
    if depth == 8:
        return flat.astype(np.uint8)
    per = 8 // depth
    n = (w * c + per - 1) // per
    pad = np.zeros((h, n * per), np.int64)
    pad[:, :w * c] = flat
    v = pad.reshape(h, n, per)
    out = np.zeros((h, n), np.int64)
    for k in range(per):
        out |= v[:, :, k] << (8 - depth * (k + 1))
    return out.astype(np.uint8)


def _paeth(a, b, c):
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    return np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))


def filter_rows(raw, bpp, types):
    """Filtered rows (filter byte first) of raw rows [h, rb]: types[r] in 0 .. 4 for row r."""
    raw = raw.astype(np.int64)
    h, rb = raw.shape
    out = np.zeros((h, rb + 1), np.int64)
    for r in range(h):
        x = raw[r]
        prior = raw[r - 1] if r else np.zeros(rb, np.int64)
        a = np.concatenate([np.zeros(bpp, np.int64), x[:-bpp]])[:rb] if rb else x
        c = np.concatenate([np.zeros(bpp, np.int64), prior[:-bpp]])[:rb] if rb else x
        t = types[r]
        pred = [0 * x, a, prior, (a + prior) >> 1, _paeth(a, prior, c)][t]
        out[r, 0] = t
        out[r, 1:] = (x - pred) % 256
    return out.astype(np.uint8)


def image_data(s, ctype, depth, interlace=0, filters=0, seed=0):
    """The filtered bytes of samples s: filters an int (every row), a list (cycled over the rows) or 'random'."""
    h, w, c = s.shape
    bpp = max(1, c * depth // 8)
    rs = np.random.RandomState(seed)
    passes = [(0, 0, 1, 1)] if not interlace else ADAM7
    parts = []
    for x0, y0, dx, dy in passes:
        sub = s[y0::dy, x0::dx]
        if sub.shape[0] == 0 or sub.shape[1] == 0:
            continue
        raw = pack_rows(sub, depth)
        n = raw.shape[0]
        if filters == "random":
            types = list(rs.randint(0, 5, n))
        elif isinstance(filters, int):
            types = [filters] * n
        else:
            types = [filters[i % len(filters)] for i in range(n)]
        parts.append(filter_rows(raw, bpp, types).ravel())
    return np.concatenate(parts).tobytes() if parts else b""


def deflate(data, level=6, strategy="default", wbits=15):
    co = zlib.compressobj(level, zlib.DEFLATED, wbits, 8, STRATEGIES[strategy])
    return co.compress(data) + co.flush()


def exif_payload(orientation, order="II"):
    """An eXIf payload: a TIFF header whose IFD0 holds one SHORT orientation entry."""
    e = "<" if order == "II" else ">"
    return order.encode() + struct.pack(e + "HI", 42, 8) + struct.pack(e + "H", 1) + \
        struct.pack(e + "HHIHH", 0x0112, 3, 1, orientation, 0) + struct.pack(e + "I", 0)


def ihdr(h, w, ctype, depth, interlace=0):
    return chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, depth, ctype, 0, 0, interlace))


def build(s, ctype, depth, interlace=0, filters=0, level=6, strategy="default", wbits=15, split=None, plte=None,
          trns=None, exif=None, exif_after=False, before=(), after=(), zdata=None, seed=0):
    """A PNG stream of samples s [h, w, c].  split: IDAT data sizes (cycled; 0 gives empty chunks), default one chunk;
    plte: [k, 3] RGB entries (palette images default to 256 seeded entries); before / after: extra chunks ahead of
    / behind the IDATs; zdata: the zlib stream itself."""
    h, w, _ = s.shape
    z = deflate(image_data(s, ctype, depth, interlace, filters, seed), level, strategy, wbits) if zdata is None else zdata
    out = SIG + ihdr(h, w, ctype, depth, interlace)
    if ctype == 3 and plte is None:
        plte = np.random.RandomState(seed + 99).randint(0, 256, (256, 3))
    if plte is not None:
        out += chunk(b"PLTE", np.asarray(plte, np.uint8).tobytes())
    if trns is not None:
        out += chunk(b"tRNS", trns)
    if exif is not None and not exif_after:
        out += chunk(b"eXIf", exif)
    out += b"".join(before)
    out += idat_chunks(z, split)
    out += b"".join(after)
    if exif is not None and exif_after:
        out += chunk(b"eXIf", exif)
    return out + chunk(b"IEND", b"")


def idat_chunks(z, split=None):
    if not split:
        return chunk(b"IDAT", z)
    out, at, k = b"", 0, 0
    while at < len(z):
        n = split[k % len(split)]
        out += chunk(b"IDAT", z[at:at + n])
        at += n
        k += 1
    return out


def expected(s, ctype, depth, plte=None, seed=0):
    """What cv2.imdecode returns for samples s, restated from the colour rules (BGR uint8)."""
    h, w, c = s.shape
    if ctype == 3:
        pal = np.zeros((256, 3), np.int64)
        p = np.random.RandomState(seed + 99).randint(0, 256, (256, 3)) if plte is None else np.asarray(plte)
        pal[:len(p)] = p
        return pal[s[..., 0]][..., ::-1].astype(np.uint8)
    v = s >> 8 if depth == 16 else s * (255 // ((1 << depth) - 1)) if depth < 8 else s
    if ctype in (0, 4):
        return np.repeat(v[..., :1], 3, -1).astype(np.uint8)
    return v[..., 2::-1].astype(np.uint8)


def chunks_of(blob):
    """[(type, data)] of a stream's chunks."""
    out, i = [], 8
    while i + 12 <= len(blob):
        n = struct.unpack(">I", blob[i:i + 4])[0]
        out.append((blob[i + 4:i + 8], blob[i + 8:i + 8 + n]))
        i += 12 + n
    return out


def zlib_of(blob):
    return b"".join(d for t, d in chunks_of(blob) if t == b"IDAT")


def with_zlib(blob, z, split=None):
    """blob with its IDAT data replaced by z (CRCs recomputed): damage meant for the inflater."""
    cs = chunks_of(blob)
    first = next(i for i, (t, _) in enumerate(cs) if t == b"IDAT")
    rest = [c for c in cs[first:] if c[0] != b"IDAT"]
    return SIG + b"".join(chunk(t, d) for t, d in cs[:first]) + idat_chunks(z, split) + \
        b"".join(chunk(t, d) for t, d in rest)


def bad_crc(blob, kind, k=0):
    """blob with the CRC of its k-th chunk of type `kind` flipped."""
    i, seen = 8, 0
    while i + 12 <= len(blob):
        n = struct.unpack(">I", blob[i:i + 4])[0]
        if blob[i + 4:i + 8] == kind:
            if seen == k:
                j = i + 8 + n
                return blob[:j] + bytes([blob[j] ^ 0x5A]) + blob[j + 1:]
            seen += 1
        i += 12 + n
    raise ValueError(kind)
