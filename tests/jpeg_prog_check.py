"""Shared by tests/test_jpeg_progressive_host.py and tests/test_gpu_jpeg_progressive.py: a JPEG writer that controls
every part of a progressive stream, and the host build of the progressive path of csrc/jpeg_core.h
(tests/cuda/jpeg_prog_host.cpp).

write(comps, h, w, script, ...) takes quantised coefficient blocks per component and a scan script and restates
libjpeg's jcphuff.c encoder (DC first / refinement, AC first with EOB runs up to 32767, AC refinement with its
correction bits) or, for a script of None, jchuff.c's one interleaved sequential scan (SOF0).  Each scan may carry its
own restart interval, quantisation tables written before it, and Huffman tables of its own (DHT before the scan, the
table ids it names in its SOS) or none (a DC refinement scan); every table codes every symbol, so crafted coefficients
and symbols reach the decoder.  A scan's `emit` replaces its entropy data with raw symbols (crafted streams)."""
import ctypes
import os
import struct
import subprocess

import numpy as np

from conftest import ROOT
import jpeg_check as jc

HOST_SRC = os.path.join(ROOT, "tests", "cuda", "jpeg_prog_host.cpp")
ZZ = jc._ZIGZAG
DC_SYMS = list(range(16))
AC_SYMS = [r << 4 for r in range(15)] + [0xF0] + [(r << 4) | s for r in range(16) for s in range(1, 16)]


def compile_core(so, core=None, asan=False):
    """The host core as a ctypes library (asan: a standalone executable); `core` replaces jpeg_core.h."""
    cmd = ["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-I", jc.CSRC, "-o", so, HOST_SRC]
    cmd[1:1] = ["-O1", "-g", "-fsanitize=address,undefined", "-fno-sanitize-recover=all", "-DJPEG_PROG_HOST_MAIN"] \
        if asan else ["-shared", "-fPIC"]
    if core:
        cmd.insert(1, '-DJPEG_CORE="%s"' % core)
    subprocess.run(cmd, check=True)
    if asan:
        return so
    lib = ctypes.CDLL(so)
    lib.prog_decode.argtypes = [ctypes.c_char_p, ctypes.c_longlong, ctypes.c_void_p, ctypes.c_longlong,
                                ctypes.POINTER(ctypes.c_uint)]
    lib.prog_info.argtypes = [ctypes.c_char_p, ctypes.c_longlong, ctypes.c_int, ctypes.c_void_p, ctypes.c_char_p,
                              ctypes.c_int]
    return lib


def info(lib, blob, progressive=True):
    """(rc, h, w, oriented h, oriented w, supported, progressive, reason) of the host parse."""
    out = np.zeros(6, np.int32)
    reason = ctypes.create_string_buffer(256)
    rc = lib.prog_info(blob, len(blob), int(progressive), out.ctypes.data, reason, 256)
    return (rc,) + tuple(int(v) for v in out) + (reason.value.decode(),)


def decode(lib, blob):
    """(rc, status, frame) of the host decoder with progressive streams on; frame [oh, ow, 3] when rc == 0."""
    oh, ow = info(lib, blob)[3:5]
    cap = max(3, 3 * oh * ow)
    out = np.zeros(cap, np.uint8)
    st = ctypes.c_uint(0)
    rc = lib.prog_decode(blob, len(blob), out.ctypes.data, cap, ctypes.byref(st))
    return rc, st.value, (out[:3 * oh * ow].reshape(oh, ow, 3) if rc == 0 else None)


def mismatch(lib, blob):
    """None when the host core equals cv2.imdecode, else a description."""
    import cv2
    want = cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR)
    rc, st, got = decode(lib, blob)
    if want is None:
        return "cv2 returns None"
    if rc != 0 or st != 0:
        return "rc %d status %d" % (rc, st)
    if got.shape != want.shape:
        return "shape %s vs %s" % (got.shape, want.shape)
    bad = int((got != want).any(-1).sum())
    return "%d pixels differ" % bad if bad else None


def cv2_progressive(img, quality=90, sampling="420", restart=0):
    return jc.encode(img, quality, sampling, restart, progressive=True)


# ------------------------------------------------------------------------------------------------------- the writer
CV2_SCRIPT_YCC = [((0, 1, 2), 0, 0, 0, 1), ((0,), 1, 5, 0, 2), ((2,), 1, 63, 0, 1), ((1,), 1, 63, 0, 1),
                  ((0,), 6, 63, 0, 2), ((0,), 1, 63, 2, 1), ((0, 1, 2), 0, 0, 1, 0), ((2,), 1, 63, 1, 0),
                  ((1,), 1, 63, 1, 0), ((0,), 1, 63, 1, 0)]
CV2_SCRIPT_GRAY = [((0,), 0, 0, 0, 1), ((0,), 1, 5, 0, 2), ((0,), 6, 63, 0, 2), ((0,), 1, 63, 2, 1),
                   ((0,), 0, 0, 1, 0), ((0,), 1, 63, 1, 0)]


def spectral_only(nc):
    """Spectral selection without successive approximation: DC interleaved, then bands per component."""
    out = [(tuple(range(nc)), 0, 0, 0, 0)]
    for c in range(nc):
        out += [((c,), 1, 2, 0, 0), ((c,), 3, 9, 0, 0), ((c,), 10, 30, 0, 0), ((c,), 31, 63, 0, 0)]
    return out


def successive(nc, top=13):
    """Successive approximation from Al top down to 0, every coefficient: DC per component (non-interleaved), AC
    whole band."""
    out = [((c,), 0, 0, 0, top) for c in range(nc)] + [((c,), 1, 63, 0, top) for c in range(nc)]
    for al in range(top - 1, -1, -1):
        out += [((c,), 0, 0, al + 1, al) for c in range(nc)] + [((c,), 1, 63, al + 1, al) for c in range(nc)]
    return out


class _Bits:
    def __init__(self):
        self.bits = []

    def put(self, v, n):
        self.bits.extend((int(v) >> (n - 1 - i)) & 1 for i in range(n))

    def flush(self):
        """Pads to a byte with ones and stuffs 0xFF bytes."""
        self.bits.extend([1] * (-len(self.bits) % 8))
        out = bytearray()
        for i in range(0, len(self.bits), 8):
            b = int("".join(map(str, self.bits[i:i + 8])), 2)
            out.append(b)
            if b == 0xFF:
                out.append(0)
        self.bits = []
        return bytes(out)


def _table(syms, length):
    """A DHT body coding syms canonically: as many as fit at `length` bits (no code all ones, at most 255), the rest one bit
    longer; and symbol -> (code, length)."""
    first = min(len(syms), (1 << length) - 1, 255)      # a DHT count is one byte
    counts = [0] * 16
    counts[length - 1] = first
    counts[length] = len(syms) - first
    codes = {s: (i, length) for i, s in enumerate(syms[:first])}
    codes.update({s: ((first << 1) + i, length + 1) for i, s in enumerate(syms[first:])})
    return bytes(counts) + bytes(syms), codes


DC_SPEC, DC_CODE = _table(DC_SYMS, 5)
AC_SPEC, AC_CODE = _table(AC_SYMS, 9)


def _size(v):
    v = int(v)
    s = abs(v).bit_length()
    return s, (v if v >= 0 else v + (1 << s) - 1)


def _seg(marker, payload):
    return bytes([0xFF, marker]) + struct.pack(">H", len(payload) + 2) + payload


def _geometry(h, w, samp):
    hmax = max(s[0] for s in samp)
    vmax = max(s[1] for s in samp)
    mx, my = -(-w // (8 * hmax)), -(-h // (8 * vmax))
    g = []
    for hs, vs in samp:
        dw, dh = -(-w * hs // hmax), -(-h * vs // vmax)
        g.append(dict(h=hs, v=vs, bw=mx * hs, bh=my * vs, wb=-(-dw // 8), hb=-(-dh // 8)))
    return mx, my, g


def _units(comps, g, mx, my):
    """The blocks of each unit of a scan of these components: [(component, by, bx), ...] per unit."""
    if len(comps) == 1:
        c = comps[0]
        return [[(c, by, bx)] for by in range(g[c]["hb"]) for bx in range(g[c]["wb"])]
    return [[(c, my_ * g[c]["v"] + y, mx_ * g[c]["h"] + x) for c in comps for y in range(g[c]["v"])
             for x in range(g[c]["h"])] for my_ in range(my) for mx_ in range(mx)]


def _irs(v, n):
    return int(v) >> n      # libjpeg's IRIGHT_SHIFT: arithmetic


class _AcEncoder:
    """jcphuff.c's AC first and refinement encoders for one scan: the EOB run and, for refinement, the correction bits
    buffered behind it (BE)."""

    def __init__(self, bw, ss, se, ah, al, eob_max=0x7FFF):
        self.bw, self.ss, self.se, self.ah, self.al, self.eob_max = bw, ss, se, ah, al, eob_max
        self.eobrun, self.be = 0, []

    def emit_eobrun(self):
        if self.eobrun:
            r = self.eobrun.bit_length() - 1
            self.bw.put(*AC_CODE[r << 4])
            if r:
                self.bw.put(self.eobrun - (1 << r), r)
            self.eobrun = 0
            for b in self.be:
                self.bw.put(b, 1)
            self.be = []

    def first(self, zz):
        r = 0
        for k in range(self.ss, self.se + 1):
            v = int(zz[k])
            if v == 0:
                r += 1
                continue
            t = _irs(v, self.al) if v >= 0 else -_irs(-v, self.al)
            if t == 0:
                r += 1
                continue
            self.emit_eobrun()
            while r > 15:
                self.bw.put(*AC_CODE[0xF0])
                r -= 16
            s, bits = _size(t)
            self.bw.put(*AC_CODE[(r << 4) | s])
            self.bw.put(bits, s)
            r = 0
        if r > 0:
            self.eobrun += 1
            if self.eobrun == self.eob_max:
                self.emit_eobrun()

    def refine(self, zz):
        absv = [abs(int(zz[k])) >> self.al for k in range(64)]
        eob = 0
        for k in range(self.ss, self.se + 1):
            if absv[k] == 1:
                eob = k
        r, br = 0, []
        for k in range(self.ss, self.se + 1):
            t = absv[k]
            if t == 0:
                r += 1
                continue
            while r > 15 and k <= eob:
                self.emit_eobrun()
                self.bw.put(*AC_CODE[0xF0])
                r -= 16
                for b in br:
                    self.bw.put(b, 1)
                br = []
            if t > 1:
                br.append(t & 1)
                continue
            self.emit_eobrun()
            self.bw.put(*AC_CODE[(r << 4) | 1])
            self.bw.put(0 if int(zz[k]) < 0 else 1, 1)
            for b in br:
                self.bw.put(b, 1)
            br, r = [], 0
        if r > 0 or br:
            self.eobrun += 1
            self.be += br
            if self.eobrun == self.eob_max or len(self.be) > 1000 - 63:
                self.emit_eobrun()


def write(comps, h, w, script, samp=None, qts=None, restart=0, scan_restart=None, dqt_before=None, undefined_dc=(),
          dc_ids=None, emit=None, eob_max=0x7FFF, ids=None):
    """A JPEG stream of the quantised blocks comps[c] ([bh_c, bw_c, 64] int, natural order, MCU-padded planes) of an
    h x w frame: sampling samp[c] = (h, v) (default 1 x 1 each), quantisation tables qts[c] (64 values, natural order;
    default all 1).  script: a list of (components, Ss, Se, Ah, Al) scans (a progressive SOF2 stream), or None for one
    sequential scan (SOF0).  restart: the DRI before the first scan; scan_restart {scan: interval} writes a DRI before
    that scan.  dqt_before {scan: [(table id, 64 values)]}: DQT segments before that scan.  undefined_dc: scans whose
    SOS names DC table 3, which no DHT defines (DC refinement scans need none).  emit {scan: f(bits, segment)}: f writes
    each restart segment's entropy data in place of the encoder (bits.put(value, n); a symbol's code: DC_CODE /
    AC_CODE)."""
    nc = len(comps)
    samp = samp or [(1, 1)] * nc
    qts = qts if qts is not None else [np.ones(64, np.int64)] * nc
    ids = ids or list(range(1, nc + 1))
    mx, my, g = _geometry(h, w, samp)
    comps = [np.asarray(c, np.int64) for c in comps]
    for c in range(nc):
        assert comps[c].shape == (g[c]["bh"], g[c]["bw"], 64), (comps[c].shape, g[c])
    out = bytearray(b"\xff\xd8")
    out += _seg(0xE0, b"JFIF\0\x01\x01\0\0\x01\0\x01\0\0")
    for c in range(nc):
        out += _seg(0xDB, bytes([c]) + bytes(int(qts[c][ZZ[k]]) for k in range(64)))
    sof = struct.pack(">BHHB", 8, h, w, nc) + b"".join(bytes([ids[c], (samp[c][0] << 4) | samp[c][1], c])
                                                      for c in range(nc))
    out += _seg(0xC0 if script is None else 0xC2, sof)
    if restart:
        out += _seg(0xDD, struct.pack(">H", restart))
    rst = restart
    scans = [(tuple(range(nc)), 0, 63, 0, 0)] if script is None else script
    for si, (sc, ss, se, ah, al) in enumerate(scans):
        for tid, vals in (dqt_before or {}).get(si, []):
            out += _seg(0xDB, bytes([tid]) + bytes(int(vals[ZZ[k]]) for k in range(64)))
        if scan_restart and si in scan_restart:
            rst = scan_restart[si]
            out += _seg(0xDD, struct.pack(">H", rst))
        refine_dc = ss == 0 and ah > 0
        if not refine_dc:
            out += _seg(0xC4, bytes([0x00]) + DC_SPEC + bytes([0x10]) + AC_SPEC)
        dc_id = 3 if si in undefined_dc else 0
        out += _seg(0xDA, bytes([len(sc)]) + b"".join(bytes([ids[c], dc_id << 4]) for c in sc) +
                    bytes([ss, se, (ah << 4) | al]))
        bw = _Bits()
        units = _units(sc, g, mx, my)
        per = rst if rst else len(units)
        for s0 in range(0, len(units), per):
            if s0:
                out += bytes([0xFF, 0xD0 + (s0 // per - 1) % 8])
            if emit and si in emit:
                emit[si](bw, s0 // per)
                out += bw.flush()
                continue
            pred = [0] * nc
            enc = _AcEncoder(bw, 1, 63, 0, 0) if script is None else _AcEncoder(bw, ss, se, ah, al, eob_max)
            for unit in units[s0:s0 + per]:
                for c, by, bx in unit:
                    blk = comps[c][by, bx]
                    zz = [int(blk[ZZ[k]]) for k in range(64)] + [0] * 16      # Se past 63 in invalid scripts
                    if script is None:            # sequential: DC then AC of the block
                        s, bits = _size(zz[0] - pred[c])
                        pred[c] = zz[0]
                        bw.put(*DC_CODE[s])
                        bw.put(bits, s)
                        enc.first(zz)
                        enc.emit_eobrun()
                    elif ss == 0 and ah == 0:
                        t = _irs(zz[0], al)
                        s, bits = _size(t - pred[c])
                        pred[c] = t
                        bw.put(*DC_CODE[s])
                        bw.put(bits, s)
                    elif ss == 0:
                        bw.put((zz[0] >> al) & 1, 1)
                    elif ah == 0:
                        enc.first(zz)
                    else:
                        enc.refine(zz)
            enc.emit_eobrun()
            out += bw.flush()
    return bytes(out + b"\xff\xd9")


def random_blocks(h, w, samp, seed, amp=60, decay=0.12):
    """Seeded quantised blocks with photo-like spectra (large DC, AC falling off with frequency), MCU-padded."""
    rs = np.random.RandomState(seed)
    _, _, g = _geometry(h, w, samp)
    out = []
    for c in g:
        zz_scale = amp * np.exp(-decay * np.arange(64))
        b = np.zeros((c["bh"], c["bw"], 64), np.int64)
        vals = np.round(rs.laplace(0, 1, (c["bh"], c["bw"], 64)) * zz_scale).astype(np.int64)
        vals[..., 0] = rs.randint(-60, 60) + np.cumsum(rs.randint(-20, 21, (c["bh"], c["bw"])), 1)
        for k in range(64):
            b[..., ZZ[k]] = vals[..., k]
        out.append(b)
    return out


SAMP = {"444": [(1, 1)] * 3, "422": [(2, 1), (1, 1), (1, 1)], "420": [(2, 2), (1, 1), (1, 1)],
        "440": [(1, 2), (1, 1), (1, 1)], "411": [(4, 1), (1, 1), (1, 1)], "gray": [(1, 1)]}
