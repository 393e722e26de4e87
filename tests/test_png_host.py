"""CPU: PNG decoding (DESIGN.md 2.17) - csrc/png_core.h compiled for the host, walking an image the way the kernels do,
against cv2.imdecode(buf, cv2.IMREAD_COLOR) bit for bit: every colour type and bit depth, Adam7 at 1 x 1 .. 9 x 9 (empty
passes), every filter forced, mixed and cv2's own adaptive choice, zlib levels 0 .. 9 with every strategy (stored,
fixed and dynamic blocks), window bits 9 .. 15, IDAT splits down to empty chunks, 258-byte matches at distance 32 768,
sizes from 1 x 1 to 3000 x 4000, cv2.imencode at every compression level and strategy, the device encoder's own files,
the colour rules (bit replication, 16-bit strip, palette entries past PLTE, alpha dropped, tRNS and gAMA ignored), eXIf
orientation before and after IDAT, and each stream cv2 refuses.  Malformed streams are refused by name; damage inside
the image data sets the status bit of its kind, without a read or write outside the buffers (AddressSanitizer).  Each
of eight planted mistakes changes the output of several cases."""
import os
import struct
import subprocess
import zlib

import numpy as np
import pytest

from conftest import ROOT
import png_check as pc
import png_enc_check as pec

cv2 = pytest.importorskip("cv2")

CORE = os.path.join(ROOT, "pytorch_realtime_multi-person_pose_estimation_b200", "csrc", "png_core.h")


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    return pc.compile_core(str(tmp_path_factory.mktemp("png") / "libpngcore.so"))


def _mismatch(lib, blob):
    """None when the host core equals cv2.imdecode (a frame), else a description."""
    want = pc.cv2_decode(blob)
    rc, st, got = pc.core_decode(lib, blob)
    if want is None:
        return "cv2 refuses the stream"
    if rc != 0 or st != 0:
        return "rc %d status %d" % (rc, st)
    if got.shape != want.shape:
        return "shape %s vs %s" % (got.shape, want.shape)
    bad = int((got != want).any(-1).sum())
    return "%d pixels differ" % bad if bad else None


def _refused(lib, blob):
    """(host rc, status) for a stream cv2 refuses; the test asserts cv2 does."""
    assert pc.cv2_decode(blob) is None
    rc, st, _ = pc.core_decode(lib, blob)
    return rc, st


def _case(ct, d, h, w, seed=0, kind="noise", **kw):
    s = pc.samples(h, w, ct, d, seed, kind)
    return s, pc.build(s, ct, d, seed=seed, **kw)


@pytest.mark.parametrize("ct,d", pc.PAIRS, ids=lambda v: str(v))
def test_every_type_and_depth(core, ct, d):
    bad = []
    for il in (0, 1):
        for filt in (0, 1, 2, 3, 4, [0, 1, 2, 3, 4], "random"):
            for kind in ("noise", "smooth"):
                s, b = _case(ct, d, 13, 21, ct + d, kind, interlace=il, filters=filt)
                m = _mismatch(core, b)
                if m or not np.array_equal(pc.cv2_decode(b), pc.expected(s, ct, d, seed=ct + d)):
                    bad.append((il, filt, kind, m))
    assert not bad, bad


@pytest.mark.parametrize("ct,d", [(0, 1), (0, 2), (3, 4), (2, 8), (6, 16), (4, 16)], ids=lambda v: str(v))
def test_adam7_small_sizes_with_empty_passes(core, ct, d):
    bad = [(h, w, m) for h in range(1, 10) for w in range(1, 10)
           for m in [_mismatch(core, _case(ct, d, h, w, h * 10 + w, interlace=1, filters="random")[1])] if m]
    assert not bad, bad


def test_colour_rules(core):
    # gray below 8 bits is replicated: 2-bit value 1 is 85
    s = np.array([[[0], [1], [2], [3]]], np.int64)
    assert pc.cv2_decode(pc.build(s, 0, 2))[0, :, 0].tolist() == [0, 85, 170, 255]
    # 16-bit samples keep their high byte
    s = np.array([[[0x00FF], [0xFE80], [0xFFFF]]], np.int64)
    b = pc.build(s, 0, 16)
    assert pc.cv2_decode(b)[0, :, 0].tolist() == [0, 254, 255] and _mismatch(core, b) is None
    # a palette index past PLTE is black; alpha is dropped without compositing
    s = np.array([[[0], [1], [7]]], np.int64)
    b = pc.build(s, 3, 4, plte=[[10, 20, 30], [40, 50, 60]])
    assert pc.cv2_decode(b)[0].tolist() == [[30, 20, 10], [60, 50, 40], [0, 0, 0]] and _mismatch(core, b) is None
    s = np.array([[[10, 20, 30, 0], [40, 50, 60, 128]]], np.int64)
    b = pc.build(s, 6, 8)
    assert pc.cv2_decode(b)[0].tolist() == [[30, 20, 10], [60, 50, 40]] and _mismatch(core, b) is None


def test_chunks_that_change_nothing(core):
    s = pc.samples(12, 17, 2, 8, 4)
    plain = pc.cv2_decode(pc.build(s, 2, 8))
    gama = pc.chunk(b"gAMA", struct.pack(">I", 45455))
    text = pc.chunk(b"tEXt", b"Comment\0hello")
    sbit = pc.chunk(b"sBIT", b"\5\6\5")
    iccp = pc.chunk(b"iCCP", b"p\0\0" + zlib.compress(b"x" * 40))
    bad_anc = pc.chunk(b"tEXt", b"Title\0x", crc=1)
    for extra in ([gama], [text, sbit], [iccp], [bad_anc], [gama, bad_anc]):
        b = pc.build(s, 2, 8, before=extra, after=[text])
        assert _mismatch(core, b) is None and np.array_equal(pc.cv2_decode(b), plain)
    for ct, d, trns in ((2, 8, b"\0\1\0\2\0\3"), (0, 8, b"\0\7"), (3, 8, bytes(range(40)))):
        s = pc.samples(9, 11, ct, d, 5)
        b = pc.build(s, ct, d, trns=trns)
        assert _mismatch(core, b) is None and np.array_equal(pc.cv2_decode(b), pc.cv2_decode(pc.build(s, ct, d)))


@pytest.mark.parametrize("after", [False, True], ids=["before_idat", "after_idat"])
@pytest.mark.parametrize("order", ["II", "MM"])
def test_exif_orientation(core, after, order):
    for o in range(1, 9):
        s, b = _case(2, 8, 2, 3, o, exif=pc.exif_payload(o, order), exif_after=after)
        assert _mismatch(core, b) is None, o
    _, b = _case(2, 8, 2, 3, exif=pc.exif_payload(6, order), exif_after=after)
    assert pc.cv2_decode(b).shape == (3, 2, 3)


@pytest.mark.parametrize("strategy", list(pc.STRATEGIES))
def test_levels_and_strategies(core, strategy):
    bad = []
    for level in range(10):
        for kind in ("noise", "smooth"):
            m = _mismatch(core, _case(2, 8, 40, 57, level, kind, filters="random", level=level, strategy=strategy)[1])
            if m:
                bad.append((level, kind, m))
    assert not bad, bad


def test_window_bits_and_idat_splits(core):
    bad = []
    for wbits in range(9, 16):
        for split in (None, [1], [0, 3], [7, 0, 0, 100], [8192]):
            m = _mismatch(core, _case(0, 8, 60, 90, wbits, "smooth", filters=[0, 2], wbits=wbits, split=split)[1])
            if m:
                bad.append((wbits, split, m))
    assert not bad, bad


def test_long_matches_at_the_window_edge(core):
    # rows of 32 767 bytes + filter byte: each row repeats the one above, a match of 258 at distance 32 768
    rs = np.random.RandomState(3)
    row = rs.randint(0, 256, (1, 32767 // 3 + 1, 3))[:, :32767 // 3]
    s = np.repeat(row, 6, 0).astype(np.int64)
    for strategy in ("default", "filtered"):
        b = pc.build(s, 2, 8, filters=0, level=9, strategy=strategy)
        assert _mismatch(core, b) is None


@pytest.mark.parametrize("h,w", [(1, 1), (1, 2000), (2000, 1), (7, 13), (480, 640), (1080, 1920)], ids=str)
def test_sizes(core, h, w):
    for ct, d in ((2, 8), (0, 1), (6, 16)):
        assert _mismatch(core, _case(ct, d, h, w, h + w, "smooth", filters="random", interlace=(h + w) % 2)[1]) is None


def test_3000x4000(core):
    img = pec.frame(3000, 4000, 1, "drawn")
    assert _mismatch(core, cv2.imencode(".png", img)[1].tobytes()) is None


def test_cv2_encoder_at_every_level_and_strategy(core):
    bad = []
    for level in range(10):
        for strat in (cv2.IMWRITE_PNG_STRATEGY_DEFAULT, cv2.IMWRITE_PNG_STRATEGY_FILTERED,
                      cv2.IMWRITE_PNG_STRATEGY_HUFFMAN_ONLY, cv2.IMWRITE_PNG_STRATEGY_RLE, cv2.IMWRITE_PNG_STRATEGY_FIXED):
            for img in (pec.frame(70, 90, level, "drawn"), cv2.cvtColor(pec.frame(33, 47, level, "photo"), cv2.COLOR_BGR2GRAY)):
                b = cv2.imencode(".png", img, [cv2.IMWRITE_PNG_COMPRESSION, level, cv2.IMWRITE_PNG_STRATEGY, strat])[1]
                m = _mismatch(core, b.tobytes())
                if m:
                    bad.append((level, strat, img.ndim, m))
    assert not bad, bad


def test_round_trip_through_the_device_encoders_core(core, tmp_path):
    enc = pec.compile_core(str(tmp_path / "libpngenc.so"))
    for kind in ("photo", "noise", "flat", "stripes", "norun", "drawn"):
        img = pec.frame(45, 61, 2, kind)
        b = pec.core_encode(enc, img)
        rc, st, got = pc.core_decode(core, b)
        assert rc == 0 and st == 0 and np.array_equal(got, img), kind


def _good():
    return pc.build(pc.samples(20, 30, 2, 8, 1, "smooth"), 2, 8, filters="random", split=[200])


def _damaged_inflate():
    """Damage inside the zlib data, CRCs recomputed: (name, stream, status bit)."""
    z = pc.zlib_of(_good())
    stored = pc.deflate(pc.image_data(pc.samples(4, 5, 2, 8, 1), 2, 8), level=0)
    return [("adler", pc.with_zlib(_good(), z[:-1] + bytes([z[-1] ^ 1])), 4),
            ("too_little_data", pc.build(pc.samples(20, 30, 2, 8, 1), 2, 8,
                                         zdata=zlib.compress(pc.image_data(pc.samples(19, 30, 2, 8, 1), 2, 8))), 2),
            ("cut_stream", pc.with_zlib(_good(), z[:len(z) // 2]), 2),
            ("block_type_3", pc.with_zlib(_good(), z[:2] + bytes([z[2] | 6]) + z[3:]), 1),
            ("stored_nlen", pc.with_zlib(_good(), stored[:5] + bytes([stored[5] ^ 1]) + stored[6:]), 1),
            ("cinfo_8", pc.with_zlib(_good(), bytes([0x88, 0x1D]) + z[2:]), 1),
            ("fcheck", pc.with_zlib(_good(), bytes([z[0], z[1] ^ 1]) + z[2:]), 1),
            ("filter_type_5", pc.build(pc.samples(3, 4, 2, 8, 1), 2, 8,
                                       zdata=zlib.compress(b"\5" + bytes(12) + (b"\0" + bytes(12)) * 2)), 16)]


def test_streams_cv2_refuses(core):
    for name, blob, bit in _damaged_inflate():
        rc, st = _refused(core, blob)
        assert rc == 0 and st == bit, (name, rc, st)
    good = _good()
    assert _refused(core, pc.bad_crc(good, b"IDAT", 1)) == (0, 8)
    for name, blob in _malformed(good):
        rc, st = _refused(core, blob)
        assert rc == 1, name


def test_data_after_the_last_row_is_ignored(core):
    s = pc.samples(10, 12, 2, 8, 2)
    data = pc.image_data(s, 2, 8)
    # more rows than the image has, and bytes behind the zlib stream
    more = pc.build(s, 2, 8, zdata=zlib.compress(data + bytes(200)))
    behind = pc.build(s, 2, 8, zdata=zlib.compress(data) + b"junk")
    # more rows and a bad Adler-32 together: libpng stops at the last row
    z = zlib.compress(data + bytes(200))
    both = pc.build(s, 2, 8, zdata=z[:-1] + bytes([z[-1] ^ 1]))
    for name, b in (("more", more), ("behind", behind), ("more_bad_adler", both)):
        assert _mismatch(core, b) is None, name


def _tail_cases():
    """(name, stream): what comes after the last row, where libpng's outcome depends on the IDAT boundaries."""
    s = pc.samples(10, 12, 2, 8, 2)
    data = pc.image_data(s, 2, 8)
    co = zlib.compressobj()
    never_ends = co.compress(data + bytes(100)) + co.flush(zlib.Z_SYNC_FLUSH)
    z = zlib.compress(data)
    bad_adler = z[:-1] + bytes([z[-1] ^ 1])
    co = zlib.compressobj()
    no_end = co.compress(data) + co.flush(zlib.Z_SYNC_FLUSH)
    # a stored stream whose final block is cut and followed by damaged data
    far = zlib.compress(data, 0)[:-4]
    big = pc.image_data(pc.samples(40, 300, 2, 8, 3), 2, 8)
    return [("extra_rows_stream_never_ends", pc.build(s, 2, 8, zdata=never_ends)),
            ("stream_without_final_block", pc.build(s, 2, 8, zdata=no_end)),
            ("bad_adler_in_own_idat", pc.build(s, 2, 8, zdata=bad_adler, split=[len(bad_adler) - 4, 4])),
            ("bad_adler_split_2", pc.build(s, 2, 8, zdata=bad_adler, split=[len(bad_adler) - 2, 2])),
            ("bad_adler_one_idat", pc.build(s, 2, 8, zdata=bad_adler)),
            ("bad_adler_12_byte_idats", pc.build(s, 2, 8, zdata=bad_adler, split=[12])),
            ("extra_rows_bad_adler", pc.build(s, 2, 8, zdata=(lambda y: y[:-1] + bytes([y[-1] ^ 1]))(
                zlib.compress(data + bytes(50))), split=[7])),
            ("stored_then_damaged_tail", pc.build(s, 2, 8, zdata=far[:-5] + bytes([far[-5] & 0xFE]) + far[-4:] +
                                               bytes([0x03, 0x60, 0xff, 0x1f, 0x00]) + bytes(4))),
            ("bad_adler_8192_pieces", pc.build(pc.samples(40, 300, 2, 8, 3), 2, 8,
                                               zdata=(lambda y: y[:-1] + bytes([y[-1] ^ 1]))(zlib.compress(big, 0)))),
            ("bad_adler_8193_idats", pc.build(pc.samples(40, 300, 2, 8, 3), 2, 8, split=[8193],
                                              zdata=(lambda y: y[:-1] + bytes([y[-1] ^ 1]))(zlib.compress(big, 0))))]


def _agrees(lib, blob):
    """The host core refuses a stream (rc or status) exactly when cv2 does, and otherwise gives cv2's frame."""
    want = pc.cv2_decode(blob)
    rc, st, got = pc.core_decode(lib, blob)
    if want is None:
        return rc != 0 or st != 0
    return rc == 0 and st == 0 and np.array_equal(got, want)


def test_data_after_the_last_row_follows_the_idat_boundaries(core):
    bad = [name for name, blob in _tail_cases() if not _agrees(core, blob)]
    assert not bad, bad
    refused = {name for name, blob in _tail_cases() if pc.cv2_decode(blob) is None}
    # both outcomes occur, so the boundaries decide something
    assert {"extra_rows_stream_never_ends", "bad_adler_one_idat"} <= refused
    assert "bad_adler_in_own_idat" not in refused


@pytest.mark.parametrize("base", range(9))
def test_random_damage_with_random_idat_splits(core, base):
    ct, d = [(2, 8), (0, 8), (6, 16), (3, 4), (0, 1), (2, 16), (4, 8), (2, 8), (0, 2)][base]
    s = pc.samples(20 + base, 30 + 40 * (base == 7) * 8, ct, d, base, "smooth" if base % 2 else "noise")
    z = pc.deflate(pc.image_data(s, ct, d, base % 2, "random", base), level=base)
    rs = np.random.RandomState(base)
    bad = []
    for k in range(300):
        zz = bytearray(z)
        for _ in range(1 + k % 3):
            zz[rs.randint(0, len(zz))] ^= 1 << rs.randint(8)
        split = [int(v) for v in rs.randint(0, 60, 1 + k % 5)] if k % 4 else None
        if split is not None and sum(split) == 0:
            split = [13]
        if not _agrees(core, pc.build(s, ct, d, base % 2, zdata=bytes(zz), split=split, seed=base)):
            bad.append(k)
    assert not bad, bad


def test_plte_in_rgb_images_is_passed_over(core):
    for ct in (2, 6):
        s = pc.samples(6, 7, ct, 8, 1)
        for name, blob in (("length", pc.build(s, ct, 8, before=[pc.chunk(b"PLTE", b"\1\2\3\4")])),
                           ("after_idat", pc.build(s, ct, 8, after=[pc.chunk(b"PLTE", b"\1\2\3")])),
                           ("twice", pc.build(s, ct, 8, plte=[[1, 2, 3]], before=[pc.chunk(b"PLTE", b"\1\2\3")]))):
            assert pc.cv2_decode(blob) is not None and _mismatch(core, blob) is None, (ct, name)


def _malformed(good):
    cs = pc.chunks_of(good)
    rebuild = lambda parts: pc.SIG + b"".join(pc.chunk(t, d) for t, d in parts)
    idats = [c for c in cs if c[0] == b"IDAT"]
    return [("signature", b"\x89PNG\r\n\x1b\n" + good[8:]),
            ("ihdr_crc", pc.bad_crc(good, b"IHDR")),
            ("ihdr_depth", rebuild([(b"IHDR", struct.pack(">IIBBBBB", 30, 20, 3, 2, 0, 0, 0))] + cs[1:])),
            ("ihdr_method", rebuild([(b"IHDR", struct.pack(">IIBBBBB", 30, 20, 8, 2, 1, 0, 0))] + cs[1:])),
            ("ihdr_interlace", rebuild([(b"IHDR", struct.pack(">IIBBBBB", 30, 20, 8, 2, 0, 0, 2))] + cs[1:])),
            ("ihdr_zero_width", rebuild([(b"IHDR", struct.pack(">IIBBBBB", 0, 20, 8, 2, 0, 0, 0))] + cs[1:])),
            ("chunk_past_end", good[:-20]),
            ("no_idat", rebuild([cs[0], cs[-1]])),
            ("no_iend", rebuild(cs[:-1])),
            ("idat_interrupted", rebuild([cs[0], idats[0], (b"tEXt", b"a\0b")] + idats[1:] + [cs[-1]])),
            ("palette_without_plte", rebuild([(b"IHDR", struct.pack(">IIBBBBB", 30, 20, 8, 3, 0, 0, 0))] + cs[1:])),
            ("unknown_critical", rebuild([cs[0], (b"ABCD", b"xyz")] + cs[1:])),
            ("plte_crc", pc.bad_crc(pc.build(pc.samples(4, 4, 3, 8, 0), 3, 8), b"PLTE"))]


def test_refusals_name_the_reason(core):
    for name, blob in _malformed(_good()):
        rc, *_, reason = pc.core_info(core, blob)
        assert rc == 1 and reason, name
    fctl = pc.chunk(b"fcTL", struct.pack(">IIIIIHHBB", 0, 30, 20, 0, 0, 1, 10, 0, 0))
    apng = pc.build(pc.samples(20, 30, 2, 8, 1), 2, 8, before=[pc.chunk(b"acTL", struct.pack(">II", 1, 0)), fctl])
    rc, _, _, oh, ow, sup, reason = pc.core_info(core, apng)
    assert rc == 0 and sup == 0 and "APNG" in reason and (oh, ow) == (20, 30)
    assert pc.cv2_decode(apng).shape == (20, 30, 3)


def test_damaged_streams_stay_in_bounds_under_asan(tmp_path):
    exe = str(tmp_path / "png_asan")
    subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                    "-I", pc.CSRC, "-DPNG_HOST_MAIN", "-o", exe, pc.HOST_SRC], check=True)
    good = _good()
    cases = [(n, b) for n, b, _ in _damaged_inflate()] + _malformed(good)
    rs = np.random.RandomState(5)
    z = pc.zlib_of(good)
    for k in range(24):       # random bytes of the zlib data flipped, CRCs recomputed
        zz = bytearray(z)
        for _ in range(1 + k % 4):
            zz[rs.randint(2, len(zz))] ^= 1 << rs.randint(8)
        cases.append(("flip_%d" % k, pc.with_zlib(good, bytes(zz))))
    cases += [("cut_%d" % k, good[:k]) for k in (0, 7, 8, 20, 40, 60)]
    files = []
    for name, blob in cases:
        p = tmp_path / (name + ".png")
        p.write_bytes(blob)
        files.append(str(p))
    r = subprocess.run([exe] + files, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    res = [tuple(int(v) for v in line.split()) for line in r.stdout.split("\n") if line]
    assert len(res) == len(cases)
    for (name, blob), (rc, st) in zip(cases, res):
        refused = pc.cv2_decode(blob) is None
        assert refused == (rc != 0 or st != 0), (name, rc, st)


def _set():
    """The compact comparison set for the planted mistakes."""
    out = []
    for k, (ct, d) in enumerate(pc.PAIRS):
        s, b = _case(ct, d, 11, 13, k, "smooth" if k % 2 else "noise", interlace=k % 2, filters="random",
                     trns=b"\0\1\0\2\0\3" if ct == 2 else None)
        out.append(("%d_%d" % (ct, d), b))
        out.append(("%d_%d_adam7" % (ct, d), _case(ct, d, 9, 9, k, "noise", interlace=1, filters=[3, 4])[1]))
    for o in (5, 6, 7, 8):
        out.append(("exif%d" % o, _case(2, 8, 4, 7, o, exif=pc.exif_payload(o))[1]))
    for ct in (0, 2):       # samples of a narrow range: many Paeth ties between distinct predictors
        s = np.random.RandomState(ct).randint(0, 8, (9, 14, pc.CHANNELS[ct])).astype(np.int64)
        out.append(("paeth_ties_%d" % ct, pc.build(s, ct, 8, filters=4)))
    out.append(("long_matches", pc.build(np.repeat(pc.samples(1, 4000, 2, 8, 1), 4, 0), 2, 8, level=9)))
    return out


PLANTS = {
    # a tie between a and b decides nothing (it needs a == b, or c between them, which gives pc = 0 < pb): the b / c tie
    "paeth_tie_order": ("if (pb <= pc) return (unsigned)b;", "if (pb < pc) return (unsigned)b;"),
    "average_rounds_up": ("v += (unsigned)((a + b) >> 1);", "v += (unsigned)((a + b + 1) >> 1);"),
    "16bit_scaled": ("if (im.depth == 16) return row[2 * s];", "if (im.depth == 16) return (row[2 * s] * 65535u + row[2 * s + 1] * 257u) / 65535u / 257u + (row[2 * s + 1] > 127 && row[2 * s] < 255);"),
    "subbyte_shifted": ("return im.depth == 1 ? v * 255u : im.depth == 2 ? v * 85u : v * 17u;", "return v << (8 - im.depth);"),
    "adam7_6_7_swapped": ("const int q = pat[sy & 7][sx & 7];", "const int q0 = pat[sy & 7][sx & 7], q = q0 == 5 ? 6 : q0 == 6 ? 5 : q0;"),
    "dist_extra_off_by_one": ("B2P_PN_HD int pn_dist_xbits(int i) { return i < 4 ? 0 : i / 2 - 1; }",
                              "B2P_PN_HD int pn_dist_xbits(int i) { return i < 4 ? 0 : i == 10 ? 5 : i / 2 - 1; }"),
    "alpha_composited": ("        bgr[0] = (unsigned char)pn_sample(im, row, c, 2);",
                         "        if (im.ctype == 6) { const unsigned al = pn_sample(im, row, c, 3); bgr[0] = (unsigned char)(pn_sample(im, row, c, 2) * al / 255); bgr[1] = (unsigned char)(pn_sample(im, row, c, 1) * al / 255); bgr[2] = (unsigned char)(pn_sample(im, row, c, 0) * al / 255); return; }\n        bgr[0] = (unsigned char)pn_sample(im, row, c, 2);"),
    "exif_ignored": ("if (o >= 0) P->orientation = o;", "(void)o;"),
}
# cases of the compact set each plant must change at least: enough that a mistake is not caught by one stray case
MIN_CAUGHT = 2


@pytest.mark.parametrize("name", sorted(PLANTS))
def test_planted_mistakes_are_caught(tmp_path, name):
    old, new = PLANTS[name]
    src = open(CORE).read()
    assert old in src, name
    path = tmp_path / ("png_core_%s.h" % name)
    path.write_text(src.replace(old, new))
    lib = pc.compile_core(str(tmp_path / ("lib_%s.so" % name)), core=str(path))
    cases = _set()
    caught = [case for case, blob in cases if _mismatch(lib, blob) is not None]
    print("%s: %d of %d cases differ" % (name, len(caught), len(cases)))
    assert len(caught) >= MIN_CAUGHT, "planted mistake %s changed only %s" % (name, caught)
