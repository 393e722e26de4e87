"""CPU: JPEG decoding (DESIGN.md 2.13) - csrc/jpeg_core.h compiled for the host, walking an image the way the kernels
do, against cv2.imdecode(buf, cv2.IMREAD_COLOR) bit for bit: every sampling factor and grayscale, qualities 1 .. 100 and
separate luma / chroma quality, restart intervals 0, 1, 7, 50 and 300 with and without optimised tables (segments that
straddle the Huffman kernel's windows), sizes from 1 x 1 to 3000 x 4000, 0 / 255 checkerboards, crafted coefficient
streams whose IDCT sums leave the sample range (the SIMD islow's saturation and 16-bit wraps), and EXIF orientations
1 .. 8 in both byte orders among extra APPn / COM segments and non-Exif APP1 segments.  The parse's sizes match cv2's
shapes and it refuses progressive, arithmetic and CMYK headers by name; damaged streams are reported as errors without
a read or write outside their buffers (AddressSanitizer).  Each of eight planted mistakes changes the output of several
cases."""
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
import jpeg_check as jc

cv2 = pytest.importorskip("cv2")

CORE = os.path.join(ROOT, "pytorch_realtime_multi-person_pose_estimation_b200", "csrc", "jpeg_core.h")
QUALITIES = (1, 10, 50, 75, 90, 95, 100)
SIZES = [(1, 1), (1, 17), (8, 8), (15, 17), (33, 47), (368, 368), (480, 640), (427, 640), (1080, 1920)]
KINDS = list(jc.SAMPLING) + ["gray"]


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    return jc.compile_core(str(tmp_path_factory.mktemp("jpeg") / "libjpegcore.so"))


def _blob(h, w, seed, kind, **kw):
    img = jc.content(h, w, seed, kw.pop("content", "photo"))
    return jc.encode(jc.gray(img) if kind == "gray" else img, sampling="420" if kind == "gray" else kind, **kw)


def _mismatch(lib, blob):
    """None when the host core equals cv2.imdecode, else a description."""
    want = cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR)
    rc, st, got = jc.core_decode(lib, blob)
    if rc != 0 or st != 0:
        return "rc %d status %d" % (rc, st)
    if got.shape != want.shape:
        return "shape %s vs %s" % (got.shape, want.shape)
    bad = int((got != want).any(-1).sum())
    return "%d pixels differ" % bad if bad else None


def _set(kinds=KINDS):
    """The compact comparison set: every kind at three qualities, two restart intervals, optimised tables, a
    checkerboard and two orientations."""
    out = []
    for k, kind in enumerate(kinds):
        for q, rst, opt in ((10, 0, False), (75, 7, True), (100, 1, False)):
            out.append(("%s_q%d_r%d" % (kind, q, rst), _blob(33, 47, k, kind, quality=q, restart=rst, optimize=opt)))
        out.append(("%s_checker" % kind, _blob(24, 40, 3, kind, quality=95, content="checker")))
        out.append(("%s_rst_exif" % kind, jc.with_exif(_blob(40, 24, k, kind, quality=90, restart=1), 5)))
        out.append(("%s_exif7" % kind, jc.with_exif(_blob(40, 24, k, kind, quality=90), 7, "MM")))
    return out + _exif_cases() + jc.idct_range_set()[:16]


@pytest.mark.parametrize("kind", KINDS)
def test_qualities_restarts_and_tables(core, kind):
    bad = []
    for q in QUALITIES:
        for rst in (0, 1, 7):
            for opt in (False, True):
                m = _mismatch(core, _blob(33, 47, q + rst, kind, quality=q, restart=rst, optimize=opt))
                if m:
                    bad.append((q, rst, opt, m))
    assert not bad, bad


@pytest.mark.parametrize("luma,chroma", [(90, 10), (10, 90), (100, 1), (50, 95)])
def test_separate_luma_and_chroma_quality(core, luma, chroma):
    for kind in jc.SAMPLING:
        assert _mismatch(core, _blob(37, 53, 5, kind, luma=luma, chroma=chroma)) is None, kind


@pytest.mark.parametrize("h,w", SIZES, ids=lambda v: str(v))
def test_sizes(core, h, w):
    for kind in KINDS:
        assert _mismatch(core, _blob(h, w, h + w, kind, quality=90)) is None, kind


@pytest.mark.parametrize("kind", ["420", "gray"])
def test_3000x4000(core, kind):
    assert _mismatch(core, _blob(3000, 4000, 1, kind, quality=95)) is None


@pytest.mark.parametrize("kind", KINDS)
def test_restart_segments_across_windows(core, kind):
    for h, w, rst in ((480, 640, 50), (480, 640, 300), (1080, 1920, 7), (1080, 1920, 120)):
        assert _mismatch(core, _blob(h, w, rst, kind, quality=95, restart=rst)) is None, (h, w, rst)


def test_idct_past_the_sample_range(core):
    bad = [(name, m) for name, blob in jc.idct_range_set() for m in [_mismatch(core, blob)] if m]
    assert not bad, bad


@pytest.mark.parametrize("kind", KINDS)
def test_checkerboards(core, kind):
    for q in (50, 95, 100):
        for seed in range(3):
            assert _mismatch(core, _blob(32, 48, seed, kind, quality=q, content="checker")) is None, (q, seed)


@pytest.mark.parametrize("order", ["II", "MM"])
@pytest.mark.parametrize("orientation", range(1, 9))
def test_exif_orientation(core, orientation, order):
    for kind in ("420", "444", "gray"):
        for extra in (False, True):
            blob = jc.with_exif(_blob(21, 38, orientation, kind, quality=90, restart=2 * extra), orientation, order, extra)
            assert _mismatch(core, blob) is None, (kind, extra)


def _exif_cases(kind="420"):
    """APP1 layouts: (name, stream).  cv2 takes the first orientation entry among the APP1 segments that begin
    "Exif\\0\\0", passing over XMP and other APP1 segments, Exif segments without an orientation entry and segments
    whose identifier differs."""
    b = _blob(21, 38, 4, kind, quality=90)
    ex = lambda o, **kw: jc.app1(jc.exif_payload(o, **kw))
    return [("xmp_then_exif6", jc.with_segments(b, [jc.app1(jc.XMP), ex(6)])),
            ("junk_then_exif7", jc.with_segments(b, [jc.app1(b"ABCDEFGHIJKLMNOP"), ex(7, order="MM")])),
            ("exif6_then_xmp", jc.with_segments(b, [ex(6), jc.app1(jc.XMP)])),
            ("exif6_then_exif3", jc.with_segments(b, [ex(6), ex(3)])),
            ("exif3_then_exif6", jc.with_segments(b, [ex(3), ex(6)])),
            ("no_orientation_then_exif5", jc.with_segments(b, [ex(1, tag=0x0110), ex(5)])),
            ("bad_tiff_then_exif8", jc.with_segments(b, [jc.app1(b"Exif\0\0XX\0\0\0\0\0\0"), ex(8)])),
            ("exif9_then_exif6", jc.with_segments(b, [ex(9), ex(6)])),
            ("other_identifier6", jc.with_segments(b, [ex(6, ident=b"Exif\0x")])),
            ("short_app1_then_exif6", jc.with_segments(b, [jc.app1(b"Exif\0\0"), ex(6)])),
            ("exif6_in_app2", jc.with_segments(b, [b"\xff\xe2" + ex(6)[2:]]))]


@pytest.mark.parametrize("kind", ["420", "444", "gray"])
def test_exif_segment_selection(core, kind):
    bad = [(name, m) for name, blob in _exif_cases(kind) for m in [_mismatch(core, blob)] if m]
    assert not bad, bad


def test_info_matches_cv2_shapes(core):
    for name, blob in _set():
        rc, h, w, oh, ow, sup, reason = jc.core_info(core, blob)
        want = cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR).shape
        assert rc == 0 and sup == 1 and (oh, ow, 3) == want, (name, reason)


def test_refusals_name_the_reason(core):
    img = jc.content(40, 56, 2)
    prog = jc.encode(img, 90, "420", progressive=True)
    rc, _, _, oh, ow, sup, reason = jc.core_info(core, prog)
    assert rc == 0 and sup == 0 and "progressive (SOF2)" in reason
    assert (oh, ow) == (40, 56)
    rc, _, _, _, _, sup, reason = jc.core_info(core, jc.set_sof(jc.encode(img, 90, "420"), 0xC9))
    assert rc == 0 and sup == 0 and "arithmetic-coded (SOF9)" in reason
    rc, _, _, _, _, sup, reason = jc.core_info(core, jc.cmyk_header(jc.encode(jc.gray(img), 90)))
    assert rc == 0 and sup == 0 and "CMYK" in reason
    for blob, what in ((b"\x89PNG\r\n", "SOI"), (jc.encode(img)[:60], "malformed header")):
        rc, *_, reason = jc.core_info(core, blob)
        assert rc == 1 and what in reason, reason


def test_damaged_streams_stay_in_bounds_under_asan(tmp_path):
    exe = str(tmp_path / "jpeg_asan")
    subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=address,undefined", "-fno-sanitize-recover=all",
                    "-DJPEG_HOST_MAIN", "-o", exe, jc.HOST_SRC], check=True)
    cases = jc.corrupt_set()
    img = jc.encode(jc.content(40, 56, 2), 90, "420")
    cases += [("header_cut_%d" % k, img[:k]) for k in (3, 20, 100, 200)]
    files = []
    for name, blob in cases:
        p = tmp_path / (name + ".jpg")
        p.write_bytes(blob)
        files.append(str(p))
    r = subprocess.run([exe] + files, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    res = [tuple(int(v) for v in line.split()) for line in r.stdout.split("\n") if line]
    assert len(res) == len(cases)
    quiet = [name for (name, _), (rc, st) in zip(cases, res) if rc == 0 and st == 0]
    assert not quiet, "damaged streams decoded without an error: %s" % quiet


def _planted(tmp_path, name, old, new):
    src = open(CORE).read()
    assert old in src, name
    path = tmp_path / ("jpeg_core_%s.h" % name)
    path.write_text(src.replace(old, new))
    return jc.compile_core(str(tmp_path / ("lib_%s.so" % name)), core=str(path))


PLANTS = {
    "ifast_constant": ("kFix1847759065 = 15137", "kFix1847759065 = (473 << 5)"),
    "box_upsampling": ("const bool fancy_h = fx == 2 && cp.dw > 2;", "const bool fancy_h = false;"),
    "cb_cr_swapped": ("jp_chroma(im, planes, 1, sy, sx), jp_chroma(im, planes, 2, sy, sx)",
                      "jp_chroma(im, planes, 2, sy, sx), jp_chroma(im, planes, 1, sy, sx)"),
    "dc_not_reset_at_rst": ("*head = j == 0 && (im.restart ? m % im.restart == 0 : m == 0);", "*head = j == 0 && m == 0;"),
    "orient_5_7_swapped": ("r[9] = {0, 0, 0, 180, 180, 90, 90, 270, 270}", "r[9] = {0, 0, 0, 180, 180, 270, 90, 90, 270}"),
    "no_pass1_shortcut": ("if (i >= 8 && coef[i]) ac_rows_zero = false;", "ac_rows_zero = false;"),
    "idct_wrap_not_saturate": ("jp_clamp64(jp_descale(o[c], kIdctConst + kIdctPass1 + 3), -128, 127) + 128",
                               "(jp_descale(o[c], kIdctConst + kIdctPass1 + 3) & 255) ^ 128"),
    "first_app1_only": ("if (!exif_found && sl > 6 && !memcmp(s, \"Exif\\0\\0\", 6)) {",
                        "if (!exif_found && sl > 6) {\n                exif_found = true;"),
}
# cases of the compact set each plant must change at least: enough that a mistake is not caught by one stray case
MIN_CAUGHT = 2


@pytest.mark.parametrize("name", sorted(PLANTS))
def test_planted_mistakes_are_caught(tmp_path, name):
    lib = _planted(tmp_path, name, *PLANTS[name])
    cases = _set()
    caught = [case for case, blob in cases if _mismatch(lib, blob) is not None]
    print("%s: %d of %d cases differ" % (name, len(caught), len(cases)))
    assert len(caught) >= MIN_CAUGHT, "planted mistake %s changed only %s" % (name, caught)
