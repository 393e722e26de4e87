"""CPU: progressive JPEG decoding (DESIGN.md 2.18) - the progressive path of csrc/jpeg_core.h compiled for the host,
walking an image the way the kernels do, against cv2.imdecode(buf, cv2.IMREAD_COLOR) bit for bit: cv2's own progressive
output at qualities 1 .. 100, every sampling and grayscale, restart intervals 0, 1, 7 and 50, EXIF orientations 1 .. 8,
sizes from 1 x 1 to 3000 x 4000; and streams of tests/jpeg_prog_check.py's writer - spectral selection only, successive
approximation down from Al 13, non-interleaved DC, DC refinement naming undefined tables, a DQT after a component's first
scan, EOB runs up to 32767 and across restart boundaries, a run past Se, refinement sizes other than 1 and DC values
whose << Al wraps.  Incomplete progressions are refused when zig-zag coefficients 0 .. 9 lack bits (cv2 smooths those)
and decoded at 10 and above; invalid progressions are malformed exactly where cv2 returns None; damaged streams report an
error without a read or write outside their buffers (AddressSanitizer).  Each of eight planted mistakes changes the
output of several cases."""
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
import jpeg_check as jc
import jpeg_prog_check as pc

cv2 = pytest.importorskip("cv2")

CORE = os.path.join(ROOT, "pytorch_realtime_multi-person_pose_estimation_b200", "csrc", "jpeg_core.h")
KINDS = list(jc.SAMPLING) + ["gray"]


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    return pc.compile_core(str(tmp_path_factory.mktemp("jpegprog") / "libjpegprog.so"))


def _img(h, w, seed, kind):
    img = jc.content(h, w, seed)
    return jc.gray(img) if kind == "gray" else img


def _cv2(h, w, seed, kind, quality=90, restart=0):
    return pc.cv2_progressive(_img(h, w, seed, kind), quality, "420" if kind == "gray" else kind, restart)


def _blocks(kind, h=37, w=53, seed=3):
    samp = pc.SAMP[kind]
    qts = [np.random.RandomState(c).randint(1, 30, 64) for c in range(len(samp))]
    return pc.random_blocks(h, w, samp, seed), h, w, samp, qts


@pytest.mark.parametrize("kind", KINDS)
def test_cv2_progressive_qualities_and_restarts(core, kind):
    bad = []
    for q in (1, 10, 50, 75, 90, 95, 100):
        for rst in (0, 1, 7, 50):
            m = pc.mismatch(core, _cv2(37, 53, q + rst, kind, q, rst))
            if m:
                bad.append((q, rst, m))
    assert not bad, bad


@pytest.mark.parametrize("orientation", range(1, 9))
def test_cv2_progressive_exif_orientation(core, orientation):
    for kind in ("420", "444", "gray"):
        for rst in (0, 7):
            blob = jc.with_exif(_cv2(21, 38, orientation, kind, 90, rst), orientation, "II", bool(rst))
            assert pc.mismatch(core, blob) is None, (kind, rst)


@pytest.mark.parametrize("h,w", [(1, 1), (1, 17), (8, 8), (15, 17), (33, 47), (368, 368), (427, 640), (1080, 1920)],
                         ids=str)
def test_cv2_progressive_sizes(core, h, w):
    for kind in KINDS:
        assert pc.mismatch(core, _cv2(h, w, h + w, kind, 90)) is None, kind


@pytest.mark.parametrize("kind", ["420", "gray"])
def test_cv2_progressive_3000x4000(core, kind):
    assert pc.mismatch(core, _cv2(3000, 4000, 1, kind, 95)) is None


def _scripts(nc):
    return {"cv2": pc.CV2_SCRIPT_YCC if nc == 3 else pc.CV2_SCRIPT_GRAY, "spectral": pc.spectral_only(nc),
            "successive13": pc.successive(nc, 13), "successive4": pc.successive(nc, 4)}


@pytest.mark.parametrize("kind", list(pc.SAMP))
def test_writer_scripts_equal_the_baseline_stream(core, kind):
    """The writer first: the same blocks as one sequential scan and under complete scan scripts give one cv2 output;
    then the core equals it on every script (non-interleaved DC in the successive scripts), with restarts too."""
    blocks, h, w, samp, qts = _blocks(kind)
    want = cv2.imdecode(np.frombuffer(pc.write(blocks, h, w, None, samp, qts), np.uint8), cv2.IMREAD_COLOR)
    for name, script in _scripts(len(samp)).items():
        for rst in (0, 1, 3):
            blob = pc.write(blocks, h, w, script, samp, qts, restart=rst)
            got = cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR)
            assert got is not None and (got == want).all(), (name, rst)
            assert pc.mismatch(core, blob) is None, (name, rst)


def _crafted():
    """(name, stream) of the writer's crafted cases, all complete progressions of a 2 x 3-block gray frame."""
    h, w = 16, 24
    z = [np.zeros((2, 3, 64), np.int64)]
    blocks = pc.random_blocks(h, w, pc.SAMP["gray"], 9)
    out = []
    ac = pc.AC_CODE

    q8 = [np.full(64, 8)]

    def past_se(ss, r):         # a run of r from Ss lands past Se and stores there (up to jpeg_natural_order's guards)
        def f(bits, seg):
            for k in range(6):
                bits.put(*ac[(r << 4) | 7])
                bits.put(70 + 9 * k, 7)
        return f
    for ss, se, r in ((1, 5, 10), (2, 2, 15)):
        script = [((0,), 0, 0, 0, 0), ((0,), ss, se, 0, 0), ((0,), se + 1, 63, 0, 0)] + \
            ([((0,), 1, ss - 1, 0, 0)] if ss > 1 else [])
        out.append(("run_past_se_%d_%d" % (ss, r), pc.write(z, h, w, script, qts=q8, emit={1: past_se(ss, r)})))

    def size_n(n):              # a refinement symbol of size n != 1: one sign bit is read, the coefficient gets +-1
        def f(bits, seg):
            for k in range(6):
                bits.put(*ac[(k % 3 << 4) | n])
                bits.put(k & 1, 1)
                bits.put(*ac[0x00])
        return f
    for n in (3, 15):
        out.append(("refine_size_%d" % n, pc.write(z, h, w, [((0,), 0, 0, 0, 0), ((0,), 1, 63, 0, 1), ((0,), 1, 63, 1, 0)],
                                                   qts=q8, emit={2: size_n(n)})))

    def dc_wrap(bits, seg):      # DC first at Al 13: predictions 7, 3, -6, ... << 13 wrap in 16 bits
        for d in (7, -4, -9, 12, -3, 5):
            s, v = pc._size(d)
            bits.put(*pc.DC_CODE[s])
            bits.put(v, s)
    script = [((0,), 0, 0, 0, 13)] + [((0,), 0, 0, a + 1, a) for a in range(12, -1, -1)] + [((0,), 1, 63, 0, 0)]
    out.append(("dc_wrap_al13", pc.write(blocks, h, w, script, emit={0: dc_wrap})))

    out.append(("undefined_dc_in_refinement", pc.write(blocks, h, w, pc.successive(1, 3), undefined_dc={4, 6, 8})))
    q2 = np.arange(1, 65)
    out.append(("dqt_after_first_scan", pc.write(blocks, h, w, pc.CV2_SCRIPT_GRAY, qts=[np.full(64, 3)],
                                                 dqt_before={1: [(0, q2)], 4: [(0, q2)]})))
    cblocks, ch, cw, csamp, cqts = _blocks("444")
    out.append(("dqt_after_first_scan_444", pc.write(cblocks, ch, cw, pc.CV2_SCRIPT_YCC, csamp, cqts,
                                                     dqt_before={3: [(1, q2), (2, q2[::-1])]})))
    return out


def _eob_restart_cases():
    """EOB runs at and across restart boundaries: sparse blocks (long runs the encoder ends at each restart), and
    crafted runs longer than their segment, which the restart cuts off."""
    out = []
    h, w = 40, 64
    blocks = pc.random_blocks(h, w, pc.SAMP["gray"], 4, amp=4, decay=0.5)
    for rst in (1, 3, 7):
        out.append(("sparse_rst%d" % rst, pc.write(blocks, h, w, pc.successive(1, 2), restart=rst)))
    out.append(("eob_max_5", pc.write(blocks, h, w, pc.successive(1, 2), eob_max=5)))
    z = [np.zeros((5, 8, 64), np.int64)]
    ac = pc.AC_CODE

    def long_run(bits, seg):
        # 40 blocks, restart interval 10: each segment's first block gets a +-1 at zig-zag 1 + seg, then an EOB run of
        # 16 + seg that the restart cuts off after 9 blocks
        bits.put(*ac[(seg << 4) | 1])
        bits.put(seg & 1 if seg < 3 else 1, 1)
        bits.put(*ac[4 << 4])
        bits.put(seg, 4)
    script = [((0,), 0, 0, 0, 0), ((0,), 1, 63, 0, 1), ((0,), 1, 63, 1, 0)]
    out.append(("eob_across_rst_first", pc.write(z, h, w, script, restart=10, emit={1: long_run})))
    out.append(("eob_across_rst_refine", pc.write(z, h, w, script, restart=10, emit={2: long_run})))
    return out


def test_crafted_streams(core):
    bad = [(name, m) for name, blob in _crafted() for m in [pc.mismatch(core, blob)] if m]
    assert not bad, bad


def test_eob_runs_at_and_across_restarts(core):
    bad = [(name, m) for name, blob in _eob_restart_cases() for m in [pc.mismatch(core, blob)] if m]
    assert not bad, bad


def test_eob_run_of_32767(core):
    """A gray frame of 182 x 182 blocks whose AC band is empty: EOB runs of 32767 (the most one symbol codes) and the
    rest."""
    h = w = 182 * 8
    rs = np.random.RandomState(2)
    b = np.zeros((182, 182, 64), np.int64)
    b[..., 0] = rs.randint(-50, 50, (182, 182))
    b[::97, ::31, 1] = 3
    blob = pc.write([b], h, w, [((0,), 0, 0, 0, 0), ((0,), 1, 63, 0, 0)])
    assert pc.mismatch(core, blob) is None


def _truncated(kind, scans):
    blocks, h, w, samp, qts = _blocks(kind)
    script = _scripts(len(samp))["cv2"]
    return pc.write(blocks, h, w, script[:scans], samp, qts), (blocks, h, w, samp, qts, script[:scans])


def test_incomplete_progressions_refused_at_zigzag_9_and_below(core):
    for kind in ("420", "gray"):
        for scans in range(1, len(_scripts(3 if kind != "gray" else 1)["cv2"])):
            blob, _ = _truncated(kind, scans)
            rc, *_, sup, prog, reason = pc.info(core, blob)
            assert rc == 0 and sup == 0 and "incomplete progression" in reason, (kind, scans, reason)
    # the line is real: cv2 smooths such a stream, so its output differs from the unsmoothed decode of the same bits
    blob, (blocks, h, w, samp, qts, _) = _truncated("gray", 3)          # AC bands at Al 2, no refinement
    known = [np.where(b < 0, -((-b) >> 2 << 2), b >> 2 << 2) for b in blocks]
    for b, src in zip(known, blocks):
        b[..., 0] = src[..., 0] >> 1 << 1
    smooth = cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR)
    plain = cv2.imdecode(np.frombuffer(pc.write(known, h, w, None, samp, qts), np.uint8), cv2.IMREAD_COLOR)
    assert (smooth != plain).any()


def test_incomplete_progressions_decoded_at_zigzag_10_and_above(core):
    for kind in ("420", "444", "gray"):
        blocks, h, w, samp, qts = _blocks(kind)
        nc = len(samp)
        full = [((c,), 0, 0, 0, 0) for c in range(nc)] + [((c,), 1, 9, 0, 0) for c in range(nc)]
        for tail in ([], [((0,), 10, 63, 0, 1)], [((c,), 10, 40, 0, 2) for c in range(nc)]):
            blob = pc.write(blocks, h, w, full + tail, samp, qts)
            rc, *_, sup, prog, reason = pc.info(core, blob)
            assert rc == 0 and sup == 1 and prog == 1, (kind, tail, reason)
            assert pc.mismatch(core, blob) is None, (kind, tail)


def _invalid():
    """(name, script) of scans that are not a valid progression: libjpeg stops (JERR_BAD_PROGRESSION)."""
    dc = [((0,), 0, 0, 0, 0)]
    return [("dc_se_5", [((0,), 0, 5, 0, 0)]), ("ac_ss_gt_se", dc + [((0,), 9, 5, 0, 0)]),
            ("ac_se_64", dc + [((0,), 1, 64, 0, 0)]), ("ac_two_components", [((0, 1, 2), 0, 0, 0, 0), ((1, 2), 1, 63, 0, 0)]),
            ("ah_al_gap", dc + [((0,), 1, 63, 0, 3), ((0,), 1, 63, 3, 1)]), ("al_14", [((0,), 0, 0, 0, 14)])]


def _bogus():
    """(name, script) of bogus progressions: libjpeg warns and decodes."""
    dc = [((0,), 0, 0, 0, 0)]
    return [("ac_before_dc", [((0,), 1, 63, 0, 0), ((0,), 0, 0, 0, 0)]),
            ("ah_not_the_known_bits", dc + [((0,), 1, 63, 0, 2), ((0,), 1, 63, 1, 0)]),
            ("dc_refinement_of_unknown_bits", dc + [((0,), 0, 0, 2, 1)])]


def test_refusals_and_malformed_scans_are_named(core):
    blocks, h, w, samp, qts = _blocks("444")
    for name, script in _invalid():
        blob = pc.write(blocks, h, w, script, samp, qts)
        rc, *_, reason = pc.info(core, blob)
        assert rc == 1 and "not a valid progression" in reason, (name, reason)
        assert cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR) is None, name
    gblocks, gh, gw, gsamp, gqts = _blocks("gray")
    for name, script in _bogus():
        blob = pc.write(gblocks, gh, gw, script, gsamp, gqts)
        rc, *_, sup, prog, reason = pc.info(core, blob)
        assert rc == 0 and sup == 0 and "bogus progression" in reason, (name, reason)
        assert cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR) is not None, name
    # more than 256 scans; off: the old refusal; an AC scan naming an undefined table
    script = [((0,), 0, 0, 0, 13)] + [((0,), 0, 0, a + 1, a) for a in range(12, -1, -1)]
    script += [((0,), k, k, 0, 13) for k in range(1, 64)]
    script += [((0,), k, k, a + 1, a) for a in range(12, 8, -1) for k in range(1, 64)]
    blob = pc.write(gblocks, gh, gw, script[:300], gsamp, gqts)
    rc, *_, sup, prog, reason = pc.info(core, blob)
    assert rc == 0 and sup == 0 and "more than 256 scans" in reason, reason
    blob = _cv2(40, 56, 2, "420")
    rc, *_, sup, prog, reason = pc.info(core, blob, progressive=False)
    assert rc == 0 and sup == 0 and "progressive (SOF2)" in reason
    assert pc.info(core, blob)[5:7] == (1, 1)
    i = blob.index(b"\xff\xda")
    i = blob.index(b"\xff\xda", i + 2)       # the second scan (an AC band) names AC table 3
    n = blob[i + 4]
    bad = bytearray(blob)
    bad[i + 6] = (bad[i + 6] & 0xF0) | 3
    rc, *_, sup, prog, reason = pc.info(core, bytes(bad))
    assert rc == 0 and sup == 0 and "undefined Huffman table" in reason and n == 1, reason


def _damaged():
    rs = np.random.RandomState(11)
    out = []
    for k, (h, w, s, rst) in enumerate([(64, 80, "420", 0), (57, 43, "444", 3), (96, 96, "422", 1), (40, 72, "gray", 0)]):
        blob = _cv2(h, w, k, s, 85, rst)
        b = blob.index(b"\xff\xda")
        e = blob.rindex(b"\xff\xd9")
        for frac in (0.3, 0.7, 0.97):
            out.append(("truncated_%d_%g" % (k, frac), blob[:b + int((e - b) * frac)]))
        for t in range(4):
            arr = bytearray(blob)
            for _ in range(24):
                p = rs.randint(b + 20, e)
                if arr[p] != 0xFF and arr[p - 1] != 0xFF:
                    arr[p] ^= 1 << rs.randint(8)
            out.append(("flipped_%d_%d" % (k, t), bytes(arr)))
    return out


def test_damaged_streams_stay_in_bounds_under_asan(tmp_path):
    exe = pc.compile_core(str(tmp_path / "jpeg_prog_asan"), asan=True)
    cases = _damaged()
    files = []
    for name, blob in cases:
        p = tmp_path / (name + ".jpg")
        p.write_bytes(blob)
        files.append(str(p))
    r = subprocess.run([exe] + files, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    res = [tuple(int(v) for v in line.split()) for line in r.stdout.split("\n") if line]
    assert len(res) == len(cases)
    # a damaged stream is refused (1 malformed, 2 unsupported: e.g. cut between scans) or decodes with status bits
    quiet = [name for (name, blob), (rc, st) in zip(cases, res) if rc == 0 and st == 0 and
             cv2.imdecode(np.frombuffer(blob, np.uint8), cv2.IMREAD_COLOR) is None]
    assert not quiet, "damaged streams decoded without an error where cv2 fails: %s" % quiet
    silent = [name for (name, _), (rc, st) in zip(cases, res) if rc == 0 and st == 0]
    assert not silent, "damaged streams decoded without an error: %s" % silent


PLANTS = {
    "refine_adds_p1_to_negatives": ("*c >= 0 ? *c + p1 : *c + m1", "*c + p1"),
    "eobrun_not_reset_at_restart": ("int pred[3] = {0, 0, 0}, eobrun = 0;", "int pred[3] = {0, 0, 0};\n    static int eobrun = 0;"),
    "eobrun_off_by_one": ("eobrun = (1 << r) + (int)jp_getbits(d, nbytes, &p, r) - 1;",
                          "eobrun = (1 << r) + (int)jp_getbits(d, nbytes, &p, r);"),
    "dc_refinement_ignored": ("if (jp_getbits(d, nbytes, &p, 1)) blk[0] = (short)(blk[0] | (1 << sc.al));",
                              "jp_getbits(d, nbytes, &p, 1);"),
    "noninterleaved_on_mcu_geometry": ("const long long wb = (cp.dw + 7) / 8;", "const long long wb = cp.bw;"),
    "quant_table_of_the_last_dqt": ("if (!T.latched[c]) {", "if (true) {"),
    "run_past_se_clamped": ("                        j += r;\n", "                        j += r;\n                        if (j > sc.se) j = sc.se;\n"),
    "refine_size_not_1_invalid": ("            if (s) {\n                s = jp_getbits(",
                                  "            if (s > 1) return false;\n            if (s) {\n                s = jp_getbits("),
}
MIN_CAUGHT = 2


def _compact_set():
    out = []
    for k, kind in enumerate(KINDS):
        for q, rst in ((50, 0), (90, 7)):
            out.append(("%s_q%d_r%d" % (kind, q, rst), _cv2(37, 53, k, kind, q, rst)))
    for kind in ("420", "gray"):
        blocks, h, w, samp, qts = _blocks(kind)
        out.append(("%s_successive" % kind, pc.write(blocks, h, w, pc.successive(len(samp), 6), samp, qts, restart=2)))
    return out + _crafted() + _eob_restart_cases()


@pytest.mark.parametrize("name", sorted(PLANTS))
def test_planted_mistakes_are_caught(tmp_path, name):
    old, new = PLANTS[name]
    src = open(CORE).read()
    assert old in src, name
    path = tmp_path / ("jpeg_core_%s.h" % name)
    path.write_text(src.replace(old, new))
    lib = pc.compile_core(str(tmp_path / ("lib_%s.so" % name)), core=str(path))
    cases = _compact_set()
    caught = [case for case, blob in cases if pc.mismatch(lib, blob) is not None]
    print("%s: %d of %d cases differ: %s" % (name, len(caught), len(cases), caught))
    assert len(caught) >= MIN_CAUGHT, "planted mistake %s changed only %s" % (name, caught)
