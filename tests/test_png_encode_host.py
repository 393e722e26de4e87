"""CPU: PNG encoding (DESIGN.md 2.15) - csrc/png_enc_core.h compiled for the host, split the way the kernels run it
(per-byte filter and run starts, per-byte symbols from each run's ends, per-block trees, per-image layout, per-group
packing, per-chunk framing), against cv2.imencode('.png', frame) byte for byte: 1 x 1, one row, one column, every
width residue mod 3, the sizes where libpng rewrites the zlib header, run-free frames whose last block is empty,
noise, flat, striped, photo-like and drawn frames, runs of 1 .. 520 bytes at row ends, across rows and at the end of
the data, 1080p, 3000 x 4000, and a frame that drives zlib's code-length limit.  Each of eight planted mistakes
changes several cases of a compact set."""
import os
import zlib

import numpy as np
import pytest

import png_enc_check as pe

cv2 = pytest.importorskip("cv2")

# The zlib cv2 runs on decides the deflate bytes; a machine with another zlib shows up here first.
ZLIB = zlib.ZLIB_RUNTIME_VERSION


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    return pe.compile_core(str(tmp_path_factory.mktemp("png_enc") / "libpngenccore.so"))


def _mismatch(lib, img):
    """None when the host core's file equals cv2.imencode's, else a description."""
    got, want = pe.core_encode(lib, img), pe.cv2_encode(img)
    if got == want:
        return None
    first = next((k for k in range(min(len(got), len(want))) if got[k] != want[k]), min(len(got), len(want)))
    return "%d vs %d bytes, first difference at byte %d (zlib %s)" % (len(got), len(want), first, ZLIB)


def test_records_the_zlib_version():
    print("zlib runtime %s, OpenCV %s" % (ZLIB, cv2.__version__))
    assert ZLIB


@pytest.mark.parametrize("kind", ["photo", "noise", "flat", "norun"])
def test_one_pixel_one_row_one_column(core, kind):
    bad = [(h, w, m) for h, w in ((1, 1), (1, 2), (1, 97), (1, 1500), (2, 1), (97, 1), (1500, 1))
           for m in [_mismatch(core, pe.frame(h, w, h + w, kind))] if m]
    assert not bad, bad


def test_every_width_residue_mod_3(core):
    bad = [(h, w, kind, m) for h in (1, 5, 31) for w in range(2, 14) for kind in ("photo", "noise", "stripes")
           for m in [_mismatch(core, pe.frame(h, w + 3 * h, h * w, kind))] if m]
    assert not bad, bad


# (h, w) -> filtered bytes h (3w + 1) and the zlib header cv2 writes
HEADERS = {(1, 1): (4, "081d"), (40, 49): (5920, "5809"), (60, 80): (14460, "6805"), (129, 42): (16383, "6805"),
           (64, 85): (16384, "6805"), (113, 48): (16385, "7801"), (100, 60): (18100, "7801")}


@pytest.mark.parametrize("hw", sorted(HEADERS))
def test_small_image_zlib_headers(core, hw):
    h, w = hw
    n, hdr = HEADERS[hw]
    assert h * (3 * w + 1) == n
    for kind in ("photo", "noise"):
        img = pe.frame(h, w, n, kind)
        want = pe.cv2_encode(img)
        assert want[41:43].hex() == hdr, (hw, kind, want[41:43].hex())
        assert pe.core_encode(core, img) == want, (hw, kind, _mismatch(core, img))


@pytest.mark.parametrize("hw", [(129, 42), (258, 42)])
def test_run_free_frames_end_in_an_empty_block(core, hw):
    """16 383 and 32 766 literals: the last full block ends the data, and zlib still sends an empty final block."""
    img = pe.frame(*hw, 5, "norun")
    f = np.concatenate([np.ones((hw[0], 1), np.uint8), _filtered(img)], axis=1).reshape(-1)
    assert (f[1:] != f[:-1]).all()
    assert _mismatch(core, img) is None


def _filtered(img):
    """The Sub-filtered R, G, B bytes of each row (filter bytes left out)."""
    raw = img[:, :, ::-1].reshape(img.shape[0], -1).astype(np.int64)
    f = raw.copy()
    f[:, 3:] = (raw[:, 3:] - raw[:, :-3]) % 256
    return f.astype(np.uint8)


@pytest.mark.parametrize("kind", ["photo", "noise", "flat", "stripes", "norun", "drawn"])
def test_contents(core, kind):
    bad = [(h, w, m) for h, w in ((17, 23), (42, 129), (100, 300), (368, 368), (480, 640))
           for m in [_mismatch(core, pe.frame(h, w, h * 7 + w, kind))] if m]
    assert not bad, bad


def _runs_frame(L, seed):
    """A 3 x 200 frame whose filtered data holds a run of L bytes ending at the end of row 0 (the next filter byte
    stops it), one of L bytes of value 1 ending row 1 and going on through row 2's filter byte into row 2, and one of
    L bytes ending the data; the bytes around them are never equal to their neighbours."""
    rs = np.random.RandomState(seed)
    f = np.zeros((3, 600), np.int64)
    for r in range(3):
        prev = 1
        for x in range(600):
            v = int(rs.randint(10, 256))
            while v == prev:
                v = int(rs.randint(10, 256))
            f[r, x] = prev = v
    f[0, 600 - L:] = 7
    f[1, 600 - L:] = 1
    f[2, :L % 5] = 1
    f[2, 600 - L:] = 9
    return pe.unfilter(f, 3, 200)


def test_runs_of_1_to_520_at_row_ends_across_rows_and_at_the_end(core):
    bad = [(L, m) for L in range(1, 521) for m in [_mismatch(core, _runs_frame(L, L))] if m]
    assert not bad, bad


def test_1080p(core):
    for kind in ("photo", "drawn", "noise"):
        assert _mismatch(core, pe.frame(1080, 1920, 4, kind)) is None, kind


def test_3000x4000(core):
    assert _mismatch(core, pe.frame(3000, 4000, 3)) is None


def _fibonacci_frame():
    """18 literal values with counts 1, 1, 3, 5, 9, .. (each the two before plus one, so that no tie breaks the chain)
    in one block, never two equal bytes in a row: the Huffman tree is 17 deep, so gen_bitlen has to cut it to 15."""
    counts = [1, 1]
    while len(counts) < 18:
        counts.append(counts[-1] + counts[-2] + 1)
    counts[-1] += 3000 * 5 - sum(counts)          # fills 5 rows of 1000 pixels
    left = {10 + i: c for i, c in enumerate(counts)}
    seq, prev = [], None
    while left:
        v = max((s for s in left if s != prev), key=lambda s: (left[s], -s))
        seq.append(v)
        prev = v
        left[v] -= 1
        if not left[v]:
            del left[v]
    return pe.unfilter(np.array(seq).reshape(5, 3000), 5, 1000)


def test_code_length_limit(core, tmp_path):
    img = _fibonacci_frame()
    assert _mismatch(core, img) is None
    lib = _planted(tmp_path, "no_length_limit", "if (bits > max_length) {", "if (false) {")
    assert pe.core_encode(lib, img) != pe.cv2_encode(img)


def test_imwrite_writes_what_imencode_gives(tmp_path):
    img = pe.frame(61, 83, 2, "drawn")
    path = str(tmp_path / "frame.png")
    assert cv2.imwrite(path, img)
    assert open(path, "rb").read() == pe.cv2_encode(img)


def test_bound_covers_noise_and_run_free_frames(core):
    for h, w, kind in ((64, 80, "noise"), (1080, 1920, "noise"), (129, 42, "norun"), (300, 200, "norun"), (1, 1, "noise")):
        assert len(pe.cv2_encode(pe.frame(h, w, 2, kind))) <= core.core_encode_bound(h, w), (h, w, kind)


def _planted(tmp_path, name, old, new):
    src = open(os.path.join(pe.CSRC, "png_enc_core.h")).read()
    assert old in src, name
    path = tmp_path / ("png_enc_core_%s.h" % name)
    path.write_text(src.replace(old, new))
    return pe.compile_core(str(tmp_path / ("lib_%s.so" % name)), core=str(path))


def _set():
    """The compact comparison set: the header sizes, run-free frames, noise over several blocks and chunks, photo-like,
    drawn, flat and striped frames."""
    cases = [(40, 49, "photo"), (60, 80, "drawn"), (113, 48, "photo"), (129, 42, "norun"), (258, 42, "norun"),
             (100, 100, "noise"), (64, 85, "noise"), (50, 70, "flat"), (90, 130, "stripes"), (200, 300, "photo"),
             (120, 160, "drawn")]
    return [("%s_%dx%d" % (kind, h, w), pe.frame(h, w, h + w, kind)) for h, w, kind in cases]


PLANTS = {
    "up_filter": ("    if (col == 0) return w == 1 ? 0u : 1u;\n    const long long x = col - 1;\n"
                  "    const unsigned v = png_raw(frame, w, row, x);\n"
                  "    return x < 3 ? v : (v - png_raw(frame, w, row, x - 3)) & 255u;",
                  "    if (col == 0) return w == 1 ? 0u : 2u;\n    const long long x = col - 1;\n"
                  "    const unsigned v = png_raw(frame, w, row, x);\n"
                  "    return row == 0 ? v : (v - png_raw(frame, w, row - 1, x)) & 255u;"),
    "no_bgr_swap": ("return frame[(row * w + x / 3) * 3 + 2 - x % 3];", "return frame[(row * w + x / 3) * 3 + x % 3];"),
    "flush_at_16384": ("kPngBlockSymbols = 16383;", "kPngBlockSymbols = 16384;"),
    "no_empty_final_block": ("return symbols / kPngBlockSymbols + 1;",
                             "return (symbols + kPngBlockSymbols - 1) / kPngBlockSymbols;"),
    "no_forced_second_distance_code": ("while (hp.heap_len < 2) {", "while (hp.heap_len < 2 - (kind == 1 && max_code >= 0)) {"),
    "depth_tie_break_reversed": ("hp.depth[n] <= hp.depth[m]", "hp.depth[n] >= hp.depth[m]"),
    "no_header_rewrite": ("    if (n <= 16384) {\n        cinfo = 0;", "    if (false) {\n        cinfo = 0;"),
    "idat_4096": ("kPngChunk = 8192;", "kPngChunk = 4096;"),
}

# cases of the compact set each plant must change at least: enough that a mistake is not caught by one stray case
MIN_CAUGHT = 2


@pytest.mark.parametrize("name", sorted(PLANTS))
def test_planted_mistakes_are_caught(tmp_path, name):
    lib = _planted(tmp_path, name, *PLANTS[name])
    cases = _set()
    caught = [case for case, img in cases if pe.core_encode(lib, img) != pe.cv2_encode(img)]
    print("%s: %d of %d cases differ" % (name, len(caught), len(cases)))
    assert len(caught) >= MIN_CAUGHT, "planted mistake %s changed only %s" % (name, caught)


def test_the_compact_set_passes_unplanted(core):
    bad = [case for case, img in _set() if pe.core_encode(core, img) != pe.cv2_encode(img)]
    assert not bad, bad
