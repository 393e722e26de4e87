"""CPU: JPEG encoding (DESIGN.md 2.14) - csrc/jpeg_enc_core.h compiled for the host, split the way the kernels run it
(per-block coefficients and code lengths, per-image scan, per-block packing, per-image stuffing), against
cv2.imencode('.jpg', frame, [quality, sampling]) byte for byte: every quality 1 .. 100, all five samplings, sizes from
1 x 1 through every residue of h and w mod 16 to 3000 x 4000, photo-like content, checkerboards, noise, flat and
saturated frames.  Each of seven planted mistakes changes several cases of a compact set."""
import numpy as np
import pytest

import jpeg_enc_check as je

cv2 = pytest.importorskip("cv2")


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    return je.compile_core(str(tmp_path_factory.mktemp("jpeg_enc") / "libjpegenccore.so"))


def _mismatch(lib, img, quality=95, sampling="420"):
    """None when the host core's stream equals cv2.imencode's, else a description."""
    got, want = je.core_encode(lib, img, quality, sampling), je.cv2_encode(img, quality, sampling)
    if got == want:
        return None
    first = next((k for k in range(min(len(got), len(want))) if got[k] != want[k]), min(len(got), len(want)))
    return "%d vs %d bytes, first difference at byte %d" % (len(got), len(want), first)


def test_header_bytes_on_the_ski_image(core):
    from conftest import ROOT
    import os
    img = cv2.imread(os.path.join(ROOT, "readme", "ski.jpg"))
    for s in je.SAMPLING:
        got, want = je.core_encode(core, img, 95, s), je.cv2_encode(img, 95, s)
        assert len(got) > 623 and got[:623] == want[:623], s
        assert got == want, s


def test_every_quality(core):
    img = je.frame(37, 53, 1)
    bad = [(q, s, m) for q in range(1, 101) for s in ("420", "444") for m in [_mismatch(core, img, q, s)] if m]
    assert not bad, bad


@pytest.mark.parametrize("sampling", sorted(je.SAMPLING))
def test_every_residue_mod_16(core, sampling):
    bad = []
    for h in range(1, 17):
        for w in range(1, 17):
            hh, ww = h + 16 * (w % 2), w + 16 * (h % 3)
            m = _mismatch(core, je.frame(hh, ww, h * 17 + w), 90, sampling)
            if m:
                bad.append((hh, ww, m))
    assert not bad, bad


@pytest.mark.parametrize("sampling", sorted(je.SAMPLING))
@pytest.mark.parametrize("kind", ["photo", "checker", "noise", "flat", "saturated"])
def test_contents(core, sampling, kind):
    bad = []
    for h, w in ((1, 1), (8, 8), (23, 41), (480, 640)):
        for q in (1, 50, 75, 95, 100):
            m = _mismatch(core, je.frame(h, w, h + q, kind), q, sampling)
            if m:
                bad.append((h, w, q, m))
    assert not bad, bad


@pytest.mark.parametrize("sampling", ["420", "444"])
def test_3000x4000(core, sampling):
    assert _mismatch(core, je.frame(3000, 4000, 3), 95, sampling) is None


def test_1080p_every_sampling(core):
    img = je.frame(1080, 1920, 4)
    bad = [(s, m) for s in je.SAMPLING for m in [_mismatch(core, img, 90, s)] if m]
    assert not bad, bad


def test_bound_covers_noise_at_quality_100(core):
    for s in je.SAMPLING:
        img = je.frame(64, 80, 2, "noise")
        assert len(je.cv2_encode(img, 100, s)) <= core.core_encode_bound(64, 80, je.SAMPLING[s])


def _planted(tmp_path, name, old, new):
    src = open(je.os.path.join(je.CSRC, "jpeg_enc_core.h")).read()
    assert old in src, name
    path = tmp_path / ("jpeg_enc_core_%s.h" % name)
    path.write_text(src.replace(old, new))
    return je.compile_core(str(tmp_path / ("lib_%s.so" % name)), core=str(path))


def _set():
    """The compact comparison set: every sampling at partial-MCU sizes, three qualities, photo, noise and flat."""
    out = []
    for k, s in enumerate(sorted(je.SAMPLING)):
        for h, w, q, kind in ((33, 47, 75, "photo"), (17, 23, 95, "noise"), (40, 24, 50, "photo"), (9, 30, 90, "flat")):
            out.append(("%s_%dx%d_q%d_%s" % (s, h, w, q, kind), je.frame(h, w, k + h, kind), q, s))
    return out


PLANTS = {
    "no_alternating_bias": ("return (sum + (x & 1)) >> 1;      // h2v1", "return sum >> 1;      // h2v1"),
    "dummy_dc_zero": ("zz[0] = (short)jenc_quant(sum, recip[0], corr[0], shift[0]);", "zz[0] = 0;"),
    "shared_dc_predictor": ("if (b > 0 && im.mcu_comp[b - 1] == c) return g - 1;", "if (g > 0) return g - 1;"),
    "no_stuffing": ("    if (b != 0xFFu) return 1;\n    dst[1] = 0;\n    return 2;", "    return 1;"),
    "zero_bit_padding": ("if (k == (bits - 1) >> 3 && (bits & 7)) b |= 0xFFu >> (bits & 7);", ""),
    "cb_cr_swapped": ("if (c == 1) return (-kJencFixCbR", "if (c == 2) return (-kJencFixCbR"),
    "ifast_constant": ("kFdct0541196100 = 4433", "kFdct0541196100 = (139 << 5)"),
}
# A rounded division in place of jcdctmgr.c's reciprocal is not a mistake any stream can show: the core's reciprocal,
# correction and shift (jenc_reciprocal, read from the header's host build) give a rounded division on every
# coefficient the DCT can produce, for every table value.  The streams above check that they are also cv2's.


def test_reciprocal_equals_rounded_division(core):
    x = np.arange(0, 32768, dtype=np.int64)
    rcs = np.zeros(3, np.uint32)
    for q in range(1, 256):
        core.core_reciprocal(q, rcs.ctypes.data)
        recip, corr, shift = (int(v) for v in rcs)
        d = q << 3
        assert (((x + corr) * recip) >> (shift + 16) == (x + d // 2) // d).all(), q


# cases of the compact set each plant must change at least: enough that a mistake is not caught by one stray case
MIN_CAUGHT = 2


@pytest.mark.parametrize("name", sorted(PLANTS))
def test_planted_mistakes_are_caught(tmp_path, name):
    lib = _planted(tmp_path, name, *PLANTS[name])
    cases = _set()
    caught = [case for case, img, q, s in cases if je.core_encode(lib, img, q, s) != je.cv2_encode(img, q, s)]
    print("%s: %d of %d cases differ" % (name, len(caught), len(cases)))
    assert len(caught) >= MIN_CAUGHT, "planted mistake %s changed only %s" % (name, caught)


def test_the_compact_set_passes_unplanted(core):
    bad = [case for case, img, q, s in _set() if je.core_encode(core, img, q, s) != je.cv2_encode(img, q, s)]
    assert not bad, bad
