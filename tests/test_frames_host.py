"""CPU: video-frame ingestion (DESIGN.md 2.10) - csrc/frame_core.h compiled for the host against OpenCV:
cv2.cvtColor(COLOR_YUV2BGR_NV12 / _I420) on every (Y, U, V) triple, cv2.rotate in all four orientations (with and
without the flip mirror, pitched planes with garbage in their padding), and conversion + rotation + crop_with_factor
against cv2.resize.  The comparison is shown to catch three planted mistakes in the core."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT

cv2 = pytest.importorskip("cv2")

CORE = os.path.join(ROOT, "pytorch_realtime_multi-person_pose_estimation_b200", "csrc", "frame_core.h")
FORMATS = {"bgr": 0, "nv12": 1, "i420": 2}
CV_ROTATE = {0: None, 90: cv2.ROTATE_90_CLOCKWISE, 180: cv2.ROTATE_180, 270: cv2.ROTATE_90_COUNTERCLOCKWISE}


def _compile(so, core=None):
    cmd = ["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-o", so,
           os.path.join(ROOT, "tests", "cuda", "frame_core_host.cpp")]
    if core:
        cmd.insert(1, '-DFRAME_CORE="%s"' % core)
    subprocess.run(cmd, check=True)
    lib = ctypes.CDLL(so)
    lib.core_convert_frame.argtypes = [ctypes.c_void_p] * 2 + [ctypes.c_int] * 5 + [ctypes.c_void_p]
    lib.core_convert_crop.argtypes = [ctypes.c_void_p] * 2 + [ctypes.c_int] * 6 + [ctypes.c_void_p]
    return lib


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    return _compile(str(tmp_path_factory.mktemp("frames") / "libframecore.so"))


def _padded(plane, extra, rs):
    """plane stored with `extra` garbage bytes after every row and a garbage row below it: (buffer, pitch)."""
    h, row = plane.shape[0], plane.shape[1] * (plane.shape[2] if plane.ndim == 3 else 1)
    buf = rs.randint(0, 256, (h + 1, row + extra)).astype(np.uint8)
    buf[:h, :row] = plane.reshape(h, row)
    return buf, row + extra


def _planes(bgr, fmt):
    """A seeded BGR frame as the planes of `fmt` (what a decoder would hand out) and the packed cv2 array."""
    h, w = bgr.shape[:2]
    if fmt == "bgr":
        return [bgr], bgr
    i420 = cv2.cvtColor(bgr, cv2.COLOR_BGR2YUV_I420)
    y, flat, q = i420[:h], i420.reshape(-1), (h // 2) * (w // 2)
    u = flat[h * w:h * w + q].reshape(h // 2, w // 2)
    v = flat[h * w + q:].reshape(h // 2, w // 2)
    if fmt == "i420":
        return [y, u, v], i420
    uv = np.stack([u, v], -1).reshape(h // 2, w)
    return [y, uv], np.concatenate([y, uv])


def _to_bgr(packed, fmt):
    code = {"nv12": cv2.COLOR_YUV2BGR_NV12, "i420": cv2.COLOR_YUV2BGR_I420}
    return packed if fmt == "bgr" else cv2.cvtColor(packed, code[fmt])


def _convert(lib, planes, pitches, h, w, fmt, rot, mirror=False):
    ptrs = (ctypes.c_void_p * 3)(*([p.ctypes.data for p in planes] + [None] * (3 - len(planes))))
    pit = (ctypes.c_int * 3)(*(list(pitches) + [0] * (3 - len(pitches))))
    oh, ow = (w, h) if rot in (90, 270) else (h, w)
    out = np.empty((oh, ow, 3), np.uint8)
    lib.core_convert_frame(ptrs, pit, h, w, FORMATS[fmt], rot, int(mirror), out.ctypes.data)
    return out


def _convert_packed(lib, planes, h, w, fmt, rot, mirror=False):
    planes = [np.ascontiguousarray(p) for p in planes]
    return _convert(lib, planes, [p.strides[0] for p in planes], h, w, fmt, rot, mirror)


def _every_triple(fmt):
    """8192 x 8192 frame: 2x2 block k has Y = k // 65536 in all four luma samples and (U, V) = divmod(k % 65536, 256),
    so the 2^24 blocks carry every (Y, U, V) triple once.  Returns planes and the packed cv2 array."""
    n = 4096
    k = np.arange(n * n, dtype=np.int64)
    yb = (k // 65536).astype(np.uint8).reshape(n, n)
    ub = ((k % 65536) // 256).astype(np.uint8).reshape(n, n)
    vb = (k % 256).astype(np.uint8).reshape(n, n)
    y = np.repeat(np.repeat(yb, 2, 0), 2, 1)
    if fmt == "nv12":
        uv = np.stack([ub, vb], -1).reshape(n, 2 * n)
        return [y, uv], np.concatenate([y, uv])
    return [y, ub, vb], np.concatenate([y, ub.reshape(n // 2, 2 * n), vb.reshape(n // 2, 2 * n)])


@pytest.mark.parametrize("fmt", ["nv12", "i420"])
def test_conversion_equals_cvtcolor_on_every_yuv_triple(core, fmt):
    planes, packed = _every_triple(fmt)
    got = _convert_packed(core, planes, 8192, 8192, fmt, 0)
    want = _to_bgr(packed, fmt)
    bad = int((got != want).any(-1).sum())
    assert bad == 0, "%d of %d pixels differ from cv2.cvtColor" % (bad, 8192 * 8192)


SHAPES = [(6, 6), (8, 14), (14, 8), (30, 52), (52, 30)]


@pytest.mark.parametrize("fmt", ["bgr", "nv12", "i420"])
@pytest.mark.parametrize("rot", [0, 90, 180, 270])
def test_rotation_and_mirror_equal_cv2_rotate_on_pitched_planes(core, fmt, rot):
    rs = np.random.RandomState(rot + 7 * FORMATS[fmt])
    for h, w in SHAPES:
        planes, packed = _planes(rs.randint(0, 256, (h, w, 3)).astype(np.uint8), fmt)
        want = _to_bgr(packed, fmt)
        if CV_ROTATE[rot] is not None:
            want = cv2.rotate(want, CV_ROTATE[rot])
        assert np.array_equal(_convert_packed(core, planes, h, w, fmt, rot), want), (h, w)
        pitched = [_padded(p, 1 + 5 * k, rs) for k, p in enumerate(planes)]
        bufs, pitches = [b for b, _ in pitched], [p for _, p in pitched]
        assert np.array_equal(_convert(core, bufs, pitches, h, w, fmt, rot), want), ("pitched", h, w)
        assert np.array_equal(_convert(core, bufs, pitches, h, w, fmt, rot, mirror=True), want[:, ::-1]), ("mirror", h, w)


def _crop_reference(bgr, dest, factor):
    """crop_with_factor's arithmetic (lib/network/im_transform.py:113-134) with cv2: resize, zero padding."""
    h, w = bgr.shape[:2]
    scale = dest / min(h, w)
    res = cv2.resize(bgr, None, fx=scale, fy=scale)
    ph, pw = -(-res.shape[0] // factor) * factor, -(-res.shape[1] // factor) * factor
    out = np.zeros((ph, pw, 3), np.uint8)
    out[:res.shape[0], :res.shape[1]] = res
    return out


@pytest.mark.parametrize("fmt", ["nv12", "i420"])
def test_conversion_rotation_crop_equals_cv2_resize(core, fmt):
    """(h, w, dest): (240, 320, 120) is an exact 2x reduction, which cv::resize switches to INTER_AREA."""
    rs = np.random.RandomState(5 + FORMATS[fmt])
    for (h, w, dest) in [(240, 320, 120), (180, 242, 368), (96, 160, 64)]:
        planes, packed = _planes(rs.randint(0, 256, (h, w, 3)).astype(np.uint8), fmt)
        for rot in (0, 90, 180, 270):
            bgr = _to_bgr(packed, fmt)
            if CV_ROTATE[rot] is not None:
                bgr = cv2.rotate(bgr, CV_ROTATE[rot])
            want = _crop_reference(bgr, dest, 8)
            got = np.empty_like(want)
            planes_c = [np.ascontiguousarray(p) for p in planes]
            ptrs = (ctypes.c_void_p * 3)(*([p.ctypes.data for p in planes_c] + [None] * (3 - len(planes_c))))
            pit = (ctypes.c_int * 3)(*([p.strides[0] for p in planes_c] + [0] * (3 - len(planes_c))))
            core.core_convert_crop(ptrs, pit, h, w, FORMATS[fmt], rot, dest, 8, got.ctypes.data)
            assert np.array_equal(got, want), (h, w, dest, rot)


# Each mistake as a textual edit of the core: (name, [(old, new), ...]).  The edits must apply.
MISTAKES = [
    ("u_v_swapped", [("U = uv[0];\n        V = uv[1];", "U = uv[1];\n        V = uv[0];"),
                     ("U = f.plane[1][", "U = f.plane[2]["), ("V = f.plane[2][", "V = f.plane[1][")]),
    ("chroma_row_rounded_up", [("const int cy = sy >> 1", "const int cy = (sy + 1) >> 1")]),
    ("rotation_direction_swapped", [("case 90: *sy = h - 1 - x; *sx = y;", "case 90: *sy = x; *sx = w - 1 - y;"),
                                    ("case 270: *sy = x; *sx = w - 1 - y;", "case 270: *sy = h - 1 - x; *sx = y;")]),
]


@pytest.mark.parametrize("name,edits", MISTAKES, ids=[m[0] for m in MISTAKES])
def test_comparison_catches_planted_mistakes(tmp_path, name, edits):
    text = open(CORE).read()
    for old, new in edits:
        assert text.count(old) == 1, old
        text = text.replace(old, new)
    bad_core = tmp_path / "frame_core.h"
    bad_core.write_text(text)
    lib = _compile(str(tmp_path / "libbad.so"), str(bad_core))
    rs = np.random.RandomState(1)
    caught = set()
    for fmt in ("nv12", "i420"):
        h, w = 30, 52
        planes, packed = _planes(rs.randint(0, 256, (h, w, 3)).astype(np.uint8), fmt)
        # a garbage row below every plane: the planted chroma-row mistake reads one row past the last
        padded = [_padded(p, 0, rs) for p in planes]
        for rot in (0, 90, 270):
            want = _to_bgr(packed, fmt)
            if CV_ROTATE[rot] is not None:
                want = cv2.rotate(want, CV_ROTATE[rot])
            got = _convert(lib, [b for b, _ in padded], [p for _, p in padded], h, w, fmt, rot)
            if not np.array_equal(got, want):
                caught.add((fmt, rot))
    if name == "rotation_direction_swapped":
        assert {r for _, r in caught} == {90, 270}, caught
    else:
        assert {f for f, _ in caught} == {"nv12", "i420"}, caught


def test_frame_entry_points_are_declared_exported_and_bound(built):
    from conftest import pkg_module
    nat = pkg_module("_native")
    for name in ("b200pose_net_convert_frames", "b200pose_infer_frames"):
        assert name in nat.EXPORTED
        assert getattr(nat.lib(), name).argtypes is not None
    assert [nat.rotation_of(c) for c in (None, cv2.ROTATE_90_CLOCKWISE, cv2.ROTATE_180,
                                          cv2.ROTATE_90_COUNTERCLOCKWISE)] == [0, 90, 180, 270]


def test_frame_table_takes_pitches_from_strides_and_checks_plane_shapes(built):
    from conftest import pkg_module
    eng, nat = pkg_module("engine"), pkg_module("_native")
    surface = np.zeros((120 + 60, 256), np.uint8)         # a decoder surface: rows padded to 256 bytes
    y, uv = surface[:120, :160], surface[120:, :160]
    table, _, on_dev, sizes = eng.frame_table([(y, uv), (y, uv.reshape(60, 80, 2))], "nv12")
    assert sizes == [(120, 160)] * 2 and not on_dev
    assert [table[0].pitch[k] for k in range(2)] == [256, 256]
    assert table[0].plane[0] == y.ctypes.data and table[0].plane[1] == uv.ctypes.data      # read in place
    i420 = np.zeros((180, 160), np.uint8)
    table, _, _, _ = eng.frame_table([i420], "i420")
    assert [table[0].pitch[k] for k in range(3)] == [160, 80, 80]
    assert table[0].plane[1] - table[0].plane[0] == 120 * 160 and table[0].plane[2] - table[0].plane[1] == 60 * 80
    for bad, fmt in (((y, uv[:, :80]), "nv12"), ((y, uv, uv), "nv12"), (np.zeros((121, 160), np.uint8), "i420"),
                     (np.zeros((120, 160, 4), np.uint8), "bgr")):
        with pytest.raises(nat.B200PoseError):
            eng.frame_table([bad], fmt)
    with pytest.raises(nat.B200PoseError):
        eng.frame_table([i420], "yuyv")
