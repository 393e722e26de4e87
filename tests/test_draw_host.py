"""CPU: drawing of detected persons (DESIGN.md 2.12) - csrc/draw_core.h compiled for the host against OpenCV:
cv2.circle(r 3, thickness 3) at every centre of a range crossing every border of small frames, cv2.line(thickness 3)
between every pair of endpoints of a grid straddling a 10x10 frame, long lines far outside a 1080p frame, degenerate
lines, and the whole composition against the package's draw_humans(frame, humans_from_rows(rows, net_w, net_h)).
The comparison is shown to catch four planted mistakes."""
import os

import numpy as np
import pytest

from conftest import ROOT, pkg_module
import draw_check as dc

cv2 = pytest.importorskip("cv2")

CORE = os.path.join(ROOT, "pytorch_realtime_multi-person_pose_estimation_b200", "csrc", "draw_core.h")
COL = (255, 85, 0)
# (frame h, w, net h, w, persons, spread): crowds on frames smaller and larger than the network input
COMPOSITIONS = [(1080, 1920, 368, 656, 8, None), (1080, 1920, 368, 656, 30, None), (200, 150, 368, 280, 6, None),
                (480, 640, 368, 496, 5, 400), (736, 736, 368, 368, 12, None), (368, 368, 368, 368, 6, None),
                (9, 13, 368, 528, 4, None)]


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    return dc.compile_core(str(tmp_path_factory.mktemp("draw") / "libdrawcore.so"))


def _circle(lib, h, w, cx, cy):
    img = np.zeros((h, w, 3), np.uint8)
    lib.core_circle(img.ctypes.data, h, w, cx, cy, np.array(COL, np.uint8).ctypes.data)
    return img


def _line(lib, h, w, p, q):
    img = np.zeros((h, w, 3), np.uint8)
    lib.core_line(img.ctypes.data, h, w, p[0], p[1], q[0], q[1], np.array(COL, np.uint8).ctypes.data)
    return img


def _cv_circle(h, w, c):
    img = np.zeros((h, w, 3), np.uint8)
    cv2.circle(img, c, 3, COL, thickness=3, lineType=8, shift=0)
    return img


def _cv_line(h, w, p, q):
    img = np.zeros((h, w, 3), np.uint8)
    cv2.line(img, p, q, COL, 3)
    return img


@pytest.mark.parametrize("h,w", [(1, 1), (5, 7), (12, 12)])
def test_circles_at_every_centre_across_the_borders(core, h, w):
    for cy in range(-9, h + 9):
        for cx in range(-9, w + 9):
            np.testing.assert_array_equal(_circle(core, h, w, cx, cy), _cv_circle(h, w, (cx, cy)), err_msg=str((cx, cy)))


def test_lines_between_every_pair_of_a_grid_straddling_the_frame(core):
    grid = [(x, y) for y in range(-3, 13) for x in range(-3, 13)]
    bad = [(p, q) for p in grid for q in grid if not np.array_equal(_line(core, 10, 10, p, q), _cv_line(10, 10, p, q))]
    assert not bad, "%d of %d lines differ, e.g. %s" % (len(bad), len(grid) ** 2, bad[:3])


def test_long_lines_far_outside_a_1080p_frame(core):
    rs = np.random.RandomState(5)
    for _ in range(40):
        p, q = [tuple(int(v) for v in rs.randint(-5000, 7000, 2)) for _ in range(2)]
        np.testing.assert_array_equal(_line(core, 1080, 1920, p, q), _cv_line(1080, 1920, p, q), err_msg=str((p, q)))


@pytest.mark.parametrize("p,q", [((5, 5), (5, 5)), ((0, 0), (0, 0)), ((-2, 3), (-2, 3)), ((3, 9), (90, 9)),
                                 ((7, -4), (7, 60)), ((2, 2), (40, 40)), ((40, 2), (2, 40)), ((-30, 10), (80, 10))])
def test_zero_length_horizontal_vertical_and_diagonal_lines(core, p, q):
    np.testing.assert_array_equal(_line(core, 32, 48, p, q), _cv_line(32, 48, p, q))


def _draw_humans(frame, rows, net_h, net_w):
    common, p2p = pkg_module("lib.utils.common"), pkg_module("lib.utils.paf_to_pose")
    return common.draw_humans(frame, p2p.humans_from_rows(rows, net_w, net_h))


def _composition_mismatch(lib, case, seed):
    h, w, nh, nw, persons, spread = case
    rows = dc.person_rows(persons, seed, nh, nw, spread=spread)
    base = np.random.RandomState(seed).randint(0, 256, (h, w, 3)).astype(np.uint8)
    want = _draw_humans(base.copy(), rows, nh, nw)
    got = dc.core_draw(lib, base.copy(), rows, nh, nw)
    return int((got != want).any(-1).sum()), rows


@pytest.mark.parametrize("case", COMPOSITIONS, ids=lambda c: "%dx%d_net%dx%d_p%d" % c[:5])
def test_composition_equals_draw_humans(core, case):
    diff, rows = _composition_mismatch(core, case, 3)
    assert diff == 0, "%d pixels differ" % diff


def test_crowds_overlap(core):
    h, w, nh, nw, persons, _ = COMPOSITIONS[1]
    rows = dc.person_rows(persons, 3, nh, nw)
    n = dc.overlap_pixels((h, w), rows, nh, nw, core)
    print("pixels covered by primitives of different colours: %d" % n)
    assert n > 0


def _planted(tmp_path, name, old, new):
    src = open(CORE).read()
    assert old in src, name
    path = tmp_path / ("draw_core_%s.h" % name)
    path.write_text(src.replace(old, new))
    return dc.compile_core(str(tmp_path / ("lib_%s.so" % name)), core=str(path))


def test_planted_mistakes_are_caught(tmp_path):
    plants = {
        "radius2": _planted(tmp_path, "radius2", "constexpr int kDrawCircleR = 3;", "constexpr int kDrawCircleR = 2;"),
        "limbs_first": _planted(tmp_path, "limbs_first", "    if (slot < kDrawParts) {",
                                "    slot = (slot + kDrawParts) % kDrawPrimsPerPerson;\n    if (slot < kDrawParts) {"),
        "half_even": _planted(tmp_path, "half_even",
                              "return (int)dr_add(dr_mul(dr_div((double)v, (double)net), (double)size), 0.5);",
                              "return (int)dr_round(dr_mul(dr_div((double)v, (double)net), (double)size));"),
        "reversed": dc.compile_core(str(tmp_path / "lib_reversed.so"), reverse_persons=True),
    }
    for name, lib in plants.items():
        diff = sum(_composition_mismatch(lib, case, 3)[0] for case in COMPOSITIONS)
        assert diff > 0, "planted mistake %s went unnoticed" % name
