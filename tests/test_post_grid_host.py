"""CPU: the scenarios of tests/test_gpu_post_grid.py do what they claim about limb_score_kernel's work queue (computed
from the oracle's peak counts and the item rule: ceil(na nb / 2048) items per (image, limb) in (image, limb) order,
grabbed four at a time), the oracle's connection getters agree with each other, and the grid hook is declared and
bound."""
import os
import re

import numpy as np
import pytest

import post_grid_check as pgc
import post_params_check as ppc
from conftest import ROOT, pkg_module
from oracle import pafprocess_oracle, post_params

SCENARIOS = pgc.scenarios()


def _items(name):
    return pgc.work_items([pgc.part_counts(h) for h, _ in SCENARIOS[name][0]])


@pytest.mark.parametrize("tag", ["46x46_l0", "46x46_l1", "97x127_l0", "97x127_l1"])
def test_same_limb_batch_puts_li0_and_li19_in_one_group(tag):
    """Only limb 0 has pairs, in both images: li 0 is followed directly by li 19 in the item order, both in the first
    group, and the two images' limb-0 PAF planes differ (a plane cache keyed by limb alone would score image 1 against
    image 0's field)."""
    images = SCENARIOS["samelimb" + tag][0]
    items = _items("samelimb" + tag)
    assert {l for _, l in items} == {0}
    li = [img * 19 + l for img, l in items]
    k = li.index(19)
    assert li[k - 1] == 0 and li[:k] == [0] * k and k % pgc.GROUP != 0
    assert (0, 0) in pgc.groups(items)[0] and (1, 0) in pgc.groups(items)[0]
    cx, cy = pgc.LIMB_PAF_CH[0]
    for ch in (cx, cy):
        assert not np.array_equal(images[0][1][:, :, ch], images[1][1][:, :, ch])


@pytest.mark.parametrize("tag", ["46x46_l0", "46x46_l1", "97x127_l0", "97x127_l1"])
def test_crossing_batch_has_groups_across_limbs_and_images(tag):
    items = _items("crossing" + tag)
    per = {}
    for it in items:
        per[it] = per.get(it, 0) + 1
    assert len(per) >= 6 and all(c % pgc.GROUP for c in per.values()), per
    gs = pgc.groups(items)
    assert any(len({img for img, _ in g}) > 1 for g in gs)
    assert any(len({(img, l) for img, l in g}) > 1 and len({img for img, _ in g}) == 1 for g in gs)


def test_noise_batch_outnumbers_the_largest_score_grid():
    """More groups than 12 x 132 blocks (the largest score grid on a 132-SM H100): every block loops."""
    for h, _ in SCENARIOS["noise46"][0]:
        assert len(ppc.joint_list(h)) > 7000
    assert len(pgc.groups(_items("noise46"))) > 12 * pgc.H100_SMS


def test_scenario_layouts_and_sizes():
    """Both layouts at 46x46 (PAF planes staged in shared memory) and at 97x127 (read from global memory)."""
    for kind in ("samelimb", "crossing"):
        for h, w in ((46, 46), (97, 127)):
            for layout in (0, 1):
                images, lay, _ = SCENARIOS["%s%dx%d_l%d" % (kind, h, w, layout)]
                assert lay == layout and all(im[0].shape[:2] == (h, w) for im in images)
    assert 2 * 46 * 46 * 4 <= 96 * 1024 < 2 * 97 * 127 * 4
    assert SCENARIOS["loose46"][2] in post_params.SETS and SCENARIOS["loose46"][2] != "default"


def test_port_connection_getters():
    """The port's per-limb connections equal what the parameterised port records at the reference's constants, each
    peak is used once per limb and the scores do not increase (the greedy loop walks the sorted candidates)."""
    port, pport = pafprocess_oracle.load_port(), post_params.load_port("default")
    total = 0
    for name in ("golden46", "crossing46x46_l1", "edges23x31"):
        for heat, paf in SCENARIOS[name][0]:
            jl = ppc.joint_list(heat)
            rows = ppc.oracle_rows(port, jl, paf, *heat.shape[:2])
            assert ppc.same_bits(ppc.oracle_rows(pport, jl, paf, *heat.shape[:2]), rows)
            for l in range(19):
                a, b, s = pport.connections(l)
                ga, gb, gs = port.connections(l)
                assert np.array_equal(ga, a) and np.array_equal(gb, b) and ppc.same_bits(gs, s)
                assert len(set(a)) == len(a) and len(set(b)) == len(b) and np.all(np.diff(s) <= 0)
                total += len(a)
    assert total > 500


def test_sort_inputs_are_the_device_sort_tests():
    sizes = [len(k) for k in pgc.sort_inputs()]
    assert len(sizes) == 162 and max(sizes) == 300000


def test_grid_hook_is_declared_and_bound():
    with open(os.path.join(ROOT, "include", "b200pose.h")) as f:
        header = f.read()
    sig = pkg_module("_native")._SIGNATURES
    for name in ("b200pose_post_set_grids", "b200pose_post_debug_connections"):
        assert re.search(r"\bint %s\(b200pose_post\* post," % name, header), name
        assert name in sig
    assert sig["b200pose_post_set_grids"][0][1:] == [sig["b200pose_post_set_grids"][0][1]] * 2
