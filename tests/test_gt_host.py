"""CPU: COCO training targets (DESIGN.md 2.19) - csrc/gt_core.h compiled for the host and the numpy port (tests/gt_port.py)
against the reference's own get_ground_truth outputs (tests/golden/gt_*.npz), bit for bit; the core's exp against
np.exp; planted mistakes that the comparison must catch; the kernels' resource use and the C ABI."""
import os
import subprocess

import numpy as np
import pytest

import gt_check as gc
import gt_port
from conftest import ROOT, pkg_module

GOLDENS = gc.goldens()


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    return gc.compile_core(str(tmp_path_factory.mktemp("gt") / "libgtcore.so"))


def _equal(got, want):
    return np.array_equal(gc.bits(got), gc.bits(want))


def test_goldens_cover_the_scenarios():
    assert {"p1", "p5", "p30", "crowd", "borders", "zero_length", "round_ties", "axis_limbs", "neck_visibility",
            "size_656x368", "size_64x128", "overlap", "width_edges"} <= set(GOLDENS)
    assert len(GOLDENS["p30"]["kp"]) == 30 and tuple(GOLDENS["size_656x368"]["size"]) == (656, 368)
    kp = GOLDENS["neck_visibility"]["kp"]
    assert sorted((int(k[6, 2]), int(k[5, 2])) for k in kp) == [(a, b) for a in range(3) for b in range(3)]
    assert np.any(GOLDENS["borders"]["kp"][:, :, 0] == 368.0) and np.any(GOLDENS["borders"]["kp"][:, :, 1] == 368.0)
    # limbs of the crowd overlap: PAF cells averaged over 2 .. 4 persons have non-unit vectors
    p = GOLDENS["crowd"]["paf64"]
    mag = np.hypot(p[0::2], p[1::2])
    assert np.any((mag > 0) & (mag < 0.99))
    assert np.any(GOLDENS["overlap"]["heat"][:18] == 1.0)


@pytest.mark.parametrize("name", sorted(GOLDENS))
def test_core_equals_golden_bit_for_bit(core, name):
    g = GOLDENS[name]
    heat, paf, paf64 = gc.core_gt(core, [g["kp"]], [tuple(g["size"])], want64=True)
    assert heat.shape[1:] == g["heat"].shape and paf.shape[1:] == g["paf"].shape
    assert _equal(heat[0], g["heat"]) and _equal(paf[0], g["paf"])
    assert _equal(paf64[0], g["paf64"])


@pytest.mark.parametrize("name", sorted(GOLDENS))
def test_port_equals_golden_bit_for_bit(name):
    g = GOLDENS[name]
    heat, paf = gt_port.ground_truth(g["kp"], g["size"])
    assert _equal(heat, g["heat"]) and _equal(paf, g["paf"])
    assert _equal(gt_port.ground_truth(g["kp"], g["size"], float64=True)[1], g["paf64"])


def test_limb_norm_is_the_recorded_one(core):
    n = 0
    for g in GOLDENS.values():
        for (dx, dy), want in zip(g["norm_d"], g["norm"]):
            assert core.core_limb_norm(dx, dy) == want and gt_port.limb_norm(dx, dy) == want, (dx, dy)
            n += 1
    assert n > 1000
    # the fixtures' components are float32 keypoints over 8, whose squares are exact in float64, so any formula agrees
    # there; on general float64 vectors the fused form is the one the core and the port share
    d = np.random.RandomState(4).uniform(-40, 40, (20000, 2))
    fused = [core.core_limb_norm(x, y) for x, y in d]
    assert fused == [gt_port.limb_norm(x, y) for x, y in d]
    assert fused != [float(np.sqrt(x * x + y * y)) for x, y in d]


def test_exp_within_an_ulp_of_numpy(core):
    x = -np.random.RandomState(0).uniform(0, 4.6052, 1000000)
    got = np.array([core.core_exp(v) for v in x])
    d = np.abs(got.view(np.int64) - np.exp(x).view(np.int64))
    assert d.max() <= 1
    assert core.core_exp(0.0) == 1.0 and core.core_exp(-4.6052) == np.exp(-4.6052)


def test_no_persons_gives_zero_pafs_and_background_one(core):
    heat, paf = gc.core_gt(core, [np.zeros((0, 17, 3), np.float32)], [(368, 368)])
    assert np.all(heat[0, :18] == 0) and np.all(heat[0, 18] == 1) and _equal(paf, np.zeros_like(paf))
    ph, pp = gt_port.ground_truth(np.zeros((0, 17, 3)), (368, 368))
    assert _equal(heat[0], ph) and _equal(paf[0], pp)


def test_core_equals_port_on_random_ragged_scenarios(core):
    kps, hw = gc.random_scenario(11, 6, sizes=((368, 368), (368, 656), (128, 64), (100, 36)), max_persons=6)
    heat, paf = gc.core_gt(core, kps, hw)
    ph, pp = gt_port.ground_truth_batch(kps, hw)
    assert _equal(heat, ph) and _equal(paf, pp)
    for i, (h, w) in enumerate(hw):      # +0 outside each image's grid
        assert _equal(heat[i, :, h // 8:], np.zeros_like(heat[i, :, h // 8:]))
        assert _equal(paf[i, :, :, w // 8:], np.zeros_like(paf[i, :, :, w // 8:]))


@pytest.mark.parametrize("name", [k for k, _, _ in gc.PLANTED])
def test_planted_mistake_fails_the_goldens(tmp_path, name):
    lib = gc.compile_core(str(tmp_path / "lib.so"), gc.planted_header(tmp_path, name))
    failed = []
    for k, g in GOLDENS.items():
        heat, paf, paf64 = gc.core_gt(lib, [g["kp"]], [tuple(g["size"])], want64=True)
        if not (_equal(heat[0], g["heat"]) and _equal(paf[0], g["paf"])):
            failed.append(k)
    assert failed, name


@pytest.mark.parametrize("name", [k for k, _, _ in gc.EQUIVALENT])
def test_equivalent_variants_match_the_goldens(tmp_path, name):
    """These rewrites look like mistakes but give the reference's numbers exactly (gt_check.EQUIVALENT says why)."""
    lib = gc.compile_core(str(tmp_path / "lib.so"), gc.planted_header(tmp_path, name))
    for k, g in GOLDENS.items():
        heat, paf, paf64 = gc.core_gt(lib, [g["kp"]], [tuple(g["size"])], want64=True)
        assert _equal(heat[0], g["heat"]) and _equal(paf64[0], g["paf64"]), k


def test_rescale_of_a_quotient_is_exact():
    s = np.random.RandomState(1).uniform(-4, 4, 1000000)
    for c in (3, 5, 6, 7, 9, 11):
        a = s / c
        assert np.array_equal((a * c) / c, a)
        assert not np.array_equal((s * c) / c, s)      # but not of an arbitrary value


def test_gt_kernels_do_not_spill(built):
    import __graft_entry__ as g
    nvcc = os.environ.get("NVCC", "nvcc")
    r = subprocess.run([nvcc] + g.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(g.CSRC, "gt.cu"), "-o", os.devnull],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=True)
    blocks = r.stdout.split("Compiling entry function")[1:]
    names = [b.split("'")[1] for b in blocks]
    assert len(blocks) == 3 and all("gt_" in n for n in names), names
    for b in blocks:
        assert "0 bytes spill stores, 0 bytes spill loads" in b, b


def test_c_abi_declares_the_calls():
    nat = pkg_module("_native")
    header = open(os.path.join(ROOT, "include", "b200pose.h")).read()
    for name in ("b200pose_ground_truth", "b200pose_net_stage_losses"):
        assert name in nat.EXPORTED and "int %s(" % name in header


def test_ground_truth_refusals_before_any_device_work():
    """Refusals that need no device: the library checks its arguments before it touches CUDA."""
    eng = pkg_module("engine")
    nat = pkg_module("_native")
    kp = np.zeros((1, 17, 3), np.float32)
    with pytest.raises(nat.B200PoseError, match="keypoints"):
        eng.ground_truth([np.full((1, 17, 3), np.nan, np.float32)], [(368, 368)])
    with pytest.raises(nat.B200PoseError, match="sizes"):
        eng.ground_truth([kp], [(4, 368)])
    with pytest.raises(nat.B200PoseError, match="persons"):
        eng.ground_truth([np.zeros((257, 17, 3), np.float32)], [(368, 368)])
    with pytest.raises(nat.B200PoseError, match="images"):
        eng.ground_truth([kp] * 1025, [(368, 368)] * 1025)
    with pytest.raises(nat.B200PoseError, match="canvas 1025 x 46 above 1024 x 1024 cells"):
        eng.ground_truth([kp], [(368, 368)], 0, (1025, 46))
    with pytest.raises(nat.B200PoseError, match="canvas 40 x 46 below"):
        eng.ground_truth([kp], [(368, 368)], 0, (40, 46))
