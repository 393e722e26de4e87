"""CPU: training batches (DESIGN.md 2.20) - csrc/aug_core.h compiled for the host against Pillow's digests over the whole
colour cube and against the unmodified reference loader's samples (tests/golden/aug_*.npz) bit for bit; the draws and
keypoints of engine.augment_params / augment_keypoints; float64-keypoint targets; planted mistakes."""
import hashlib

import numpy as np
import pytest

import aug_check as ac
import gt_check as gc

GOLDENS = ac.goldens()


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    return ac.compile_core(str(tmp_path_factory.mktemp("aug") / "libaugcore.so"))


@pytest.fixture(scope="module")
def gt_core(tmp_path_factory):
    return gc.compile_core(str(tmp_path_factory.mktemp("gt") / "libgtcore.so"))


def _cube():
    c = np.arange(1 << 24, dtype=np.uint32)
    return np.ascontiguousarray(np.stack([(c >> 16) & 255, (c >> 8) & 255, c & 255], -1).astype(np.uint8))


def _digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def test_goldens_cover_the_draws():
    ps = {k: ac.params_of(g)[0] for k, g in GOLDENS.items()}
    assert {True, False} == {p["hflip"] for p in ps.values()}
    assert any(p["jpeg"] for p in ps.values()) and any(p["gray"] for p in ps.values())
    assert any(p["order"][0] == 1 for p in ps.values()) and any(p["order"][3] == 1 for p in ps.values())
    assert {96, 368} == {int(g["edge"]) for g in GOLDENS.values()}
    assert any(g["src"].shape[0] > g["src"].shape[1] for g in GOLDENS.values())
    assert any(max(g["src"].shape[:2]) > 2 * int(g["edge"]) for g in GOLDENS.values())


@pytest.mark.parametrize("op", ["brightness", "saturation", "hue", "contrast", "L"])
def test_core_reproduces_pillow_on_the_colour_cube(core, op):
    want = ac.cube()[op]
    cube = _cube()
    if op == "L":
        a = cube.copy()
        core.core_pixels(4, a.ctypes.data, 1 << 24, 0.0, 0)
        assert _digest(a[:, 0].reshape(4096, 4096)) == want
        return
    assert len(want) >= 5
    for key, d in want.items():
        a = cube.copy()
        if op == "contrast":
            mean, f = key.split()
            core.core_pixels(1, a.ctypes.data, 1 << 24, float(f), int(mean))
        else:
            core.core_pixels({"brightness": 0, "saturation": 2, "hue": 3}[op], a.ctypes.data, 1 << 24, float(key), 0)
        assert _digest(a.reshape(4096, 4096, 3)) == d, (op, key)


@pytest.mark.parametrize("name", sorted(GOLDENS))
def test_params_reproduce_the_reference_meta(name):
    g = GOLDENS[name]
    p = ac.params_of(g)[0]
    assert p["hflip"] == bool(g["hflip"])
    assert np.array_equal(np.array(p["scale"]), g["scale"])
    assert np.array_equal(np.array(p["crop"]) - np.array(p["pad"]), g["offset"])
    assert np.array_equal(p["valid_area"], g["valid_area"])


@pytest.mark.parametrize("name", sorted(GOLDENS))
def test_keypoints_reproduce_the_reference(name):
    g = GOLDENS[name]
    p = ac.params_of(g)
    k = ac.engine().augment_keypoints([g["kp"]], p)[0]
    want = g["kp_out"].reshape(k.shape)
    assert k.dtype == want.dtype == (np.float64 if p[0]["hflip"] else np.float32)
    assert np.array_equal(ac.bits(k), ac.bits(want))


@pytest.mark.parametrize("name", sorted(GOLDENS))
def test_core_reproduces_the_reference_images(core, name):
    g = GOLDENS[name]
    p = ac.params_of(g)[0]
    u8 = ac.colour_stages(core, g, p)
    assert np.array_equal(u8, g["u8"])
    assert np.array_equal(ac.bits(ac.to_tensor(u8, p)), ac.bits(g["image"]))


@pytest.mark.parametrize("name", sorted(GOLDENS))
def test_core_reproduces_the_reference_targets(core, gt_core, name):
    g = GOLDENS[name]
    p = ac.params_of(g)
    k = ac.engine().augment_keypoints([g["kp"]], p)[0]
    E = int(g["edge"])
    if k.dtype == np.float64:
        heat = np.empty((19, E // 8, E // 8), np.float32)
        paf = np.empty((38, E // 8, E // 8), np.float32)
        kk = np.ascontiguousarray(k)
        core.core_ground_truth_f64(kk.ctypes.data, len(kk), E, E, heat.ctypes.data, paf.ctypes.data)
    else:
        heat, paf = gc.core_gt(gt_core, [k], [(E, E)])
        heat, paf = heat[0], paf[0]
    assert np.array_equal(ac.bits(heat), ac.bits(g["heat"])) and np.array_equal(ac.bits(paf), ac.bits(g["paf"]))


def test_float32_keypoints_after_a_flip_fail_the_goldens(gt_core):
    failed = 0
    for g in GOLDENS.values():
        p = ac.params_of(g)
        if not p[0]["hflip"]:
            continue
        k = ac.engine().augment_keypoints([g["kp"]], p)[0].astype(np.float32)
        E = int(g["edge"])
        heat, paf = gc.core_gt(gt_core, [k], [(E, E)])
        failed += not (np.array_equal(ac.bits(heat[0]), ac.bits(g["heat"])) and
                       np.array_equal(ac.bits(paf[0]), ac.bits(g["paf"])))
    assert failed > 0


def test_jpeg_round_trip_is_cv2_q50(core):
    """The JPEG samples' images equal the core's colour stages followed by cv2's quality-50 encode + decode, which is
    what the device runs; without the round trip they differ."""
    n = 0
    for g in GOLDENS.values():
        p = ac.params_of(g)[0]
        if p["jpeg"]:
            n += 1
            assert np.array_equal(ac.colour_stages(core, g, p), g["u8"])
            assert not np.array_equal(ac.colour_stages(core, g, p, jpeg=False), g["u8"])
    assert n >= 2


def test_contrast_mean_without_the_pad_fails_the_goldens(core):
    failed = 0
    for g in GOLDENS.values():
        p = ac.params_of(g)[0]
        (cw, ch), (left, top) = p["cropped"], p["pad"]
        E = int(g["edge"])
        if (cw, ch) == (E, E) or p["jpeg"]:
            continue
        order = list(p["order"])
        at = order.index(1)
        # the stages before contrast over the whole image, then contrast against the mean of the pasted window only
        img = ac.colour_stages(core, g, dict(p, order=order[:at] + [9] * (4 - at), jpeg=False, gray=False))
        win = np.ascontiguousarray(img[top:top + ch, left:left + cw]).reshape(-1, 3)
        lum = win.copy()
        core.core_pixels(4, lum.ctypes.data, len(lum), 0.0, 0)
        mean = int(lum[:, 0].astype(np.int64).sum() / len(lum) + 0.5)
        a = np.ascontiguousarray(img.reshape(-1, 3))
        core.core_pixels(1, a.ctypes.data, len(a), p["factors"][1], mean)
        for op in order[at + 1:]:
            core.core_pixels(op, a.ctypes.data, len(a), p["factors"][op], 0)
        failed += not np.array_equal(a.reshape(img.shape), g["u8"])
    assert failed > 0


@pytest.mark.parametrize("name", [k for k, _, _ in ac.PLANTED])
def test_planted_mistake_fails_the_goldens(tmp_path, name):
    """Each planted mistake changes a golden sample's image or a colour-cube digest."""
    lib = ac.compile_core(str(tmp_path / "lib.so"), ac.planted_header(tmp_path, name))
    failed = 0
    for g in GOLDENS.values():
        p = ac.params_of(g)[0]
        failed += not np.array_equal(ac.colour_stages(lib, g, p), g["u8"])
    cube = _cube()
    for key, d in ac.cube()["contrast"].items():
        mean, f = key.split()
        a = cube.copy()
        lib.core_pixels(1, a.ctypes.data, 1 << 24, float(f), int(mean))
        failed += _digest(a.reshape(4096, 4096, 3)) != d
    assert failed > 0
