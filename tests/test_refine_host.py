"""CPU: the peak refinement core (csrc/refine_core.h, compiled for the host by tests/cuda/refine_core_host.cpp) and the
numpy oracle (tests/nms_modes_port.py) against cv2.resize(INTER_CUBIC, IPP off) and scipy.ndimage.gaussian_filter(sigma=3)
bit for bit, for every factor 1 .. 16 and every clipped window from 1x1 to 5x5; the oracle against the reference's own
NMS / paf_to_pose_cpp (tests/golden/nms_modes.npz); the drop-in's refusals; planted mistakes in the core."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT, golden, humans_rows_to_dicts, assert_humans_equal
import nms_modes_port as nmp
from oracle import nms_port, pafprocess_oracle, synth

cv2 = pytest.importorskip("cv2")
ndimage = pytest.importorskip("scipy.ndimage")

CSRC = os.path.join(ROOT, "pytorch_realtime_multi-person_pose_estimation_b200", "csrc")
CORE = os.path.join(CSRC, "refine_core.h")
FACTORS = range(1, 17)
SIZES = [(ph, pw) for ph in range(1, 6) for pw in range(1, 6)]


def compile_core(so, core=None):
    cmd = ["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-I" + CSRC, "-o", so,
           os.path.join(ROOT, "tests", "cuda", "refine_core_host.cpp")]
    if core:
        cmd.insert(1, '-DREFINE_CORE="%s"' % core)
    subprocess.run(cmd, check=True)
    lib = ctypes.CDLL(so)
    V, I = ctypes.c_void_p, ctypes.c_int
    lib.core_up.argtypes = [V, I, I, I, V]
    lib.core_refine.argtypes = [V, I, I, I, I, V, V]
    lib.core_refine.restype = I
    lib.core_gauss_weights.argtypes = [V]
    lib.core_gauss_rows.argtypes = [V, I, I, V]
    return lib


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    return compile_core(str(tmp_path_factory.mktemp("refine") / "librefinecore.so"))


@pytest.fixture(scope="module", autouse=True)
def no_ipp():
    old = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(False)
    yield
    cv2.ipp.setUseIPP(old)


def patches(ph, pw, seed):
    """Random, plateau (all equal, so every resized value ties) and tie-heavy (values k / 4) windows."""
    rs = np.random.RandomState(seed)
    return [rs.rand(ph, pw).astype(np.float32), np.full((ph, pw), 0.0, np.float32),
            np.full((ph, pw), 0.625, np.float32), (rs.randint(0, 5, (ph, pw)) / 4.0).astype(np.float32)]


def want(win, f, gauss):
    up = cv2.resize(win, None, fx=f, fy=f, interpolation=cv2.INTER_CUBIC)
    if gauss:
        up = ndimage.gaussian_filter(up, sigma=3)
    i = int(up.argmax())
    return up, i, up.reshape(-1)[i]


def core_refine(lib, win, f, gauss):
    ph, pw = win.shape
    win = np.ascontiguousarray(win, np.float32)
    patch = np.empty((ph * f, pw * f), np.float32)
    score = np.empty(1, np.float32)
    i = lib.core_refine(win.ctypes.data, ph, pw, f, int(gauss), score.ctypes.data, patch.ctypes.data)
    return patch, i, score[0]


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.int32)


def gauss_sum_mismatches(lib):
    """Rows of 1 .. 80 elements: the core's double sums against the oracle's (pinned to scipy), bit for bit - a
    changed rounding in the double accumulation rarely survives the final rounding to float32."""
    rs = np.random.RandomState(5)
    bad = 0
    for w in list(range(1, 26)) + [40, 64, 80]:
        a = rs.rand(6, w).astype(np.float32)
        got = np.empty((6, w), np.float64)
        lib.core_gauss_rows(a.ctypes.data, 6, w, got.ctypes.data)
        bad += int((got.view(np.int64) != nmp.gauss_rows_double(a).view(np.int64)).sum())
    return bad


def mismatches(lib, factors=FACTORS, stop=False):
    bad = []
    if gauss_sum_mismatches(lib):
        bad.append("gauss sums")
        if stop:
            return bad
    for f in factors:
        for ph, pw in SIZES:
            for k, win in enumerate(patches(ph, pw, 100 * f + 10 * ph + pw)):
                for gauss in (False, True):
                    up, i, s = want(win, f, gauss)
                    gp, gi, gs = core_refine(lib, win, f, gauss)
                    if not (np.array_equal(bits(up), bits(gp)) and i == gi and bits(s) == bits(gs)):
                        bad.append((f, ph, pw, k, gauss))
                        if stop:
                            return bad
    return bad


def test_gauss_weights_equal_scipy(core):
    from scipy.ndimage._filters import _gaussian_kernel1d
    w = np.empty(25, np.float64)
    core.core_gauss_weights(w.ctypes.data)
    ref = _gaussian_kernel1d(3, 0, 12)
    assert np.array_equal(w.view(np.int64), ref.view(np.int64))
    assert np.array_equal(nmp.GAUSS_W.view(np.int64), ref.view(np.int64))


@pytest.mark.parametrize("f", FACTORS)
def test_core_equals_cv2_and_scipy(f, core):
    """The resized patch, the smoothed patch, the first arg-max and the score, bit for bit."""
    assert mismatches(core, [f]) == []


@pytest.mark.parametrize("f", FACTORS)
def test_oracle_equals_cv2_and_scipy(f):
    for ph, pw in SIZES:
        for win in patches(ph, pw, 7 * f + ph * 5 + pw):
            up = cv2.resize(win, None, fx=f, fy=f, interpolation=cv2.INTER_CUBIC)
            assert np.array_equal(bits(up), bits(nmp.upsample_cubic(win, f))), (f, ph, pw)
            assert np.array_equal(bits(ndimage.gaussian_filter(up, sigma=3)), bits(nmp.gaussian3(up))), (f, ph, pw)


def test_gaussian_on_lines_shorter_than_the_radius():
    """Lines of 1 .. 40 elements (the reflection repeats when a line is shorter than the radius of 12)."""
    rs = np.random.RandomState(3)
    for h in (1, 2, 3, 5, 7, 12, 13, 25, 40):
        for w in (1, 2, 4, 11, 24, 40):
            a = rs.rand(h, w).astype(np.float32)
            assert np.array_equal(bits(ndimage.gaussian_filter(a, sigma=3)), bits(nmp.gaussian3(a))), (h, w)


def test_oracle_defaults_keep_the_existing_golden_files():
    for name, (heat, _) in (("p3", synth.stick_figures(3, 3)[:2]), ("noise0", synth.noise_maps(0))):
        got = nms_port.joint_list_from_nms(nmp.nms(heat, 0.1))
        np.testing.assert_array_equal(got, nms_port.joint_list_from_nms(nms_port.nms(heat, 0.1)))
        _check_golden("post_" + name, got, None, {"post_%s_joint_list" % name: golden("post_" + name)["joint_list"]})


# On the stick-figure maps the reference's cv2 resized through IPP, whose float cubic arithmetic is not OpenCV's own:
# positions are identical, scores differ by up to 5.4e-7 (p30 at f = 3, 9 ulps of the value).  The adversarial maps were
# run with IPP off (make_nms_modes_golden.py) and agree bit for bit.
GOLDEN_SCORE_TOL = 1e-6


def _check_golden(key, jl, humans, g):
    """positions identical, scores within GOLDEN_SCORE_TOL."""
    ref = g[key + "_joint_list"]
    assert jl.shape == ref.shape, key
    np.testing.assert_array_equal(jl[:, [0, 1, 3, 4]], ref[:, [0, 1, 3, 4]], err_msg=key)
    np.testing.assert_allclose(jl[:, 2], ref[:, 2], rtol=0, atol=GOLDEN_SCORE_TOL, err_msg=key)
    if humans is not None:
        assert_humans_equal(humans, humans_rows_to_dicts(g[key + "_humans"]), score_tol=GOLDEN_SCORE_TOL)


def test_oracle_equals_reference_golden():
    """The oracle at every factor and mode of the fixture against what the reference's NMS and paf_to_pose_cpp made
    of the same maps."""
    g = golden("nms_modes")
    port = pafprocess_oracle.load_port()
    for name, (heat, paf) in nmp.golden_scenarios().items():
        for f in nmp.GOLDEN_FACTORS:
            for mode, (refine, gauss) in nmp.MODES.items():
                key = nmp.golden_key(name, f, mode)
                if mode == "cubic":
                    jl, humans = nmp.paf_to_pose(heat, paf, port, thresh=nmp.GOLDEN_THRESH, upsample=f)
                else:
                    jl, humans = nms_port.joint_list_from_nms(nmp.nms(heat, nmp.GOLDEN_THRESH, 18, f, refine, gauss)), None
                _check_golden(key, jl, humans, g)


@pytest.mark.parametrize("f", [0, 17, 2.5, -8, "8", None])
def test_dropin_refuses_factors_before_cuda(f, monkeypatch):
    """NMS and paf_to_pose_cpp refuse a factor that is not an integer 1 .. 16 before any CUDA call."""
    import _b200_alias
    _b200_alias.load_package()
    import importlib
    p2p = importlib.import_module(_b200_alias.PKG + ".lib.utils.paf_to_pose")

    def no_cuda(*a, **k):
        raise AssertionError("CUDA was reached")
    monkeypatch.setattr(p2p, "_post", no_cuda)

    class C:
        class MODEL:
            DOWNSAMPLE = f
            NUM_KEYPOINTS = 18

        class TEST:
            THRESH_HEATMAP = 0.1
    heat = np.zeros((8, 8, 19), np.float32)
    with pytest.raises(NotImplementedError, match=repr(f).replace(".", r"\.")):
        p2p.NMS(heat, upsampFactor=f, config=C)
    with pytest.raises(ValueError, match=repr(f).replace(".", r"\.")):
        p2p.paf_to_pose_cpp(heat, np.zeros((8, 8, 38), np.float32), C)


def _planted(tmp_path, name, old, new):
    src = open(CORE).read()
    assert old in src, name
    path = tmp_path / ("refine_core_%s.h" % name)
    path.write_text(src.replace(old, new))
    return compile_core(str(tmp_path / ("lib_%s.so" % name)), core=str(path))


PLANTS = {
    "fma_gauss": ("t = rf_dadd(t, rf_dmul(s, w[kGaussRadius - k]));", "t = fma(s, w[kGaussRadius - k], t);"),
    "axes_swapped": ("tmp[Y * W + X] = rf_gauss_at(up + X, W, H, Y);       // axis 0\n",
                     "tmp[Y * W + X] = rf_gauss_at(up + Y * W, 1, W, X);\n"),
    "clamped_border": ("    return m >= n ? 2 * n - 1 - m : m;", "    return i < 0 ? 0 : (i > n - 1 ? n - 1 : i);"),
    "last_argmax": ("(v == bv && i < bi)", "(v == bv && i > bi)"),
}


@pytest.mark.parametrize("name", list(PLANTS))
def test_planted_mistakes_are_caught(name, tmp_path):
    old, new = PLANTS[name]
    if name == "axes_swapped":      # the second pass then runs along axis 0
        src_pass2 = ("up[Y * W + X] = rf_gauss_at(tmp + Y * W, 1, W, X);   // axis 1",
                     "up[Y * W + X] = rf_gauss_at(tmp + X, W, H, Y);")
        src = open(CORE).read().replace(old, new).replace(*src_pass2)
        assert src != open(CORE).read()
        path = tmp_path / "refine_core_axes.h"
        path.write_text(src)
        lib = compile_core(str(tmp_path / "lib_axes.so"), core=str(path))
    else:
        lib = _planted(tmp_path, name, old, new)
    assert mismatches(lib, stop=True), "planted mistake %s went unnoticed" % name
