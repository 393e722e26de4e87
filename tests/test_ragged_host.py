"""CPU: ragged batches (DESIGN.md 1, 2.8) - the grouping rule of PoseEngine.infer_images, its dispatch to the ragged
entry point, and the ragged C ABI surface."""
import ctypes
import itertools

import os
import re
import subprocess

import numpy as np

from conftest import ROOT, pkg_module


def _check_plan(shapes, cap, batches, waste):
    flat = sorted(itertools.chain.from_iterable(batches))
    assert flat == list(range(len(shapes)))                       # every frame exactly once
    for b in batches:
        assert 1 <= len(b) <= cap
        hc = max(shapes[i][0] for i in b)
        wc = max(shapes[i][1] for i in b)
        assert len(b) * hc * wc <= waste * sum(shapes[i][0] * shapes[i][1] for i in b)
        assert len({shapes[i][0] > shapes[i][1] for i in b}) == 1  # one orientation per batch


def test_grouping_rule_keeps_the_waste_bound_and_the_cap():
    eng = pkg_module("engine")
    rs = np.random.RandomState(3)
    for trial in range(50):
        n = int(rs.randint(1, 120))
        shapes = [tuple(int(v) for v in (8 * rs.randint(1, 90), 8 * rs.randint(1, 90))) for _ in range(n)]
        cap = int(rs.choice([1, 2, 7, 32]))
        batches = eng.plan_ragged_batches(shapes, cap)
        _check_plan(shapes, cap, batches, eng.RAGGED_WASTE)


def test_one_shape_gives_full_batches():
    eng = pkg_module("engine")
    assert eng.plan_ragged_batches([(368, 496)] * 32, 32) == [list(range(32))]
    assert [len(b) for b in eng.plan_ragged_batches([(368, 496)] * 70, 32)] == [32, 32, 6]


def test_near_shapes_share_a_batch_and_orientations_split():
    eng = pkg_module("engine")
    land = [(184, 240 + 8 * (i % 8)) for i in range(32)]           # 8 shapes, canvas waste 296 / 268 < 1.125
    assert eng.plan_ragged_batches(land, 32) == [sorted(range(32), key=lambda i: (land[i][1], i))]
    port = [(w, h) for h, w in land]
    mixed = land[:5] + port[:3] + land[5:8]
    batches = eng.plan_ragged_batches(mixed, 32)
    assert len(batches) == 2
    assert sorted(batches[0]) == [0, 1, 2, 3, 4, 8, 9, 10]          # landscape first ...
    assert sorted(batches[1]) == [5, 6, 7]                         # ... portrait frames in a batch of their own
    square = [(368, 368), (368, 376)]
    assert eng.plan_ragged_batches(square, 32) == [[0, 1]]          # a square frame groups with the landscape ones
    # far apart sizes do not share a canvas
    assert eng.plan_ragged_batches([(368, 368), (368, 656)], 32) == [[0], [1]]


def test_infer_images_runs_mixed_shapes_as_one_ragged_call_in_input_order(built, monkeypatch):
    """With a stand-in library: frames of different sizes go to b200pose_infer_raw_u8_ragged packed back to back in
    the batch's order, frames of one source size to the uniform entry point, and results come back in input order."""
    nat = pkg_module("_native")
    eng = pkg_module("engine")
    real = nat.lib()
    calls = []

    class Fake:
        b200pose_crop_geometry = staticmethod(real.b200pose_crop_geometry)
        b200pose_last_error = staticmethod(real.b200pose_last_error)

        @staticmethod
        def b200pose_infer_raw_u8(net, post, images, on_dev, n, sh, sw, dest, factor, mode, thresh, flip, stream):
            first = np.ctypeslib.as_array(ctypes.cast(images.value, ctypes.POINTER(ctypes.c_ubyte)), (n, sh, sw, 3))[:, 0, 0, 0]
            calls.append(("uniform", [(sh, sw)] * n, [int(v) for v in first], flip))
            return 0

        @staticmethod
        def b200pose_infer_raw_u8_ragged(net, post, images, on_dev, n, hw, dest, factor, mode, thresh, flip, stream):
            shapes = [(hw[2 * i], hw[2 * i + 1]) for i in range(n)]
            buf = ctypes.cast(images.value, ctypes.POINTER(ctypes.c_ubyte))
            off, first = 0, []
            for h, w in shapes:
                first.append(int(buf[off]))
                assert all(buf[off + k] == first[-1] for k in range(0, h * w * 3, 97))
                off += h * w * 3
            calls.append(("ragged", shapes, first, flip))
            return 0

    monkeypatch.setattr(nat, "lib", lambda: Fake)

    class StubPost:
        batch_cap = 4
        def last_ticket(self): return len(calls) - 1
    pe = object.__new__(eng.PoseEngine)
    pe.net, pe.post, pe.mode = object.__new__(eng.NativeNet), StubPost(), 0
    pe.net._h = pe.post._h = None
    pe.fetch = lambda: [("humans-of", v) for v in calls[-1][2]]
    sizes = [(184, 250), (184, 246), (250, 184), (184, 250), (184, 262), (184, 250)]
    imgs = [np.full(s + (3,), i + 1, np.uint8) for i, s in enumerate(sizes)]
    res = pe.infer_images(imgs, dest_size=184, flip=True)
    assert res == [("humans-of", i + 1) for i in range(6)]
    # landscape, by padded size: 184x248, 3 x 184x256 (cap 4), then 184x264; the portrait frame on its own
    assert [(c[0], c[2]) for c in calls] == [("ragged", [2, 1, 4, 6]), ("uniform", [5]), ("uniform", [3])]
    assert calls[0][1] == [(184, 246), (184, 250), (184, 250), (184, 250)] and calls[0][3] == 1
    assert pe._last == (1, 256, 184)


def test_ragged_entry_points_are_declared_exported_and_bound(built):
    nat = pkg_module("_native")
    for name in ("b200pose_net_forward_ragged_u8", "b200pose_infer_raw_u8_ragged"):
        assert name in nat.EXPORTED
        assert hasattr(ctypes.CDLL(nat.LIB_PATH), name)
        assert getattr(nat.lib(), name).argtypes is not None
    eng = pkg_module("engine")
    assert callable(eng.NativeNet.forward_ragged_u8_ptr) and callable(eng.PoseEngine.infer_raw_ragged_async_u8)



def test_masked_conv_epilogues_do_not_spill(built):
    """The extent masks live in the epilogues of the wgmma and CUDA-core convolutions: ptxas reports no local-memory
    spills for any of their sm_90a instantiations."""
    csrc = os.path.join(ROOT, "pytorch_realtime_multi-person_pose_estimation_b200", "csrc")
    for src, kernels in (("conv_tc.cu", "conv_tc_kernel"), ("conv_misc.cu", "conv_")):
        r = subprocess.run([os.environ.get("NVCC", "nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                            "-Xptxas", "-v", "-c", os.path.join(csrc, src), "-o", os.devnull],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-2000:]
        seen = 0
        for fn, body in re.findall(r"Compiling entry function '(\S+)' for 'sm_90a'(.*?)(?=Compiling entry|\Z)", r.stdout, re.S):
            if kernels in fn:
                seen += 1
                assert "0 bytes spill stores, 0 bytes spill loads" in body, (fn, body)
        assert seen > 0, src
