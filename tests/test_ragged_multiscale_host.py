"""CPU: multi-scale test-time averaging on ragged batches (DESIGN.md 2.7, 2.8) - infer_images(scales=...) dispatch, the
C ABI surface of b200pose_infer_raw_u8_multiscale_ragged, and the host build of the ragged bicubic resize."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT, pkg_module
from oracle import glue_port

CSRC = os.path.join(ROOT, "pytorch_realtime_multi-person_pose_estimation_b200", "csrc")
SCALES = (0.5, 1.0, 1.5, 2.0)


def _engine_with_fake_lib(monkeypatch, batch_cap):
    """A PoseEngine whose library records the multi-scale calls (frames packed as the engine sends them)."""
    nat = pkg_module("_native")
    eng = pkg_module("engine")
    real = nat.lib()
    calls = []

    def first_bytes(ptr, shapes):
        buf = ctypes.cast(ptr.value, ctypes.POINTER(ctypes.c_ubyte))
        off, first = 0, []
        for h, w in shapes:
            first.append(int(buf[off]))
            assert all(buf[off + k] == first[-1] for k in range(0, h * w * 3, 53))
            off += h * w * 3
        return first

    class Fake:
        b200pose_crop_geometry = staticmethod(real.b200pose_crop_geometry)
        b200pose_last_error = staticmethod(real.b200pose_last_error)

        @staticmethod
        def b200pose_infer_raw_u8_multiscale(net, post, images, on_dev, n, sh, sw, base, factor, scales, ns, mode, thresh,
                                             flip, stream):
            calls.append(("uniform", [(sh, sw)] * n, first_bytes(images, [(sh, sw)] * n), [scales[i] for i in range(ns)],
                          base, factor, flip))
            return 0

        @staticmethod
        def b200pose_infer_raw_u8_multiscale_ragged(net, post, images, on_dev, n, hw, base, factor, scales, ns, mode,
                                                    thresh, flip, stream):
            shapes = [(hw[2 * i], hw[2 * i + 1]) for i in range(n)]
            calls.append(("ragged", shapes, first_bytes(images, shapes), [scales[i] for i in range(ns)], base, factor,
                          flip))
            return 0

    monkeypatch.setattr(nat, "lib", lambda: Fake)

    class StubPost:
        def __init__(self): self.batch_cap = batch_cap
        def last_ticket(self): return len(calls) - 1
    pe = object.__new__(eng.PoseEngine)
    pe.net, pe.post, pe.mode = object.__new__(eng.NativeNet), StubPost(), 0
    pe.net._h = pe.post._h = None
    pe.fetch = lambda: [("humans-of", v) for v in calls[-1][2]]
    return pe, calls


def test_multiscale_infer_images_groups_mixed_sizes_into_ragged_calls(built, monkeypatch):
    """Mixed sizes with scales: groups follow plan_ragged_batches on the base padded sizes and batch_cap; a group of
    several source sizes calls the ragged multi-scale entry with its frames packed in batch order, a group of one source
    size the uniform one; results come back in input order and the engine keeps each frame's base padded size."""
    nat = pkg_module("_native")
    eng = pkg_module("engine")
    pe, calls = _engine_with_fake_lib(monkeypatch, batch_cap=4)
    sizes = [(40, 50), (40, 52), (50, 40), (40, 50), (40, 55), (40, 50), (41, 50), (40, 50), (50, 40), (40, 50)]
    imgs = [np.full(s + (3,), i + 1, np.uint8) for i, s in enumerate(sizes)]
    res = pe.infer_images(imgs, dest_size=64, factor=8, flip=True, scales=SCALES)
    assert res == [("humans-of", i + 1) for i in range(len(sizes))]
    pads = [nat.crop_geometry(h, w, 64, 8)[2] for h, w in sizes]
    groups = eng.plan_ragged_batches(pads, 4)
    assert len(calls) == len(groups)
    for call, part in zip(calls, groups):
        kind, shapes, first, scales, base, factor, flip = call
        assert first == [i + 1 for i in part] and shapes == [sizes[i] for i in part]
        assert kind == ("uniform" if len(set(shapes)) == 1 else "ragged"), (kind, shapes)
        assert scales == list(SCALES) and (base, factor, flip) == (64, 8, 1)
    kinds = [c[0] for c in calls]
    assert "ragged" in kinds and "uniform" in kinds and max(len(p) for p in groups) == 4
    for t in (len(calls) - 2, len(calls) - 1):        # the engine keeps the shapes of the last two runs
        part = groups[t]
        if kinds[t] == "ragged":
            assert pe._shape_of(t) == (len(part), [pads[i][0] for i in part], [pads[i][1] for i in part])
        else:
            assert pe._shape_of(t) == (len(part),) + pads[part[0]]


def test_multiscale_ragged_async_remembers_per_frame_base_pads(built, monkeypatch):
    nat = pkg_module("_native")
    pe, calls = _engine_with_fake_lib(monkeypatch, batch_cap=8)
    shapes = [(90, 123), (123, 90), (60, 61)]
    packed = np.concatenate([np.full(s + (3,), i + 7, np.uint8).ravel() for i, s in enumerate(shapes)])
    t = pe.infer_raw_multiscale_ragged_async_u8(packed.ctypes.data, False, shapes, (1.0, 0.5), 96, 8, 0.1, False)
    assert calls == [("ragged", shapes, [7, 8, 9], [1.0, 0.5], 96, 8, 0)]
    pads = [nat.crop_geometry(h, w, 96, 8)[2] for h, w in shapes]
    assert t == 0 and pe._shape_of(t) == (3, [p[0] for p in pads], [p[1] for p in pads])


def test_multiscale_ragged_entry_is_declared_exported_and_bound(built):
    nat = pkg_module("_native")
    with open(os.path.join(ROOT, "include", "b200pose.h")) as f:
        header = f.read()
    for name in ("b200pose_infer_raw_u8_multiscale_ragged", "b200pose_post_debug_maps"):
        assert re.search(r"\bint %s\(" % name, header), name
        assert name in nat.EXPORTED
        assert hasattr(ctypes.CDLL(nat.LIB_PATH), name)
        assert getattr(nat.lib(), name).argtypes is not None
    eng = pkg_module("engine")
    assert callable(eng.PoseEngine.infer_raw_multiscale_ragged_async_u8)


def test_multiscale_ragged_entry_rejects_null_handles(built):
    nat = pkg_module("_native")
    hw = (ctypes.c_int * 2)(64, 64)
    sc = (ctypes.c_double * 1)(1.0)
    frame = np.zeros((64, 64, 3), np.uint8)
    rc = nat.lib().b200pose_infer_raw_u8_multiscale_ragged(None, None, frame.ctypes.data, 0, 1, hw, 64, 8, sc, 1, 0,
                                                           ctypes.c_float(0.1), 0, None)
    with pytest.raises(nat.B200PoseError, match="null handle"):
        nat.check(rc, "b200pose_infer_raw_u8_multiscale_ragged")


@pytest.fixture(scope="module")
def ragged_core(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("core") / "libresize_ragged_host.so")
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-shared", "-fPIC", "-o", so,
                    os.path.join(ROOT, "tests", "cuda", "resize_ragged_host.cpp")], check=True)
    lib = ctypes.CDLL(so)
    lib.core_resize_cubic_ragged.argtypes = [ctypes.c_void_p] + [ctypes.c_int] * 3 + [ctypes.c_void_p] * 2 + \
        [ctypes.c_int] * 2
    return lib


def test_ragged_cubic_resize_core_on_host_matches_each_frame_resized_alone(built, ragged_core):
    """csrc/resize_core.h ragged_resize / rs_cubic_ragged_at (what resize_cubic_accum_kernel calls), compiled for
    the host: each frame of a mixed canvas resized from its own extent at scale s to its own base grid equals the
    oracle's resize_cubic of that frame alone, bit for bit, for the four scale ratios; the taps never read the canvas
    outside the frame (filled with NaN here), and every element outside a frame's base extent is +0."""
    nat = pkg_module("_native")
    rs = np.random.RandomState(19)
    raw = [(90, 123), (123, 90), (60, 61), (97, 96), (200, 131), (75, 150), (88, 88)]
    base = 96
    base_pads = [nat.crop_geometry(h, w, base, 8)[2] for h, w in raw]
    dhc, dwc = max(p[0] for p in base_pads) // 8, max(p[1] for p in base_pads) // 8
    for s in SCALES:
        pads = [nat.crop_geometry(h, w, int(base * s), 8)[2] for h, w in raw]
        shc, swc = max(p[0] for p in pads) // 8, max(p[1] for p in pads) // 8
        src = np.full((len(raw), shc, swc), np.nan, np.float32)
        frames = []
        for i, ((ph, pw), (bh, bw)) in enumerate(zip(pads, base_pads)):
            src[i, :ph // 8, :pw // 8] = rs.randn(ph // 8, pw // 8)
            frames += [ph // 8, pw // 8, bh // 8, bw // 8]
        hw = (ctypes.c_int * len(frames))(*frames)
        out = np.full((len(raw), dhc, dwc), -1.0, np.float32)
        ragged_core.core_resize_cubic_ragged(src.ctypes.data, len(raw), shc, swc, hw, out.ctypes.data, dhc, dwc)
        for i, ((ph, pw), (bh, bw)) in enumerate(zip(pads, base_pads)):
            want = glue_port.resize_cubic(src[i, :ph // 8, :pw // 8], bh // 8, bw // 8)
            np.testing.assert_array_equal(out[i, :bh // 8, :bw // 8], want, err_msg="scale %s frame %d" % (s, i))
            outside = np.concatenate([out[i, bh // 8:].ravel(), out[i, :bh // 8, bw // 8:].ravel()])
            assert (outside.view(np.int32) == 0).all(), (s, i)


def test_resize_cubic_accum_kernel_does_not_spill(built):
    r = subprocess.run([os.environ.get("NVCC", "nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                        "-Xptxas", "-v", "-c", os.path.join(CSRC, "resize.cu"), "-o", os.devnull],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:]
    bodies = [body for fn, body in re.findall(r"Compiling entry function '(\S+)' for 'sm_90a'(.*?)(?=Compiling entry|\Z)",
                                              r.stdout, re.S) if "resize_cubic_accum_kernel" in fn]
    assert len(bodies) == 1 and "0 bytes spill stores, 0 bytes spill loads" in bodies[0], r.stdout[-2000:]
