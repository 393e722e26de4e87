"""CPU: OpenPose_Model's static surface and oracle - the library's tensor table against the reference module's
state_dict (tests/golden/openpose_spec.json), the loader's checks, the C declarations, and the CPU oracle of the graph
(tests/openpose_port) against the unmodified module's outputs (tests/golden/openpose_{64,368}.npz).  The GPU side is
tests/test_gpu_openpose.py."""
import ctypes
import json
import os
from collections import OrderedDict

import numpy as np
import pytest
import torch

import openpose_port
from conftest import GOLDEN, ROOT, golden, pkg_module


def _spec():
    with open(os.path.join(GOLDEN, "openpose_spec.json")) as f:
        return json.load(f)


LAYOUTS = [(1, 1), (1, 11), (11, 1), (2, 3), (6, 6)]      # tests/golden/openpose_<l2>_<l1>_64.npz


@pytest.mark.parametrize("arch", [(4, 2), (1, 1), (5, 3), (1, 11), (11, 1), (2, 3), (6, 6)])
def test_static_shape_table_equals_the_reference_state_dict(built, arch):
    ref = [(k, tuple(s)) for k, s in _spec()["%d,%d" % arch]]
    nat, eng = pkg_module("_native"), pkg_module("engine")
    assert nat.openpose_shapes(*arch) == [s for _, s in ref]
    assert eng.openpose_state_dict_keys(*arch) == [k for k, _ in ref]
    assert list(openpose_port.state_dict_spec(*arch).items()) == ref
    assert nat.lib().b200pose_openpose_num_tensors(*arch) == len(ref)
    dims = (ctypes.c_long * 4)()
    assert nat.lib().b200pose_openpose_tensor_shape(arch[0], arch[1], len(ref), dims) < 0
    assert nat.lib().b200pose_openpose_tensor_shape(arch[0], arch[1], -1, dims) < 0


def test_spec_counts_of_the_default_model():
    ref = _spec()["4,2"]
    assert len(ref) == 327 and 27 + 50 * 6 == 327


@pytest.mark.parametrize("arch", [(0, 1), (1, 0), (7, 6), (-1, 2)])
def test_invalid_architectures_are_refused(built, arch):
    nat, eng = pkg_module("_native"), pkg_module("engine")
    assert nat.lib().b200pose_openpose_num_tensors(*arch) < 0
    with pytest.raises(nat.B200PoseError, match="stages"):
        nat.openpose_shapes(*arch)
    h = ctypes.c_void_p()
    assert nat.lib().b200pose_net_create_openpose(ctypes.byref(h), 0, *arch) != 0
    assert b"OpenPose_Model" in nat.lib().b200pose_last_error()


def test_declared_and_exported(built):
    with open(os.path.join(ROOT, "include", "b200pose.h")) as f:
        header = f.read()
    for decl in ("int b200pose_net_create_openpose(b200pose_net** out, int cuda_device, int l2_stages, int l1_stages);",
                 "int b200pose_openpose_num_tensors(int l2_stages, int l1_stages);",
                 "int b200pose_openpose_tensor_shape(int l2_stages, int l1_stages, int index, long dims[4]);"):
        assert decl in header
        name = decl.split("(")[0].split()[-1]
        assert name in pkg_module("_native").EXPORTED


def test_loader_names_the_first_mismatch_before_any_device_work(built):
    """openpose_engine checks every key and shape first; the refusals below happen on a machine without a GPU too."""
    nat, eng = pkg_module("_native"), pkg_module("engine")
    sd = openpose_port.he_state_dict(1, 1)
    bad = OrderedDict((k.replace("l2_stages.0.Mconv3_1.MPrelu", "l2_stages.0.Mconv3_1.Prelu"), v) for k, v in sd.items())
    with pytest.raises(nat.B200PoseError, match=r"entry \d+ is 'l2_stages.0.Mconv3_1.Prelu.weight', expected "
                                                r"'l2_stages.0.Mconv3_1.MPrelu.weight'"):
        eng.openpose_engine(bad, 1, 1)
    bad = OrderedDict(sd)
    bad["l1_stages.0.Mconv6.Mconv.weight"] = torch.zeros((256, 288, 3, 3))
    with pytest.raises(nat.B200PoseError, match=r"'l1_stages.0.Mconv6.Mconv.weight' has shape \(256, 288, 3, 3\), "
                                                r"expected \(256, 288, 1, 1\)"):
        eng.openpose_engine(bad, 1, 1)
    with pytest.raises(nat.B200PoseError, match="missing"):
        eng.openpose_engine(OrderedDict(list(sd.items())[:-1]), 1, 1)
    with pytest.raises(nat.B200PoseError, match="OpenPose_Model\\(4, 2\\) state_dict: entry 77 is 'l1_stages.0.Mconv1_0.Mconv.weight'"):
        eng.openpose_engine(sd, 4, 2)


def test_he_weights_have_negative_and_steep_slopes(built):
    sd = openpose_port.he_state_dict()
    slopes = np.concatenate([v.numpy() for k, v in sd.items() if v.dim() == 1 and not k.endswith("bias")])
    assert (slopes < 0).mean() > 0.15 and (slopes > 1).mean() > 0.15


@pytest.mark.parametrize("name", ["openpose_64", "openpose_368"])
def test_oracle_port_matches_the_reference_golden(built, name):
    g = golden(name)
    hw = int(g["hw"])
    x = torch.rand((1, 3, hw, hw), generator=torch.Generator().manual_seed(int(g["seed"]))) - 0.5
    with torch.no_grad():
        saved = [t.numpy() for t in openpose_port.forward(openpose_port.he_state_dict(), x)]
    np.testing.assert_allclose(saved[3], g["paf"], rtol=0, atol=1e-5)
    np.testing.assert_allclose(saved[5], g["heat"], rtol=0, atol=1e-5)
    for i, m in enumerate(saved):
        np.testing.assert_allclose(m.reshape(-1)[::13][:64], g["stage_sample"][i], rtol=0, atol=1e-5)
        if "maps_%d" % i in g:
            np.testing.assert_allclose(m, g["maps_%d" % i], rtol=0, atol=1e-5)


@pytest.mark.parametrize("name", ["openpose_64", "openpose_368"])
def test_exact_oracle_matches_the_reference_golden(built, name):
    g = golden(name)
    hw = int(g["hw"])
    x = torch.rand((1, 3, hw, hw), generator=torch.Generator().manual_seed(int(g["seed"]))) - 0.5
    saved = openpose_port.forward_exact(openpose_port.he_state_dict(), x.numpy())
    np.testing.assert_allclose(saved[3], g["paf"], rtol=0, atol=1e-4)
    np.testing.assert_allclose(saved[5], g["heat"], rtol=0, atol=1e-4)
    for i, m in enumerate(saved):
        if "maps_%d" % i in g:
            np.testing.assert_allclose(m, g["maps_%d" % i], rtol=0, atol=1e-4)


@pytest.mark.parametrize("layout", LAYOUTS, ids=["%d-%d" % lay for lay in LAYOUTS])
def test_oracles_match_the_reference_golden_at_other_layouts(built, layout):
    """forward and forward_exact of OpenPose_Model(l2, l1) against every saved map of the unmodified module."""
    l2, l1 = layout
    g = golden("openpose_%d_%d_64" % layout)
    assert (int(g["l2"]), int(g["l1"])) == layout
    x = torch.rand((1, 3, 64, 64), generator=torch.Generator().manual_seed(int(g["seed"]))) - 0.5
    sd = openpose_port.he_state_dict(l2, l1)
    with torch.no_grad():
        saved = [t.numpy() for t in openpose_port.forward(sd, x, l2, l1)]
    exact = openpose_port.forward_exact(sd, x.numpy(), l2, l1)
    assert len(saved) == len(exact) == l2 + l1 == len([k for k in g.files if k.startswith("maps_")])
    for i in range(l2 + l1):
        np.testing.assert_allclose(saved[i], g["maps_%d" % i], rtol=0, atol=1e-5, err_msg="forward map %d" % i)
        np.testing.assert_allclose(exact[i], g["maps_%d" % i], rtol=0, atol=1e-4, err_msg="forward_exact map %d" % i)


def test_prelu_is_one_multiply_after_the_bias():
    v = np.array([[[[-2.0, -0.0, 0.0, 3.0, -1e-30]]]], np.float32)
    s = np.array([-0.5, 1.25, 0.3, 0.7, 1.5], np.float32)
    out = openpose_port.prelu_f32(v, s)
    np.testing.assert_array_equal(out, np.array([[[[1.0, -0.0, 0.0, 3.0, np.float32(-1.5e-30)]]]], np.float32))
    assert np.signbit(out[0, 0, 0, 1])      # slope * (-0) is -0, not +0: a pad lane must not be written this way
