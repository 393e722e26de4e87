"""CPU: the stage-count surface - the C declaration and export, and rtpose_model.stages validation before any device
work (tests/test_gpu_stages.py runs the stage counts on the GPU)."""
import ctypes
import os

import pytest
import torch

from conftest import ROOT, pkg_module


def test_set_stages_is_declared_and_exported(built):
    with open(os.path.join(ROOT, "include", "b200pose.h")) as f:
        header = f.read()
    assert "int b200pose_net_set_stages(b200pose_net* net, int stages);" in header
    nat = pkg_module("_native")
    assert "b200pose_net_set_stages" in nat.EXPORTED
    assert hasattr(ctypes.CDLL(nat.LIB_PATH), "b200pose_net_set_stages")
    assert nat.lib().b200pose_net_set_stages(None, 3) != 0
    assert b"null net" in nat.lib().b200pose_last_error()


def test_stages_default_and_environment(built, monkeypatch):
    rtpose = pkg_module("lib.network.rtpose_vgg")
    monkeypatch.delenv("B200POSE_STAGES", raising=False)
    assert rtpose.get_model("vgg19").stages == 6
    monkeypatch.setenv("B200POSE_STAGES", "2")
    assert rtpose.get_model("vgg19").stages == 2


@pytest.mark.parametrize("bad", [0, 7, -1, 2.5, True, "3", None])
def test_bad_stages_raise_before_any_device_work(built, bad):
    """Every entry point of the module checks the stage count first: a CPU model and a CPU tensor would otherwise fail
    for lack of a device, so ValueError here shows that nothing reached the device."""
    import numpy as np
    from evaluate.coco_eval import get_outputs
    model = pkg_module("lib.network.rtpose_vgg").get_model("vgg19")
    model.stages = bad
    with pytest.raises(ValueError, match="stages"):
        model(torch.zeros((1, 3, 8, 8)))
    with pytest.raises(ValueError, match="stages"):
        model.pose_engine()
    with pytest.raises(ValueError, match="stages"):
        get_outputs(np.zeros((16, 16, 3), np.uint8), model, "rtpose")
    with pytest.raises(ValueError, match="stages"):
        torch.nn.DataParallel(model)(torch.zeros((1, 3, 8, 8)))
