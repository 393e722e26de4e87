"""BASELINE.json north_star: "... so evaluate/evaluation.py and demo/picture_demo.py run unmodified".

This repo's demo with the reference's command line (no extra flags), on the shipped 674x712 stand-in for
./readme/ski.jpg and a pose_model.pth written by the test."""
import os
import subprocess
import sys

import pytest
import torch

from conftest import ROOT


@pytest.mark.gpu
def test_demo_with_the_reference_command_line(built, he_sd):
    """`python demo/picture_demo.py` from the repo root, no flags: reads ./experiments/vgg19_368x368_sgd.yaml,
    pose_model.pth and ./readme/ski.jpg, writes result.png - the reference demo's contract (:30-65)."""
    weight, result = os.path.join(ROOT, "pose_model.pth"), os.path.join(ROOT, "result.png")
    torch.save(he_sd, weight)
    try:
        if os.path.exists(result):
            os.remove(result)
        r = subprocess.run([sys.executable, os.path.join("demo", "picture_demo.py")], cwd=ROOT, stdout=subprocess.PIPE,
                           stderr=subprocess.STDOUT, text=True, timeout=600)
        print(r.stdout[-2000:])
        assert r.returncode == 0 and os.path.exists(result)
        assert abs(float(r.stdout.split()[0]) - 368.0 / 674.0) < 1e-12        # print(im_scale)
        assert "humans; maps (46, 49, 19) (46, 49, 38)" in r.stdout           # 674x712 -> 368x389 -> padded 368x392
    finally:
        for f in (weight, result):
            if os.path.exists(f):
                os.remove(f)
