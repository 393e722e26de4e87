"""Generates the OpenPose_Model fixtures by running the UNMODIFIED reference module
(/root/reference/lib/network/openpose.py, imported from its file; it needs nothing but torch) on the CPU.
Usage:  python tests/golden/make_openpose_golden.py

  * openpose_spec.json       : the module's state_dict keys and shapes for OpenPose_Model(l2, l1, 38, 19), (l2, l1) in
                               (4, 2), (1, 1), (5, 3);
  * openpose_64.npz / _368.npz: OpenPose_Model(4, 2, 38, 19) with tests/openpose_port.he_state_dict() loaded (strict),
                               on a seeded input: every saved_for_loss map at 64 x 64; the final PAF / heat map and
                               per-map statistics and samples at 368 x 368.
"""
import importlib.util
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
REF = "/root/reference/lib/network/openpose.py"
OUT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import openpose_port  # noqa: E402  (needs the built library: the weights come from the package's table)
from golden.make_golden import digest  # noqa: E402

ARCHS = ((4, 2), (1, 1), (5, 3))


def main():
    spec = importlib.util.spec_from_file_location("ref_openpose", REF)
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    shapes = {}
    for l2, l1 in ARCHS:
        m = ref.OpenPose_Model(l2, l1, 38, 19)
        shapes["%d,%d" % (l2, l1)] = [[k, list(v.shape)] for k, v in m.state_dict().items()]
    with open(os.path.join(OUT, "openpose_spec.json"), "w") as f:
        json.dump(shapes, f, separators=(",", ":"))
    model = ref.OpenPose_Model(4, 2, 38, 19)
    model.load_state_dict(openpose_port.he_state_dict(4, 2), strict=True)
    model.eval()
    for name, hw, seed in (("openpose_64", 64, 21), ("openpose_368", 368, 2368)):
        g = torch.Generator().manual_seed(seed)
        x = torch.rand((1, 3, hw, hw), generator=g) - 0.5
        with torch.no_grad():
            _, (paf_ret, heat_ret) = model(x)
        saved = [t.numpy() for t in paf_ret + heat_ret]
        extra = {"maps_%d" % i: m for i, m in enumerate(saved)} if hw == 64 else {}
        np.savez_compressed(os.path.join(OUT, name + ".npz"), seed=seed, hw=hw, x_digest=digest(x.numpy()),
                            paf=saved[3], heat=saved[5],
                            stage_absmax=np.array([float(np.abs(m).max()) for m in saved]),
                            stage_mean=np.array([float(m.astype(np.float64).mean()) for m in saved]),
                            stage_sample=np.stack([m.reshape(-1)[::13][:64] for m in saved]), **extra)
        print(name, "paf absmax %.3f heat absmax %.3f" % (np.abs(saved[3]).max(), np.abs(saved[5]).max()))


if __name__ == "__main__":
    main()
