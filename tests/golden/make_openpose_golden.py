"""Generates the OpenPose_Model fixtures by running the UNMODIFIED reference module
(/root/reference/lib/network/openpose.py, imported from its file; it needs nothing but torch) on the CPU.
Usage:  python tests/golden/make_openpose_golden.py

  * openpose_spec.json       : the module's state_dict keys and shapes for OpenPose_Model(l2, l1, 38, 19), (l2, l1) in
                               (4, 2), (1, 1), (5, 3) and the LAYOUTS below;
  * openpose_64.npz / _368.npz: OpenPose_Model(4, 2, 38, 19) with tests/openpose_port.he_state_dict() loaded (strict),
                               on a seeded input: every saved_for_loss map at 64 x 64; the final PAF / heat map and
                               per-map statistics and samples at 368 x 368;
  * openpose_<l2>_<l1>_64.npz : every saved_for_loss map of OpenPose_Model(l2, l1, 38, 19) at 64 x 64, for the LAYOUTS,
                               with he_state_dict(l2, l1) loaded (strict).  The module's forward ends with
                               `paf_ret[-2], heat_ret[-2]`, which raises IndexError when l2 = 1 or l1 = 1, so the maps
                               are taken from the module's own feature_extractor, l2_stages and l1_stages, run in the
                               order forward runs them (saved_maps below); where forward returns, the two agree.
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

LAYOUTS = ((1, 1), (1, 11), (11, 1), (2, 3), (6, 6))
ARCHS = ((4, 2), (1, 1), (5, 3)) + LAYOUTS[1:]


def saved_maps(model, x):
    """saved_for_loss of OpenPose_Model.forward (paf_ret + heat_ret), from the module's own stages in forward's order."""
    features = model.feature_extractor(x)
    paf_ret, heat_ret = [], []
    x_in = features
    for stage in model.l2_stages:
        paf_pred = stage(x_in)
        x_in = torch.cat([features, paf_pred], 1)
        paf_ret.append(paf_pred)
    for stage in model.l1_stages:
        heat_pred = stage(x_in)
        x_in = torch.cat([features, heat_pred, paf_pred], 1)
        heat_ret.append(heat_pred)
    return paf_ret + heat_ret


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
    for l2, l1 in LAYOUTS:
        model = ref.OpenPose_Model(l2, l1, 38, 19)
        model.load_state_dict(openpose_port.he_state_dict(l2, l1), strict=True)
        model.eval()
        seed, hw = 64 + 12 * l2 + l1, 64
        x = torch.rand((1, 3, hw, hw), generator=torch.Generator().manual_seed(seed)) - 0.5
        with torch.no_grad():
            saved = [t.numpy() for t in saved_maps(model, x)]
            if l2 > 1 and l1 > 1:
                _, (paf_ret, heat_ret) = model(x)
                assert all(np.array_equal(a, b.numpy()) for a, b in zip(saved, paf_ret + heat_ret))
        name = "openpose_%d_%d_64" % (l2, l1)
        np.savez_compressed(os.path.join(OUT, name + ".npz"), seed=seed, hw=hw, l2=l2, l1=l1, x_digest=digest(x.numpy()),
                            stage_absmax=np.array([float(np.abs(m).max()) for m in saved]),
                            **{"maps_%d" % i: m for i, m in enumerate(saved)})
        print(name, "stage absmax", " ".join("%.3f" % float(np.abs(m).max()) for m in saved))


if __name__ == "__main__":
    main()
