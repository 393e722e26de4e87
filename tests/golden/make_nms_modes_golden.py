"""Generates tests/golden/nms_modes.npz by running the UNMODIFIED reference's NMS and paf_to_pose_cpp (its own
pafprocess.cpp compiled into oracle/_ref/, see make_golden.py for the import shims) on the scenarios of
tests/nms_modes_port.py: per scenario, factor f in GOLDEN_FACTORS and mode (cubic, gauss, none), the joint list of
NMS(heat, upsampFactor=f, bool_refine_center, bool_gaussian_filt) as float32 [P, 5]; for the cubic mode also the persons
of paf_to_pose_cpp with cfg.MODEL.DOWNSAMPLE = f, rows [k, 1 + 18 x 3] like the post_*.npz fixtures.  As for the
existing fixtures, OpenCV keeps this build's default (IPP on, whose cubic arithmetic differs from OpenCV's own by a few
ulps) on the stick-figure maps, and runs with IPP off on the adversarial post_edges maps, whose plateaus and ties turn
any such difference into a different arg-max.
Usage:  python tests/golden/make_nms_modes_golden.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import make_golden  # noqa: E402
import nms_modes_port as nmp  # noqa: E402


def main():
    _, ref_p2p, _, cfg = make_golden.import_reference()
    assert cfg.TEST.THRESH_HEATMAP == nmp.GOLDEN_THRESH
    out, ins = {}, []
    down = cfg.MODEL.DOWNSAMPLE
    import cv2
    use_ipp = cv2.ipp.useIPP()
    try:
        for name, (heat, paf) in nmp.golden_scenarios().items():
            cv2.ipp.setUseIPP(use_ipp and name in ("p3", "p30"))
            ins += [heat, paf]
            for f in nmp.GOLDEN_FACTORS:
                cfg.MODEL.DOWNSAMPLE = f
                for mode, (refine, gauss) in nmp.MODES.items():
                    key = nmp.golden_key(name, f, mode)
                    per_joint = ref_p2p.NMS(heat, upsampFactor=f, bool_refine_center=refine, bool_gaussian_filt=gauss,
                                            config=cfg)
                    out[key + "_joint_list"] = np.array([tuple(p) + (j,) for j, peaks in enumerate(per_joint)
                                                         for p in peaks]).astype(np.float32).reshape(-1, 5)
                    if mode != "cubic":
                        continue
                    humans = ref_p2p.paf_to_pose_cpp(heat, paf, cfg)
                    rows = np.full((len(humans), 1 + 18 * 3), -1.0, np.float64)
                    for i, hm in enumerate(humans):
                        rows[i, 0] = hm.score
                        for p, bp in hm.body_parts.items():
                            rows[i, 1 + 3 * p: 4 + 3 * p] = (bp.x, bp.y, bp.score)
                    out[key + "_humans"] = rows
                print(name, "f", f, "peaks", len(out[key + "_joint_list"]))
    finally:
        cfg.MODEL.DOWNSAMPLE = down
        cv2.ipp.setUseIPP(use_ipp)
    np.savez_compressed(os.path.join(HERE, "nms_modes.npz"), in_digest=make_golden.digest(*ins), **out)


if __name__ == "__main__":
    main()
