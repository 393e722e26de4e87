#!/usr/bin/env python
"""Single-picture demo on the H100 path, with the command line, the files and the flow of the reference's
demo/picture_demo.py (:30-65): `--cfg` (default ./experiments/vgg19_368x368_sgd.yaml), `--weight` (default
pose_model.pth), trailing config overrides; reads ./readme/ski.jpg, prints im_scale, writes result.png.  Run from the
repo root, like the reference.  The reference's own script runs unmodified against this repo as well (its imports are
the module paths this repo provides; tests/test_reference_scripts.py executes it); this counterpart only adds optional
switches for machines without a checkpoint (`--synthetic-weights`), other pictures and the arithmetic mode."""
import argparse
import os
import sys

sys.path.append('.')
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import cv2  # noqa: E402
import torch  # noqa: E402

from evaluate.coco_eval import get_outputs  # noqa: E402
from lib.config import cfg, update_config  # noqa: E402
from lib.network.rtpose_vgg import get_model  # noqa: E402
from lib.utils.common import draw_humans  # noqa: E402
from lib.utils.paf_to_pose import paf_to_pose_cpp  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--cfg', help='experiment configure file name', default='./experiments/vgg19_368x368_sgd.yaml', type=str)
    ap.add_argument('--weight', type=str, default='pose_model.pth')
    ap.add_argument('--synthetic-weights', action='store_true',
                    help='no checkpoint at hand: seeded random-init weights (the maps are noise, the plumbing is real)')
    ap.add_argument('--image', type=str, default='./readme/ski.jpg')
    ap.add_argument('--precision', default=None, choices=['bf16', 'bf16x3', 'fp32'])
    ap.add_argument('--out', default='result.png')
    ap.add_argument('opts', help="Modify config options using the command-line", default=None, nargs=argparse.REMAINDER)
    args = ap.parse_args()
    update_config(cfg, args)

    model = get_model('vgg19')
    if args.synthetic_weights:
        import importlib
        import _b200_alias
        arrays = importlib.import_module(_b200_alias.PKG + ".synthetic").he_state_arrays(1234)
        model.load_state_dict({k: torch.from_numpy(a) for k, a in zip(model.state_dict(), arrays)})
    else:
        model.load_state_dict(torch.load(args.weight))
    model = torch.nn.DataParallel(model).cuda()
    model.float()
    model.eval()
    if args.precision:
        model.module.precision = args.precision

    ori = cv2.imread(args.image)      # B, G, R order
    if ori is None:
        raise SystemExit("cannot read %s" % args.image)
    with torch.no_grad():
        paf, heatmap, im_scale = get_outputs(ori, model, 'rtpose')
    print(im_scale)
    humans = paf_to_pose_cpp(heatmap, paf, cfg)
    print('%d humans; maps %s %s' % (len(humans), heatmap.shape, paf.shape))
    cv2.imwrite(args.out, draw_humans(ori, humans))


if __name__ == '__main__':
    main()
