"""Counterpart of /root/reference/evaluate/evaluation.py: load a checkpoint into the rtpose VGG19 model and run the
COCO keypoint evaluation on the H100 path.  The reference hard-codes its paths (evaluation.py:12,31); here they are
arguments with the same defaults.  Run from the repository root:  python -m evaluate.evaluation --weight ... """
import argparse
from collections import OrderedDict

import torch

from ..lib.network.rtpose_vgg import get_model
from .coco_eval import run_eval


def load_model(weight_name):
    """evaluation.py:12-26: a Lightning checkpoint whose keys carry a 6-character 'model.' prefix."""
    state_dict = torch.load(weight_name, map_location="cpu")['state_dict']
    model = get_model(trunk='vgg19')
    model.load_state_dict(OrderedDict((k[6:], v) for k, v in state_dict.items()))
    model.eval()
    model.float()
    return model.cuda()


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument('--weight', default='/data/rtpose/rtpose_lr001/1/_ckpt_epoch_82.ckpt')
    ap.add_argument('--image-dir', default='/data/coco/images/val2017')
    ap.add_argument('--anno-file', default='/data/coco/annotations/person_keypoints_val2017.json')
    ap.add_argument('--vis-dir', default='/data/coco/images/vis_val2017')
    ap.add_argument('--preprocess', default='vgg', choices=['rtpose', 'vgg', 'inception', 'ssd'])
    a = ap.parse_args(argv)
    with torch.no_grad():
        model = load_model(a.weight)
        return run_eval(image_dir=a.image_dir, anno_file=a.anno_file, vis_dir=a.vis_dir, model=model,
                        preprocess=a.preprocess)


if __name__ == "__main__":
    main()
