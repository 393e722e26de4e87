#!/usr/bin/env python
"""Video-file front-end on the H100 path: the flow and command line of the reference's video_demo.py (:47-125) - `--cfg`,
`--weight`, trailing config overrides, the video path asked on stdin, every frame drawn into output.avi - with the frames
batched and pipelined through the fused engine (streaming.PoseStream) instead of one get_outputs + paf_to_pose_cpp per
frame.  Extras: `--video` (skip the prompt), `--out`, `--batch`, `--synthetic-weights`, `--max-frames`.
Run from the repo root."""
import argparse
import os
import sys
import time

sys.path.append('.')
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import cv2  # noqa: E402
import torch  # noqa: E402

from lib.config import cfg, update_config  # noqa: E402
from lib.network.rtpose_vgg import get_model  # noqa: E402


def check_rotation(path):
    """video_demo.py:27-42: the container's rotate tag, when the optional ffmpeg module is there to read it."""
    try:
        import ffmpeg
        rot = int(ffmpeg.probe(path)['streams'][0]['tags']['rotate'])
    except Exception:
        return None
    return {90: cv2.ROTATE_90_CLOCKWISE, 180: cv2.ROTATE_180, 270: cv2.ROTATE_90_COUNTERCLOCKWISE}.get(rot)


def load_model(args):
    model = get_model('vgg19')
    if args.synthetic_weights:
        import importlib
        import _b200_alias
        arrays = importlib.import_module(_b200_alias.PKG + ".synthetic").he_state_arrays(1234)
        model.load_state_dict({k: torch.from_numpy(a) for k, a in zip(model.state_dict(), arrays)})
    else:
        model.load_state_dict(torch.load(args.weight))
    model.cuda()
    model.float()
    model.eval()
    return model


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--cfg', help='experiment configure file name', default='./experiments/vgg19_368x368_sgd.yaml', type=str)
    ap.add_argument('--weight', type=str, default='pose_model.pth')
    ap.add_argument('--synthetic-weights', action='store_true')
    ap.add_argument('--video', type=str, default='')
    ap.add_argument('--out', type=str, default='output.avi')
    ap.add_argument('--batch', type=int, default=8)
    ap.add_argument('--max-frames', type=int, default=0)
    ap.add_argument('opts', help="Modify config options using the command-line", default=None, nargs=argparse.REMAINDER)
    args = ap.parse_args()
    update_config(cfg, args)
    import importlib
    import _b200_alias
    streaming = importlib.import_module(_b200_alias.PKG + ".streaming")

    model = load_model(args)
    path = args.video or input("Enter video path")
    cap = cv2.VideoCapture(path)
    ok, first = cap.read()
    if not ok:
        raise SystemExit("cannot read %s" % path)
    rotate = check_rotation(path)
    if rotate is not None:
        first = cv2.rotate(first, rotate)
    shape = tuple(first.shape[1::-1])
    print("Shape of image is ", shape)
    cap.release()
    cap = cv2.VideoCapture(path)
    out = cv2.VideoWriter(args.out, cv2.VideoWriter_fourcc(*'XVID'), 20.0, shape)
    t0, n, persons = time.time(), 0, 0
    with torch.no_grad():
        for _, humans, drawn in streaming.PoseStream(model, streaming.frames_of(cap, rotate, args.max_frames or None),
                                                     batch=args.batch):
            out.write(drawn)
            n += 1
            persons += len(humans)
            if n % 50 == 0:
                print(n, "frames processed")
    cap.release()
    out.release()
    print("%d frames, %d persons, %.1f frames/s -> %s" % (n, persons, n / max(time.time() - t0, 1e-9), args.out))


if __name__ == "__main__":
    main()
