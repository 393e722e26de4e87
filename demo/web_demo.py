#!/usr/bin/env python
"""Camera front-end on the H100 path: the flow and command line of the reference's demo/web_demo.py (:29-71) - camera 0,
every frame through the network and the post-processing, the drawn frame shown until `q` is pressed - with the capture of
frame i+1 overlapped with the inference of frame i (streaming.PoseStream, batch 1).  Extras: `--source` (a camera index
or a file), `--no-window` (headless: count frames instead of cv2.imshow), `--max-frames`, `--synthetic-weights`.
Run from the repo root."""
import argparse
import os
import sys
import time

sys.path.append('.')
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import cv2  # noqa: E402
import torch  # noqa: E402

from lib.config import cfg, update_config  # noqa: E402
from video_demo import load_model  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--cfg', help='experiment configure file name', default='./experiments/vgg19_368x368_sgd.yaml', type=str)
    ap.add_argument('--weight', type=str, default='pose_model.pth')
    ap.add_argument('--synthetic-weights', action='store_true')
    ap.add_argument('--source', type=str, default='0')
    ap.add_argument('--no-window', action='store_true')
    ap.add_argument('--max-frames', type=int, default=0)
    ap.add_argument('opts', help="Modify config options using the command-line", default=None, nargs=argparse.REMAINDER)
    args = ap.parse_args()
    update_config(cfg, args)
    import importlib
    import _b200_alias
    streaming = importlib.import_module(_b200_alias.PKG + ".streaming")

    model = load_model(args)
    cap = cv2.VideoCapture(int(args.source) if args.source.isdigit() else args.source)
    t0, n = time.time(), 0
    with torch.no_grad():
        for _, humans, drawn in streaming.PoseStream(model, streaming.frames_of(cap, None, args.max_frames or None), batch=1):
            n += 1
            if args.no_window:
                continue
            cv2.imshow('Video', drawn)
            if cv2.waitKey(1) & 0xFF == ord('q'):
                break
    cap.release()
    if not args.no_window:
        cv2.destroyAllWindows()
    print("%d frames, %.1f frames/s" % (n, n / max(time.time() - t0, 1e-9)))


if __name__ == "__main__":
    main()
