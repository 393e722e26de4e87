#!/usr/bin/env python
"""Mixed frame sizes through PoseEngine.infer_images: a fixed, seeded list of raw frames like a photo collection's (both
orientations, five aspect ratios, many distinct padded shapes) with batch_cap 32; one step = one pass over the list.
Prints ONE JSON line: frames/s (wall clock, host frames in, person rows out) and kernel launches per frame.

  python tools/bench_mixed.py --steps K --warmup W [--mode bf16|bf16x3|fp32|fp8] [--flip] [--scales S [S ...]]
                              [--dump-outputs DIR]

--scales 0.5 1.0 1.5 2.0 runs multi-scale test-time averaging around the 368 base size (passed to infer_images).
--dump-outputs DIR writes the last step's person rows (float32 [k, 73], all images in list order) and the per-image
counts as DIR/humans.npy and DIR/humans_per_image.npy, so that two builds can be compared row for row.  The script
only calls PoseEngine.infer_images_arrays, so it also runs against builds that predate ragged batches."""
import argparse
import importlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import _b200_alias  # noqa: E402

FRAMES = 96
ASPECTS = (1.0, 5 / 4, 4 / 3, 3 / 2, 16 / 9)
DEST = 368


def mixed_frames(count=FRAMES, seed=2024):
    """Raw uint8 BGR frames: short side 240 .. 480 px, one of five aspect ratios with a few per cent of jitter, 70 %
    landscape - so that crop_with_factor gives many distinct padded shapes."""
    rng = np.random.default_rng(seed)
    frames = []
    for _ in range(count):
        short = int(rng.integers(240, 481))
        long_ = max(short, int(round(short * ASPECTS[int(rng.integers(len(ASPECTS)))] * rng.uniform(0.97, 1.03))))
        h, w = (short, long_) if rng.random() < 0.7 else (long_, short)
        frames.append(rng.integers(0, 256, (h, w, 3), dtype=np.uint8))
    return frames


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--mode", default="bf16", choices=["bf16", "bf16x3", "fp32", "fp8"])
    ap.add_argument("--flip", action="store_true")
    ap.add_argument("--scales", type=float, nargs="+", default=None, metavar="S")
    ap.add_argument("--dump-outputs", default="", metavar="DIR")
    args = ap.parse_args()
    import torch
    _b200_alias.load_package()
    engine = importlib.import_module(_b200_alias.PKG + ".engine")
    nat = importlib.import_module(_b200_alias.PKG + "._native")
    syn = importlib.import_module(_b200_alias.PKG + ".synthetic")
    # random-weight maps are noise: a frame can assemble more than a thousand persons
    eng = engine.PoseEngine(syn.he_state_arrays(1234), 0, mode=args.mode, batch_cap=32, peak_cap=1024, human_cap=4096)
    frames = mixed_frames()
    pads = {nat.crop_geometry(f.shape[0], f.shape[1], DEST, 8)[2] for f in frames}
    for _ in range(max(args.warmup, 1)):
        eng.infer_images_arrays(frames, dest_size=DEST, flip=args.flip, scales=args.scales)
    torch.cuda.synchronize()
    l0 = nat.launch_count()
    t0 = time.perf_counter()
    for _ in range(args.steps):
        out = eng.infer_images_arrays(frames, dest_size=DEST, flip=args.flip, scales=args.scales)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    n = len(frames) * args.steps
    launches = nat.launch_count() - l0
    if args.dump_outputs:
        os.makedirs(args.dump_outputs, exist_ok=True)
        np.save(os.path.join(args.dump_outputs, "humans.npy"),
                np.concatenate([o.reshape(-1, nat.HUMAN_FLOATS) for o in out]).astype(np.float32))
        np.save(os.path.join(args.dump_outputs, "humans_per_image.npy"), np.array([len(o) for o in out], np.float64))
    print(json.dumps({
        "metric": "frames/sec, mixed frame sizes through PoseEngine.infer_images", "value": round(n / dt, 2),
        "unit": "frames/s", "steps": args.steps, "warmup": args.warmup, "ms_per_step": round(dt * 1e3 / args.steps, 3),
        "higher_is_better": True, "launches_per_frame": round(launches / n, 2), "gpu_launches": int(launches),
        "gpu": torch.cuda.get_device_properties(0).name,
        "config": {"frames": len(frames), "distinct_padded_shapes": len(pads), "dest_size": DEST, "batch_cap": 32,
                   "mode": args.mode, "flip": bool(args.flip), "scales": args.scales,
                   "input": "host uint8 BGR frames; crop_with_factor, network and post-processing on the device; "
                            "results read back per batch (wall clock)"}}))


if __name__ == "__main__":
    main()
