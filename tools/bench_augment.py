#!/usr/bin/env python
"""Training batches on the device (DESIGN.md 2.20): PoseEngine.training_batch at batch B (default 72, the reference's
--batch-size) of COCO-like sources (640 x 480, 480 x 640, 640 x 427, 500 x 375, 3 persons each) at edge 368, CUDA
events around whole calls on the current stream (draws, upload, augmentation kernels, the JPEG round trip of the
samples that draw it, targets); samples per second.  Before timing, every sample of the first batch is checked
against the host build of csrc/aug_core.h (tests/aug_check.py).  With --reference DIR also the reference's own
preprocess + image_transform_train per sample on one host CPU core.  The card's name and power limit are read in the
same call.  One JSON line.

  python tools/bench_augment.py [--batch B] [--runs R] [--reference DIR]"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _b200_alias  # noqa: E402

SIZES = [(480, 640), (640, 480), (427, 640), (375, 500)]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def sources(batch, seed=0):
    rs = np.random.RandomState(seed)
    ims, kps = [], []
    for i in range(batch):
        h, w = SIZES[i % len(SIZES)]
        y, x = np.mgrid[0:h, 0:w]
        im = np.stack([128 + 90 * np.sin(x / 17.0 + i), 128 + 90 * np.cos(y / 11.0), 128 + 60 * np.sin((x + y) / 23.0)], -1)
        ims.append(np.clip(im + rs.normal(0, 20, im.shape), 0, 255).astype(np.uint8))
        k = np.zeros((3, 17, 3), np.float32)
        k[:, :, 0] = rs.uniform(0, w, (3, 17))
        k[:, :, 1] = rs.uniform(0, h, (3, 17))
        k[:, :, 2] = rs.choice([0, 1, 2], (3, 17))
        kps.append(k)
    return ims, kps


def check(pe, core, ims, kps, edge):
    import aug_check as ac
    import torch
    eng = importlib.import_module(_b200_alias.PKG + ".engine")
    params = eng.augment_params([im.shape[:2] for im in ims], torch.Generator().manual_seed(1), edge)
    x, _, _ = pe.training_batch(ims, kps, edge=edge, params=params)
    x = x.cpu().numpy()
    for i, (im, p) in enumerate(zip(ims, params)):
        g = {"src": np.ascontiguousarray(im[:, :, ::-1]), "edge": edge}
        want = ac.to_tensor(ac.colour_stages(core, g, p), p)
        assert np.array_equal(ac.bits(x[i]), ac.bits(want)), "sample %d differs from the host core" % i
    return sum(p["jpeg"] for p in params)


def reference_per_sample(ref, ims, runs):
    import PIL.Image
    import torch
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import make_gt_golden
    make_gt_golden.import_reference(ref)
    from lib.datasets import transforms as tr
    pre = tr.Compose([tr.Normalize(), tr.RandomApply(tr.HFlip(), 0.5), tr.RescaleRelative(), tr.Crop(368),
                      tr.CenterPad(368)])
    torch.set_num_threads(1)
    pils = [PIL.Image.fromarray(np.ascontiguousarray(im[:, :, ::-1])) for im in ims]
    t0 = time.perf_counter()
    n = 0
    for _ in range(runs):
        for p in pils:
            image, _, _ = pre(p, [], None)
            tr.image_transform_train(image)
            n += 1
    return (time.perf_counter() - t0) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=72)
    ap.add_argument("--runs", type=int, default=20)
    ap.add_argument("--edge", type=int, default=368)
    ap.add_argument("--reference", default=None)
    a = ap.parse_args()
    import torch
    _b200_alias.load_package()
    eng = importlib.import_module(_b200_alias.PKG + ".engine")
    import aug_check as ac
    from oracle import net_port
    if not torch.cuda.is_available():
        raise SystemExit("bench_augment needs a GPU")
    core = ac.compile_core(os.path.join(ROOT, "build", "libaugcore_bench.so"))
    net = eng.NativeNet(0)
    net.load_state_dict_arrays([v.numpy() for v in net_port.he_state_dict(1234).values()])
    pe = eng.PoseEngine.from_net(net, mode="bf16", batch_cap=a.batch)
    ims, kps = sources(a.batch)
    jpeg_checked = check(pe, core, ims, kps, a.edge)
    gen = torch.Generator().manual_seed(2)
    for _ in range(3):
        pe.training_batch(ims, kps, gen, a.edge)
    torch.cuda.synchronize()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(a.runs):
        pe.training_batch(ims, kps, gen, a.edge)
    stop.record()
    torch.cuda.synchronize()
    ms = start.elapsed_time(stop) / a.runs
    out = {"card": card(), "batch": a.batch, "edge": a.edge, "sources": SIZES, "runs": a.runs,
           "checked_samples": a.batch, "checked_jpeg_samples": int(jpeg_checked),
           "training_batch_ms": round(ms, 3), "samples_per_s": round(a.batch * 1000.0 / ms, 1)}
    if a.reference:
        s = reference_per_sample(a.reference, ims[:8], 2)
        out["reference_cpu_ms_per_sample_1_core"] = round(1000 * s, 2)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
