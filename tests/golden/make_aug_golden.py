"""Generates the training-batch fixtures tests/golden/aug_*.npz and tests/golden/aug_cube.json by running the UNMODIFIED
reference loader's per-sample path on synthetic frames.  Usage:

    python tests/golden/make_aug_golden.py <reference checkout>

Per sample, with torch.manual_seed(seed): the reference's train preprocess (transforms.Compose([Normalize(),
RandomApply(HFlip(), 0.5), RescaleRelative(), Crop(edge), CenterPad(edge)]), train/train_VGG19.py:124-130), the
transforms of transforms.image_transform_train run one by one so that the PIL image ToTensor receives can be recorded,
utils.mask_valid_area and CocoKeypoints.get_ground_truth at input_x = input_y = edge (imported with the stubs of
make_gt_golden.py).  Each fixture holds `src` (RGB [h, w, 3], the PIL image the loader opens), `kp` ([P, 17, 3]
float32), `seed`, `edge`, the meta (`hflip`, `scale`, `offset`, `valid_area`), `u8` (RGB [edge, edge, 3], the image
after ColorJitter, the JPEG round trip and RandomGrayscale), `image` (the final float32 tensor [3, edge, edge]),
`kp_out` (the augmented keypoints, in the dtype the reference leaves them), `heat` and `paf` (get_ground_truth's maps,
transposed and cast to float32 as single_image_processing does).

aug_cube.json: SHA-256 of Pillow's output over all 2^24 RGB colours (a 4096 x 4096 image, colour r << 16 | g << 8 | b
at pixel index) for ImageEnhance.Brightness and Color at several factors, torchvision's adjust_hue at several
factors, Image.blend against a constant grey (Contrast's blend) at several means and factors, and convert('L').
"""
import hashlib
import json
import os
import sys

import numpy as np

OUT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, OUT)
sys.path.insert(0, os.path.dirname(os.path.dirname(OUT)))

BRIGHTNESS = SATURATION = (0.9, 0.95, 1.0, 1.05, 1.1)
HUE = (-0.5, -0.1, -0.05, -0.003, 0.0, 0.003, 0.05, 0.1, 0.5)
CONTRAST = ((0, 0.9), (37, 1.1), (128, 0.9), (128, 1.1), (201, 0.95), (255, 1.1))


def f32(v):
    return float(np.float32(v))


def cube_image():
    from PIL import Image
    c = np.arange(1 << 24, dtype=np.uint32)
    rgb = np.stack([(c >> 16) & 255, (c >> 8) & 255, c & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    return Image.fromarray(rgb)


def digest(im):
    return hashlib.sha256(np.ascontiguousarray(np.asarray(im)).tobytes()).hexdigest()


def cube_digests():
    from PIL import Image, ImageEnhance
    import torchvision.transforms.functional as F
    im = cube_image()
    out = {"brightness": {}, "saturation": {}, "hue": {}, "contrast": {}}
    for f in BRIGHTNESS:
        out["brightness"][repr(f32(f))] = digest(ImageEnhance.Brightness(im).enhance(f32(f)))
    for f in SATURATION:
        out["saturation"][repr(f32(f))] = digest(ImageEnhance.Color(im).enhance(f32(f)))
    for f in HUE:
        out["hue"][repr(f32(f))] = digest(F.adjust_hue(im, f32(f)))
    for m, f in CONTRAST:
        out["contrast"]["%d %r" % (m, f32(f))] = digest(Image.blend(Image.new("RGB", im.size, (m, m, m)), im, f32(f)))
    out["L"] = digest(im.convert("L"))
    return out


def frame(rs, h, w, kind):
    """Synthetic RGB frames: smooth colour fields with texture; 'saturated' pushes channels to 0 / 255, 'grey' has
    r = g = b (hue and saturation leave it), 'flat' is nearly one colour, 'blocks' is 48 x 48 squares of random
    colours (sharp edges for the resampling filter, and few enough distinct bytes that the COCO-sized fixtures stay
    small)."""
    if kind == "blocks":
        small = rs.randint(0, 256, (h // 48 + 1, w // 48 + 1, 3)).astype(np.uint8)
        return np.ascontiguousarray(np.repeat(np.repeat(small, 48, 0), 48, 1)[:h, :w])
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    base = np.stack([128 + 100 * np.sin(x / (7 + 13 * rs.rand()) + rs.rand() * 6),
                     128 + 100 * np.cos(y / (5 + 11 * rs.rand()) + rs.rand() * 6),
                     128 + 100 * np.sin((x + y) / (9 + 9 * rs.rand()))], -1)
    base += rs.normal(0, 18, base.shape)
    if kind == "saturated":
        base = (base - 128) * 4 + 128
    elif kind == "grey":
        base = np.repeat(base.mean(-1, keepdims=True), 3, -1)
    elif kind == "flat":
        base = base * 0.05 + rs.uniform(20, 230, 3)
    return np.clip(np.round(base), 0, 255).astype(np.uint8)


def persons(rs, h, w, n):
    out = []
    for _ in range(n):
        cx, cy, s = rs.uniform(0.2 * w, 0.8 * w), rs.uniform(0.2 * h, 0.8 * h), rs.uniform(0.1, 0.4) * min(h, w)
        x = cx + s * rs.uniform(-1, 1, 17)
        y = cy + s * rs.uniform(-1.3, 1.3, 17)
        v = rs.choice([0, 1, 2], 17, p=[0.15, 0.25, 0.6])
        v[5], v[6] = 2, 2
        out.append(np.stack([x, y, v], -1))
    return np.array(out, np.float32).reshape(-1, 17, 3)


# (name, edge, (h, w), frame kind, persons, condition on the draws)
SCENARIOS = [
    ("small_flip", 96, (61, 83), "texture", 2, lambda p: p["hflip"]),
    ("small_noflip", 96, (61, 83), "texture", 2, lambda p: not p["hflip"]),
    ("large_flip", 96, (250, 330), "texture", 3, lambda p: p["hflip"] and p["crop"] != (0, 0)),
    ("large_noflip", 96, (250, 330), "texture", 3, lambda p: not p["hflip"] and p["crop"] != (0, 0)),
    ("portrait", 96, (301, 131), "texture", 2, lambda p: p["order"][0] == 1),
    ("landscape_odd", 96, (97, 255), "texture", 1, lambda p: p["order"][3] == 1),
    ("saturated", 96, (140, 150), "saturated", 2, lambda p: p["hflip"] and p["order"][1] == 3),
    ("grey", 96, (120, 99), "grey", 1, lambda p: p["order"][0] == 3),
    ("flat", 96, (100, 120), "flat", 1, lambda p: p["order"][3] == 1 and p["hflip"]),
    ("tiny", 96, (2, 3), "texture", 1, lambda p: True),
    ("jpeg_flip", 96, (180, 160), "texture", 2, lambda p: p["jpeg"] and p["hflip"]),
    ("jpeg_noflip", 96, (77, 200), "saturated", 2, lambda p: p["jpeg"] and not p["hflip"]),
    ("gray", 96, (150, 190), "texture", 2, lambda p: p["gray"]),
    ("gray_jpeg_side", 96, (111, 96), "texture", 1, lambda p: p["gray"] and p["hflip"]),
    ("coco_flip", 368, (480, 640), "blocks", 3, lambda p: p["hflip"]),
    ("coco_jpeg", 368, (427, 640), "blocks", 2, lambda p: p["jpeg"] and not p["hflip"]),
]


def find_seed(engine, size, edge, cond):
    import torch
    for seed in range(100000):
        p = engine.augment_params([size], torch.Generator().manual_seed(seed), edge)[0]
        if cond(p):
            return seed
    raise RuntimeError("no seed")


def run_reference(ref_tr, ref_utils, ds, src_rgb, kp, edge, seed):
    import PIL.Image
    import torch
    obj = ds.CocoKeypoints.__new__(ds.CocoKeypoints)
    obj.HEATMAP_COUNT = 18
    obj.LIMB_IDS = ds.kp_connections(ds.get_keypoints())
    obj.input_y = obj.input_x = edge
    obj.stride = 8
    preprocess = ref_tr.Compose([ref_tr.Normalize(), ref_tr.RandomApply(ref_tr.HFlip(), 0.5), ref_tr.RescaleRelative(),
                                 ref_tr.Crop(edge), ref_tr.CenterPad(edge)])
    anns = [{"keypoints": k.reshape(-1).tolist(), "bbox": [0.0, 0.0, 1.0, 1.0], "segmentation": []} for k in kp]
    torch.manual_seed(seed)
    image, anns, meta = preprocess(PIL.Image.fromarray(src_rgb), anns, None)
    steps = ref_tr.image_transform_train.transforms
    for t in steps[:3]:
        image = t(image)
    u8 = np.array(image.convert("RGB"))
    tensor = steps[4](steps[3](image))
    ref_utils.mask_valid_area(tensor, meta["valid_area"])
    heat, paf = obj.get_ground_truth(anns)
    kp_out = np.array([a["keypoints"] for a in anns])
    return {"u8": u8, "image": tensor.numpy(), "kp_out": kp_out, "heat": heat.transpose((2, 0, 1)).astype(np.float32),
            "paf": paf.transpose((2, 0, 1)).astype(np.float32), "hflip": bool(meta["hflip"]),
            "scale": np.asarray(meta["scale"]), "offset": np.asarray(meta["offset"]),
            "valid_area": np.asarray(meta["valid_area"], np.float64)}


def main(ref):
    import make_gt_golden
    ds = make_gt_golden.import_reference(ref)
    from lib.datasets import transforms as ref_tr, utils as ref_utils
    import _b200_alias
    _b200_alias.load_package()
    import importlib
    engine = importlib.import_module(_b200_alias.PKG + ".engine")
    rs = np.random.RandomState(20261019)
    for name, edge, (h, w), kind, n, cond in SCENARIOS:
        src = frame(rs, h, w, kind)
        kp = persons(rs, h, w, n)
        seed = find_seed(engine, (h, w), edge, cond)
        r = run_reference(ref_tr, ref_utils, ds, src, kp, edge, seed)
        np.savez_compressed(os.path.join(OUT, "aug_%s.npz" % name), src=src, kp=kp, seed=seed, edge=edge, **r)
        print(name, "seed", seed, "flip", r["hflip"], "kp dtype", r["kp_out"].dtype)
    with open(os.path.join(OUT, "aug_cube.json"), "w") as f:
        json.dump(cube_digests(), f, indent=1, sort_keys=True)


if __name__ == "__main__":
    main(sys.argv[1])
