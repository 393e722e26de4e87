"""Drop-in for /root/reference/evaluate/coco_eval.py: the inference glue `get_outputs` (:80-114) and
`handle_paf_and_heat` (:197-242), and the evaluation loop around it (SURVEY.md 8f rank 3): `append_result` (:117-154),
`eval_coco` (:56-76), `run_eval` (:245-283).  pycocotools scores the evaluation loop where it can be imported;
elsewhere its COCOeval for keypoints runs on the device (engine.coco_keypoint_eval).  The network and the
post-processing run on the GPU through libb200pose.so.
Unlike the reference this module does not parse sys.argv at import; `cfg` is the shared lib.config node."""
import json
import os

import cv2
import numpy as np
import torch

from ..lib.config import cfg
from ..lib.datasets.preprocessing import (inception_preprocess, rtpose_preprocess, ssd_preprocess, vgg_preprocess)
from ..lib.network import im_transform
from ..lib.utils.common import draw_humans
from ..lib.utils.paf_to_pose import paf_to_pose_cpp

ORDER_COCO = [0, 15, 14, 17, 16, 5, 2, 6, 3, 7, 4, 11, 8, 12, 9, 13, 10]   # coco_eval.py:52


def get_outputs(img, model, preprocess):
    """img: HWC uint8 BGR -> (paf [h,w,38] f32, heatmap [h,w,19] f32, im_scale).

    With a model from this package's get_model() (bare, or wrapped in DataParallel as the demo does) the whole body
    runs on the device: the raw frame is uploaded as bytes, crop_with_factor and the normalisation are kernels (both
    bit-identical to the host functions the reference calls), and only the two final maps are copied back.  Any other
    nn.Module takes the reference's own sequence below."""
    core = getattr(model, "module", model)
    if (hasattr(core, "maps_from_frame") and preprocess in ('rtpose', 'vgg', 'inception', 'ssd')
            and isinstance(img, np.ndarray) and img.dtype == np.uint8 and img.ndim == 3 and img.shape[2] == 3
            and cfg.MODEL.DOWNSAMPLE % 8 == 0):
        paf_t, heat_t, im_scale = core.maps_from_frame(img, preprocess, cfg.DATASET.IMAGE_SIZE, cfg.MODEL.DOWNSAMPLE)
        heatmap = heat_t.cpu().data.numpy().transpose(0, 2, 3, 1)[0]
        paf = paf_t.cpu().data.numpy().transpose(0, 2, 3, 1)[0]
        return paf, heatmap, im_scale
    im_croped, im_scale, _ = im_transform.crop_with_factor(img, cfg.DATASET.IMAGE_SIZE, factor=cfg.MODEL.DOWNSAMPLE,
                                                           is_ceil=True)
    if preprocess == 'rtpose':
        im_data = rtpose_preprocess(im_croped)
    elif preprocess == 'vgg':
        im_data = vgg_preprocess(im_croped)
    elif preprocess == 'inception':
        im_data = inception_preprocess(im_croped)
    elif preprocess == 'ssd':
        im_data = ssd_preprocess(im_croped)
    batch_var = torch.from_numpy(np.expand_dims(im_data, 0)).cuda().float()   # unknown mode -> UnboundLocalError, as upstream
    predicted_outputs, _ = model(batch_var)
    output1, output2 = predicted_outputs[-2], predicted_outputs[-1]
    heatmap = output2.cpu().data.numpy().transpose(0, 2, 3, 1)[0]
    paf = output1.cpu().data.numpy().transpose(0, 2, 3, 1)[0]
    return paf, heatmap, im_scale


_SWAP_HEAT = np.array((0, 1, 5, 6, 7, 2, 3, 4, 11, 12, 13, 8, 9, 10, 15, 14, 17, 16, 18))
_SWAP_PAF = np.array((6, 7, 8, 9, 10, 11, 0, 1, 2, 3, 4, 5, 20, 21, 22, 23, 24, 25, 26, 27, 12, 13, 14, 15, 16, 17, 18,
                      19, 28, 29, 32, 33, 30, 31, 36, 37, 34, 35))


def handle_paf_and_heat(normal_heat, flipped_heat, normal_paf, flipped_paf):
    """Left/right-flip test-time averaging: mirror W, negate the PAF x components, swap left/right channels."""
    mirrored = flipped_paf[:, ::-1, :]
    mirrored[:, :, _SWAP_PAF[::2]] = -mirrored[:, :, _SWAP_PAF[::2]]   # in place on the caller's array, as upstream
    averaged_paf = (normal_paf + mirrored[:, :, _SWAP_PAF]) / 2.
    averaged_heatmap = (normal_heat + flipped_heat[:, ::-1, :][:, :, _SWAP_HEAT]) / 2.
    return averaged_paf, averaged_heatmap


def append_result(image_id, humans, upsample_keypoints, outputs):
    """coco_eval.py:117-154: one COCO keypoint record per person.  `upsample_keypoints` = (height, width) of the
    network input mapped back to the original image; the 18 parts are reordered to COCO's 17 (ORDER_COCO drops the
    neck), visible parts get v = 1, the record score is the constant 1."""
    for human in humans:
        keypoints = np.zeros((18, 3))
        for i in range(cfg.MODEL.NUM_KEYPOINTS):
            part = human.body_parts.get(i)
            if part is not None:
                keypoints[i] = (part.x * upsample_keypoints[1] + 0.5, part.y * upsample_keypoints[0] + 0.5, 1)
        outputs.append({"image_id": image_id, "category_id": 1, "keypoints": list(keypoints[ORDER_COCO, :].reshape(51)),
                        "score": 1.})


def _pycocotools():
    try:
        from pycocotools.coco import COCO
        from pycocotools.cocoeval import COCOeval
    except ImportError as e:       # loud: the reference imports it at module level
        raise ImportError("run_eval / eval_coco need pycocotools (not installed in this image): %s" % e)
    return COCO, COCOeval


class _CocoIndex:
    """The part of pycocotools' COCO index run_eval uses, from the parsed annotation file: getCatIds(catNms=...),
    getImgIds(catIds=...) (in the order of list(set(...)), as pycocotools returns them) and loadImgs."""

    def __init__(self, anno_file):
        with open(anno_file) as f:
            self.dataset = json.load(f)
        self.imgs = {im["id"]: im for im in self.dataset["images"]}
        self.cat_imgs = {}
        for ann in self.dataset["annotations"]:
            self.cat_imgs.setdefault(ann["category_id"], []).append(ann["image_id"])

    def getCatIds(self, catNms):
        return [c["id"] for c in self.dataset["categories"] if c["name"] in catNms]

    def getImgIds(self, catIds):
        ids = set()
        for i, c in enumerate(catIds):
            ids = set(self.cat_imgs.get(c, [])) if i == 0 else ids & set(self.cat_imgs.get(c, []))
        return list(ids)

    def loadImgs(self, img_id):
        return [self.imgs[img_id]]


def _have_pycocotools():
    try:
        _pycocotools()
    except ImportError:
        return False
    return True


def eval_coco(outputs, annFile, imgIds):
    """coco_eval.py:56-76: keypoint mAP of `outputs` with pycocotools (through a temporary results.json).  Where
    pycocotools cannot be imported, the same COCOeval for keypoints runs on the device
    (engine.coco_keypoint_eval, DESIGN.md 2.16): same stats, same printed summary, no results.json."""
    if not _have_pycocotools():
        from ..engine import coco_keypoint_eval
        ev = coco_keypoint_eval(annFile, outputs, imgIds)
        ev.summarize()
        return ev.stats[0]
    COCO, COCOeval = _pycocotools()
    with open('results.json', 'w') as f:
        json.dump(outputs, f)
    coco_gt = COCO(annFile)
    coco_dt = coco_gt.loadRes('results.json')
    ev = COCOeval(coco_gt, coco_dt, 'keypoints')
    ev.params.imgIds = imgIds
    ev.evaluate()
    ev.accumulate()
    ev.summarize()
    os.remove('results.json')
    return ev.stats[0]


EVAL_BATCH = 32      # images per device batch of the batched evaluation loop


def is_jpeg_name(name):
    return os.path.splitext(name)[1].lower() in (".jpg", ".jpeg")


def write_vis_device(post, net, frames, net_hw, paths, keep):
    """cv2.imwrite(paths[k], draw_humans(frames[k], humans)) for the frames k in `keep`, on the device: the frames are
    uploaded once into a packed buffer, the persons of the post object's selected run (frame i: image i of the run,
    coordinates of a network input net_hw[i]) are drawn on it in place (b200pose_post_draw), and the kept frames are
    encoded from the same buffer at cv2.imwrite's JPEG defaults, quality 95 and 4:2:0 (b200pose_net_encode_jpegs).  The
    host frames are left as they are."""
    dev = torch.from_numpy(np.concatenate([np.ascontiguousarray(f).reshape(-1) for f in frames]))
    dev = dev.to("cuda:%d" % net.device_index)
    sizes = [f.shape[:2] for f in frames]
    post.draw(dev.data_ptr(), True, len(frames), sizes, net_hw, torch.cuda.current_stream(dev.device).cuda_stream)
    views, at = [], 0
    for h, w in sizes:
        views.append(dev[at:at + h * w * 3].view(h, w, 3))
        at += h * w * 3
    for k, blob in zip(keep, net.encode_jpegs([views[k] for k in keep], 95, "420")):
        with open(paths[k], "wb") as f:
            f.write(blob)


def _humans_batched(core, images, preprocess, vis_paths=None):
    """images (raw BGR frames of mixed sizes) -> per image (humans, heat-map shape): one fused device pass per ragged
    batch of frames of different sizes (crop_with_factor, normalisation, network, NMS, PAF matching, assembly - nothing but the person rows comes back)
    instead of get_outputs + paf_to_pose_cpp per image.  Same kernels, same arithmetic: identical persons.
    vis_paths: per image its visualisation file; those named .jpg / .jpeg are drawn, encoded and written on the device
    here (write_vis_device), one ragged batch after the other, the others are left to the caller."""
    from .. import _native as nat
    from ..engine import plan_ragged_batches
    from ..lib.utils.paf_to_pose import humans_from_rows
    eng = core.pose_engine(batch_cap=EVAL_BATCH)
    eng.net.set_preprocess(preprocess)
    args = (cfg.DATASET.IMAGE_SIZE, cfg.MODEL.DOWNSAMPLE, float(np.float32(cfg.TEST.THRESH_HEATMAP)))
    jpeg = [bool(vis_paths) and is_jpeg_name(vis_paths[i]) for i in range(len(images))]
    if not any(jpeg):
        rows = eng.infer_images_arrays(images, *args)
    else:
        # the ragged batches infer_images_arrays would run, one call each, so that each batch's run is the selected
        # one when its frames are drawn; a batch planned again on its own frames stays one batch
        pads = [nat.crop_geometry(im.shape[0], im.shape[1], args[0], args[1])[2] for im in images]
        rows = [None] * len(images)
        for part in plan_ragged_batches(pads, eng.post.batch_cap):
            sub = [images[i] for i in part]
            for i, r in zip(part, eng.infer_images_arrays(sub, *args)):
                rows[i] = r
            keep = [k for k, i in enumerate(part) if jpeg[i]]
            if keep:
                eng.post.sync()
                write_vis_device(eng.post, eng.net, sub, [pads[i] for i in part], [vis_paths[i] for i in part], keep)
    out = []
    for img, r in zip(images, rows):
        scale, _, (ph, pw) = nat.crop_geometry(img.shape[0], img.shape[1], cfg.DATASET.IMAGE_SIZE, cfg.MODEL.DOWNSAMPLE)
        out.append((humans_from_rows(r, pw, ph, cfg.MODEL.NUM_KEYPOINTS), (ph // cfg.MODEL.DOWNSAMPLE, pw // cfg.MODEL.DOWNSAMPLE), scale))
    return out


def run_eval(image_dir, anno_file, vis_dir, model, preprocess):
    """coco_eval.py:245-283: every person image of the annotation file -> get_outputs -> paf_to_pose_cpp ->
    visualisation written to vis_dir -> COCO records -> mAP.  With a model from this package's get_model() the images
    are processed EVAL_BATCH at a time by the fused batched engine (SURVEY.md 8f rank 3); any other module takes the
    reference's image-by-image sequence; its visualisations with a .jpg / .jpeg name are then drawn and encoded on the
    device, byte for byte cv2.imwrite(draw_humans(...)).  Records, visualisations and printed progress are the same
    either way.  Without pycocotools the annotation file is indexed here and eval_coco scores on the device."""
    coco = _pycocotools()[0](anno_file) if _have_pycocotools() else _CocoIndex(anno_file)
    img_ids = coco.getImgIds(catIds=coco.getCatIds(catNms=['person']))
    print("Total number of validation images {}".format(len(img_ids)))
    outputs = []
    print("Processing Images in validation set")
    core = getattr(model, "module", model)
    batched = hasattr(core, "pose_engine") and preprocess in ('rtpose', 'vgg', 'inception', 'ssd')
    for c0 in range(0, len(img_ids), EVAL_BATCH):
        chunk = img_ids[c0:c0 + EVAL_BATCH]
        names = [coco.loadImgs(img_id)[0]['file_name'] for img_id in chunk]
        images = [cv2.imread(os.path.join(image_dir, name)) for name in names]
        if batched:
            results = _humans_batched(core, images, preprocess, [os.path.join(vis_dir, name) for name in names])
        else:
            results = []
            for ori in images:
                paf, heatmap, scale_img = get_outputs(ori, model, preprocess)
                results.append((paf_to_pose_cpp(heatmap, paf, cfg), heatmap.shape[:2], scale_img))
        for k, (img_id, name, ori, (humans, hm_shape, scale_img)) in enumerate(zip(chunk, names, images, results)):
            i = c0 + k
            if i % 10 == 0 and i != 0:
                print("Processed {} images".format(i))
            if not (batched and is_jpeg_name(name)):      # .jpg / .jpeg: written on the device by _humans_batched
                cv2.imwrite(os.path.join(vis_dir, name), draw_humans(ori, humans))
            upsample_keypoints = (hm_shape[0] * cfg.MODEL.DOWNSAMPLE / scale_img,
                                  hm_shape[1] * cfg.MODEL.DOWNSAMPLE / scale_img)
            append_result(img_id, humans, upsample_keypoints, outputs)
    return eval_coco(outputs=outputs, annFile=anno_file, imgIds=img_ids)
