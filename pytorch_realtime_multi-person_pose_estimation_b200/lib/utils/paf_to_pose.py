"""Drop-in for the live post-processing entry points of /root/reference/lib/utils/paf_to_pose.py:
`NMS` (:67-145) and `paf_to_pose_cpp` (:372-406).  Both run on the GPU through libb200pose.so; the x8
nearest-neighbour up-sampling of the maps (:382-385, 31 MB per image in the reference) is never materialised -
the kernels read the low-resolution maps at (y >> 3, x >> 3), which is the same value."""
import numpy as np

from ... import _native as nat
from ...engine import NativePost
from .common import BodyPart, Human

_posts = {}


def _post(device_index=None, peak_cap=2048, human_cap=2048):
    import torch
    if not torch.cuda.is_available():
        raise nat.B200PoseError("paf_to_pose needs a CUDA device: this build has no CPU fallback")
    idx = torch.cuda.current_device() if device_index is None else device_index
    if idx not in _posts:
        _posts[idx] = NativePost(idx, batch_cap=1, peak_cap=peak_cap, human_cap=human_cap)
    return _posts[idx]


def _run(heatmaps, pafs, config):
    if config.MODEL.DOWNSAMPLE != 8:
        raise ValueError("the H100 path supports MODEL.DOWNSAMPLE == 8 only")
    heat = np.ascontiguousarray(heatmaps, dtype=np.float32)
    paf = np.ascontiguousarray(pafs, dtype=np.float32)
    if heat.ndim != 3 or heat.shape[2] != 19 or paf.shape[:2] != heat.shape[:2] or paf.shape[2] != 38:
        raise ValueError("expected heatmaps [h,w,19] and pafs [h,w,38]")
    post = _post()
    h, w = heat.shape[:2]
    post.run(heat.ctypes.data, paf.ctypes.data, False, 1, 1, h, w, float(np.float32(config.TEST.THRESH_HEATMAP)))
    post.sync()
    post.check_status(1)
    return post, h, w


def NMS(heatmaps, upsampFactor=1., bool_refine_center=True, bool_gaussian_filt=False, config=None):
    """Returns, per joint type, an array (k, 4) of (x, y, score, id) like paf_to_pose.py:67-145
    (refine branch, no Gaussian filtering - the configuration paf_to_pose_cpp uses)."""
    if not bool_refine_center or bool_gaussian_filt or upsampFactor != 8:
        raise NotImplementedError("only NMS(..., upsampFactor=8, bool_refine_center=True, bool_gaussian_filt=False)")
    pafs = np.zeros(heatmaps.shape[:2] + (38,), np.float32)
    post, _, _ = _run(heatmaps, pafs, config)
    peaks = post.peaks(0)
    return [peaks[peaks[:, 4] == j][:, :4].astype(np.float64) for j in range(config.MODEL.NUM_KEYPOINTS)]


def humans_from_rows(rows, W, H, num_keypoints=18):
    """Person rows of the device ([k, 73]: score, 18 x (x, y, peak score, peak id | -1)) -> the Human / BodyPart objects
    paf_to_pose_cpp builds (paf_to_pose.py:388-405): coordinates normalised by the network input size."""
    humans = []
    for human_id, row in enumerate(rows):
        human = Human([])
        for part_idx in range(num_keypoints):
            x, y, s, cid = row[1 + 4 * part_idx: 5 + 4 * part_idx]
            if cid < 0:
                continue
            human.body_parts[part_idx] = BodyPart('%d-%d' % (human_id, part_idx), part_idx, float(x) / W, float(y) / H,
                                                  float(s))
        if human.body_parts:
            human.score = float(row[0])
            humans.append(human)
    return humans


def paf_to_pose_cpp(heatmaps, pafs, config):
    post, h, w = _run(heatmaps, pafs, config)
    W, H = w * config.MODEL.DOWNSAMPLE, h * config.MODEL.DOWNSAMPLE
    return humans_from_rows(post.humans(0), W, H, config.MODEL.NUM_KEYPOINTS)
