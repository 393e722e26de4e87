"""Drop-in for the live post-processing entry points of /root/reference/lib/utils/paf_to_pose.py:
`NMS` (:67-145) and `paf_to_pose_cpp` (:372-406).  Both run on the GPU through libb200pose.so; the xf
nearest-neighbour up-sampling of the maps (:382-385, 31 MB per image at f = 8 in the reference) is never materialised -
the kernels read the low-resolution maps at (y // f, x // f), which is the same value."""
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


def _factor(f):
    """The integer up-sampling factor 1 .. 16 that f stands for, or None."""
    if isinstance(f, (bool, np.bool_)) or not isinstance(f, (int, float, np.integer, np.floating)):
        return None
    return int(f) if f == int(f) and 1 <= f <= 16 else None


def _run(heatmaps, pafs, config, upsample, refine):
    heat = np.ascontiguousarray(heatmaps, dtype=np.float32)
    paf = np.ascontiguousarray(pafs, dtype=np.float32)
    if heat.ndim != 3 or heat.shape[2] != 19 or paf.shape[:2] != heat.shape[:2] or paf.shape[2] != 38:
        raise ValueError("expected heatmaps [h,w,19] and pafs [h,w,38]")
    post = _post()
    h, w = heat.shape[:2]
    post.set_refine(refine)
    post.run(heat.ctypes.data, paf.ctypes.data, False, 1, 1, h, w, float(np.float32(config.TEST.THRESH_HEATMAP)),
             upsample=upsample)
    post.sync()
    post.check_status(1)
    return post, h, w


def NMS(heatmaps, upsampFactor=1., bool_refine_center=True, bool_gaussian_filt=False, config=None):
    """Returns, per joint type, an array (k, 4) of (x, y, score, id) like paf_to_pose.py:67-145, for an integer
    upsampFactor 1 .. 16 and every refinement: the bicubic patch (bool_refine_center), smoothed first with
    gaussian_filter(sigma=3) (bool_gaussian_filt), or none at all (bool_refine_center=False: the Gaussian flag is then
    ignored, as in the reference)."""
    f = _factor(upsampFactor)
    if f is None:
        raise NotImplementedError("NMS: upsampFactor must be an integer 1 .. 16, got %r" % (upsampFactor,))
    refine = ("gauss" if bool_gaussian_filt else "cubic") if bool_refine_center else "none"
    pafs = np.zeros(heatmaps.shape[:2] + (38,), np.float32)
    post, _, _ = _run(heatmaps, pafs, config, f, refine)
    peaks = post.peaks(0)
    out = []
    for j in range(config.MODEL.NUM_KEYPOINTS):
        pj = peaks[peaks[:, 4] == j][:, :4].astype(np.float64)
        if refine == "none":
            # the device keeps pafprocess's int position f p + (f - 1) // 2; NMS reports (p + 0.5) f - 0.5 itself
            pj[:, :2] = (pj[:, :2] // f + 0.5) * f - 0.5
        out.append(pj)
    return out


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
    """paf_to_pose.py:372-406 at any integer cfg.MODEL.DOWNSAMPLE f from 1 to 16: NMS at that factor, PAF scoring on the
    xf nearest-up-sampled maps, coordinates divided by w f and h f."""
    f = _factor(config.MODEL.DOWNSAMPLE)
    if f is None:
        raise ValueError("paf_to_pose_cpp: MODEL.DOWNSAMPLE must be an integer 1 .. 16, got %r" % (config.MODEL.DOWNSAMPLE,))
    post, h, w = _run(heatmaps, pafs, config, f, "cubic")
    return humans_from_rows(post.humans(0), w * f, h * f, config.MODEL.NUM_KEYPOINTS)
