"""ORACLE (test infrastructure): NMS (/root/reference/lib/utils/paf_to_pose.py:67-145) at any integer up-sampling
factor f and with each refinement, and paf_to_pose_cpp (:372-406) at factor f, in numpy.  oracle/nms_port.py restates
the default (f = 8, bicubic refinement, no Gaussian); its results are what `nms` returns with the default keywords.

Third-party arithmetic restated (pinned bit for bit by tests/test_refine_host.py):
  * cv2.resize(patch, fx=f, fy=f, INTER_CUBIC) on float32 with IPP off (OpenCV 4.13): f = 1 returns the patch; otherwise
    interpolateCubic (A = -0.75) at source coordinate (float)((d + 0.5) / f - 0.5), replicated borders, horizontal pass
    ((s0 a0 + s1 a1) + s2 a2) + s3 a3, vertical pass s0 b0 + (s1 b1 + (s2 b2 + s3 b3)) on the columns OpenCV's 4-wide
    vector loop covers and ((s0 b0 + s1 b1) + s2 b2) + s3 b3 on the last W mod 4 columns of each row.
  * scipy.ndimage.gaussian_filter(patch, sigma=3) on float32 (SciPy 1.18: radius 12, mode 'reflect'): axis 0 then
    axis 1, each pass in double over the reflect-extended line, t = L[i] w[12] then t += (L[i-k] + L[i+k]) w[12-k] for
    k = 12 .. 1, rounded to float32 between the passes.
"""
import numpy as np

from oracle import nms_port

F32 = np.float32
WIN = nms_port.WIN
RADIUS = 12
# scipy.ndimage._filters._gaussian_kernel1d(3, 0, 12) (symmetric; w[0] is the outermost tap)
GAUSS_W = np.array([float.fromhex(x) for x in (
    "0x1.763a210dfb306p-15", "0x1.4fbe39149e277p-13", "0x1.0d8a5ad43c165p-11", "0x1.8345966f69518p-10",
    "0x1.f1e9915139406p-9", "0x1.1e6bccad344bap-7", "0x1.26defcaeb0202p-6", "0x1.0fa58939b528fp-5",
    "0x1.bfde9c12bec92p-5", "0x1.4a614d1afd337p-4", "0x1.b42a57d56c0bep-4", "0x1.01a25f86eb137p-3",
    "0x1.105a329f98197p-3")])
GAUSS_W = np.concatenate([GAUSS_W, GAUSS_W[-2::-1]])


def _axis_taps(n, f):
    """Per destination index of an n -> n f cubic resize: tap indices [N, 4] and float32 weights [N, 4]."""
    d = np.arange(n * f)
    fx = ((d + 0.5) * (1.0 / f) - 0.5).astype(F32)
    s = np.floor(fx).astype(np.int64)
    w = np.stack([nms_port._cubic_coeffs(x) for x in (fx - s.astype(F32)).astype(F32)]).astype(F32)
    return np.clip(s[:, None] - 1 + np.arange(4)[None, :], 0, n - 1), w


def upsample_cubic(patch, f):
    """cv2.resize(patch, None, fx=f, fy=f, interpolation=cv2.INTER_CUBIC) with IPP off, float32 patch."""
    patch = np.ascontiguousarray(patch, dtype=F32)
    if f == 1:
        return patch.copy()
    h, w = patch.shape
    ix, ax = _axis_taps(w, f)
    hor = patch[:, ix[:, 0]] * ax[:, 0]
    for j in (1, 2, 3):
        hor = hor + patch[:, ix[:, j]] * ax[:, j]
    iy, by = _axis_taps(h, f)
    vec = hor[iy[:, 3]] * by[:, 3:4]
    for j in (2, 1, 0):
        vec = hor[iy[:, j]] * by[:, j:j + 1] + vec
    tail = hor[iy[:, 0]] * by[:, 0:1]
    for j in (1, 2, 3):
        tail = tail + hor[iy[:, j]] * by[:, j:j + 1]
    W = w * f
    nv = W - W % 4
    return np.concatenate([vec[:, :nv], tail[:, nv:]], axis=1).astype(F32)


def gauss_rows_double(a):
    """One Gaussian pass along the last axis of a float32 array, in double, before the rounding to float32."""
    n = a.shape[-1]
    m = np.mod(np.arange(-RADIUS, n + RADIUS), 2 * n)
    m = np.where(m >= n, 2 * n - 1 - m, m)
    L = a[..., m].astype(np.float64)
    t = L[..., RADIUS:RADIUS + n] * GAUSS_W[RADIUS]
    for k in range(RADIUS, 0, -1):
        t = t + (L[..., RADIUS - k:RADIUS - k + n] + L[..., RADIUS + k:RADIUS + k + n]) * GAUSS_W[RADIUS - k]
    return t


def _gauss_axis(a, axis):
    return np.moveaxis(gauss_rows_double(np.moveaxis(a, axis, -1)).astype(F32), -1, axis)


def gaussian3(patch):
    """scipy.ndimage.gaussian_filter(patch, sigma=3) on a float32 patch."""
    return _gauss_axis(_gauss_axis(np.asarray(patch, F32), 0), 1)


def nms(heatmaps, thresh, num_keypoints=18, upsample=8, refine=True, gauss=False):
    """NMS(heatmaps, upsampFactor=upsample, bool_refine_center=refine, bool_gaussian_filt=gauss): a list of
    num_keypoints arrays (k, 4) float64 (x, y, score, id)."""
    if upsample == 8 and refine and not gauss:
        return nms_port.nms(heatmaps, thresh, num_keypoints)
    f = int(upsample)
    out, cnt = [], 0
    h, w = heatmaps.shape[:2]
    for joint in range(num_keypoints):
        m = np.ascontiguousarray(heatmaps[:, :, joint], dtype=F32)
        coords = nms_port.find_peaks(thresh, m)
        peaks = np.zeros((len(coords), 4))
        for i, (px, py) in enumerate(coords):
            if refine:
                x0, y0 = max(0, px - WIN), max(0, py - WIN)
                up = upsample_cubic(m[y0:min(h - 1, py + WIN) + 1, x0:min(w - 1, px + WIN) + 1], f)
                if gauss:
                    up = gaussian3(up)
                ay, ax = np.unravel_index(up.argmax(), up.shape)
                peaks[i] = (f * x0 + ax, f * y0 + ay, up[ay, ax], cnt)     # == paf_to_pose.py:129-140
            else:
                peaks[i] = ((px + 0.5) * f - 0.5, (py + 0.5) * f - 0.5, m[py, px], cnt)
            cnt += 1
        out.append(peaks)
    return out


def device_joint_list(jl):
    """The joint list as the device keeps it (and pafprocess reads it): positions truncated to int."""
    jl = np.array(jl, np.float32, copy=True)
    jl[:, :2] = np.trunc(jl[:, :2])
    return jl


def paf_to_pose(heat, paf, pafprocess, thresh=0.1, upsample=8, refine=True, gauss=False, num_keypoints=18):
    """paf_to_pose_cpp at factor `upsample`, NMS with the given refinement; `pafprocess` = any object exposing the
    SWIG module's functions.  Returns (joint_list [P, 5] float32, humans [(score, {part: (x / W, y / H, score)})])."""
    jl = nms_port.joint_list_from_nms(nms(heat, thresh, num_keypoints, upsample, refine, gauss))
    humans = []
    if jl.shape[0] > 0:
        f = int(upsample)
        paf_up = np.repeat(np.repeat(paf, f, axis=0), f, axis=1)      # == cv2 INTER_NEAREST x f
        heat_up = np.repeat(np.repeat(heat, f, axis=0), f, axis=1)
        pafprocess.process_paf(jl[None], np.ascontiguousarray(heat_up), np.ascontiguousarray(paf_up))
        H, W = heat_up.shape[:2]
        for hid in range(pafprocess.get_num_humans()):
            parts = {}
            for p in range(num_keypoints):
                c = int(pafprocess.get_part_cid(hid, p))
                if c < 0:
                    continue
                parts[p] = (float(pafprocess.get_part_x(c)) / W, float(pafprocess.get_part_y(c)) / H,
                            float(pafprocess.get_part_score(c)))
            if parts:
                humans.append((float(pafprocess.get_score(hid)), parts))
    return jl, humans


# ---------------------------------------------------------------------------------------- tests/golden/nms_modes.npz
# The scenarios, factors and modes of the fixture (tests/golden/make_nms_modes_golden.py runs the reference on them).
GOLDEN_THRESH = 0.1
GOLDEN_FACTORS = (1, 2, 3, 4, 8, 16)
MODES = {"cubic": (True, False), "gauss": (True, True), "none": (False, False)}     # -> (refine, gauss)
EDGE_SUBSET = (("plateau", 1, 1, 1), ("plateau", 3, 5, 5), ("quantised", 11, 1, 7), ("quantised", 13, 4, 5),
               ("checkerboard", 22, 4, 5), ("border", 43, 23, 31), ("twins", 51, 4, 5))


def scenarios(noise=True):
    """name -> (heat [h, w, 19], paf [h, w, 38]): the maps of post_p3, post_p30, post_noise0 (unless noise=False) and a
    subset of post_edges."""
    from oracle import synth
    out = {"p3": synth.stick_figures(3, 3)[:2], "p30": synth.stick_figures(30, 30)[:2]}
    if noise:
        out["noise0"] = synth.noise_maps(0)
    for c in EDGE_SUBSET:
        out[synth.edge_case_name(*c)] = synth.edge_maps(*c)
    return out


def golden_scenarios():
    """The fixture's scenarios: all but the noise maps, whose thousands of peaks per factor and mode would make it
    megabytes (the GPU tests check them against this oracle)."""
    return scenarios(noise=False)


def golden_key(name, f, mode):
    return "%s_f%d_%s" % (name, f, mode)
