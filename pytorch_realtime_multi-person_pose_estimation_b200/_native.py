"""ctypes binding of libb200pose.so (include/b200pose.h).  Loading is lazy; every failure is loud."""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# B200POSE_LIB selects another build of the same library (tools/variants.py: compile-time tuning variants); there is
# still no fallback of any kind - a missing file is an error.
LIB_PATH = os.environ.get("B200POSE_LIB") or os.path.join(_HERE, "libb200pose.so")
_lib = None

c_float_p = ctypes.POINTER(ctypes.c_float)
NUM_TENSORS = 184
HUMAN_FLOATS = 73
MODE_BF16, MODE_FP32, MODE_BF16X3, MODE_FP8, MODE_FP16 = 0, 1, 2, 3, 4
MODES = {"bf16": MODE_BF16, "fp32": MODE_FP32, "bf16x3": MODE_BF16X3, "fp8": MODE_FP8, "fp16": MODE_FP16}
PREPROCESS = {"rtpose": 1, "vgg": 2, "inception": 3, "ssd": 4}      # get_outputs' `preprocess` names


vp, ci, cl, cf = ctypes.c_void_p, ctypes.c_int, ctypes.c_long, ctypes.c_float
_SIGNATURES = {      # every exported symbol: (argtypes, restype)
    "b200pose_last_error": ([], ctypes.c_char_p),
    "b200pose_version": ([], ci),
    "b200pose_launch_count": ([], cl),
    "b200pose_net_create": ([ctypes.POINTER(vp), ci], ci),
    "b200pose_net_create_openpose": ([ctypes.POINTER(vp), ci, ci, ci], ci),
    "b200pose_openpose_num_tensors": ([ci, ci], ci),
    "b200pose_openpose_tensor_shape": ([ci, ci, ci, ctypes.POINTER(cl)], ci),
    "b200pose_net_destroy": ([vp], None),
    "b200pose_net_tensor_shape": ([ci, ctypes.POINTER(cl)], ci),
    "b200pose_net_set_tensor": ([vp, ci, vp, cl], ci),
    "b200pose_net_finalize": ([vp], ci),
    "b200pose_net_forward": ([vp, vp, ci, ci, ci, ci, ci, ctypes.POINTER(vp), ci, vp], ci),
    "b200pose_net_forward_u8": ([vp, vp, ci, ci, ci, ci, ci, ctypes.POINTER(vp), ci, vp], ci),
    "b200pose_net_set_preprocess": ([vp, ci], ci),
    "b200pose_net_set_stages": ([vp, ci], ci),
    "b200pose_net_forward_ragged_u8": ([vp, vp, ci, ci, vp, ci, ctypes.POINTER(vp), ci, vp], ci),
    "b200pose_net_profile": ([vp, vp, vp, ci, vp], ci),
    "b200pose_net_debug_run": ([vp, ci, vp], ci),
    "b200pose_net_debug_launch": ([vp, ci, vp, ci], ci),
    "b200pose_net_debug_read": ([vp, ci, ci, ci, ci, vp, cl], ci),
    "b200pose_net_debug_fp8": ([vp, ci, vp, ci, vp, ci], ci),
    "b200pose_net_overflow": ([vp, vp, ci, vp], ci),
    "b200pose_net_last_maps": ([vp, ctypes.POINTER(vp), ctypes.POINTER(vp), ctypes.POINTER(ci), ctypes.POINTER(ci),
                                ctypes.POINTER(ci)], ci),
    "b200pose_post_create": ([ctypes.POINTER(vp), ci, ci, ci, ci], ci),
    "b200pose_post_destroy": ([vp], None),
    "b200pose_post_run": ([vp, vp, vp, ci, ci, ci, ci, ci, cf, vp], ci),
    "b200pose_post_run_scaled": ([vp, vp, vp, ci, ci, ci, ci, ci, ci, cf, vp], ci),
    "b200pose_post_set_refine": ([vp, ci], ci),
    "b200pose_post_get_refine": ([vp], ci),
    "b200pose_post_sync": ([vp], ci),
    "b200pose_post_default_params": ([vp], ci),
    "b200pose_post_set_params": ([vp, vp], ci),
    "b200pose_post_get_params": ([vp, vp], ci),
    "b200pose_post_last_ticket": ([vp], cl),
    "b200pose_post_select": ([vp, cl], ci),
    "b200pose_post_debug": ([vp, vp, ci, ci], ci),
    "b200pose_post_status_accum": ([vp, ci], ci),
    "b200pose_post_debug_sort": ([vp, vp, ci, vp], ci),
    "b200pose_post_set_grids": ([vp, ci, ci], ci),
    "b200pose_post_debug_connections": ([vp, ci, ci, vp, vp, vp, ci], ci),
    "b200pose_post_debug_maps": ([vp, vp, cl, vp, cl], ci),
    "b200pose_post_num_humans": ([vp, ci], ci),
    "b200pose_post_status": ([vp, ci], ci),
    "b200pose_post_overflow": ([vp, ci], ci),
    "b200pose_post_get_humans": ([vp, ci, vp, ci], ci),
    "b200pose_post_get_peaks": ([vp, ci, vp, ci], ci),
    "b200pose_post_draw": ([vp, vp, ci, ci, vp, vp, vp], ci),
    "b200pose_infer": ([vp, vp, vp, ci, ci, ci, ci, ci, cf, vp], ci),
    "b200pose_infer_u8": ([vp, vp, vp, ci, ci, ci, ci, ci, cf, vp], ci),
    "b200pose_flip_merge": ([vp, vp, vp, vp, vp, ci, ci, ci, ci, ci, vp, vp, vp], ci),
    "b200pose_infer_flip": ([vp, vp, vp, ci, ci, ci, ci, ci, cf, vp], ci),
    "b200pose_infer_u8_flip": ([vp, vp, vp, ci, ci, ci, ci, ci, cf, vp], ci),
    "b200pose_crop_geometry": ([ci, ci, ci, ci, ctypes.POINTER(ctypes.c_double)] + [ctypes.POINTER(ci)] * 4, ci),
    "b200pose_net_crop_with_factor": ([vp, vp, ci, ci, ci, ci, ci, ci, vp, ci, vp], ci),
    "b200pose_infer_raw_u8": ([vp, vp, vp, ci, ci, ci, ci, ci, ci, ci, cf, ci, vp], ci),
    "b200pose_infer_raw_u8_multiscale": ([vp, vp, vp, ci, ci, ci, ci, ci, ci, ctypes.POINTER(ctypes.c_double), ci, ci, cf,
                                          ci, vp], ci),
    "b200pose_infer_raw_u8_ragged": ([vp, vp, vp, ci, ci, vp, ci, ci, ci, cf, ci, vp], ci),
    "b200pose_infer_raw_u8_multiscale_ragged": ([vp, vp, vp, ci, ci, vp, ci, ci, ctypes.POINTER(ctypes.c_double), ci, ci,
                                                 cf, ci, vp], ci),
    "b200pose_net_convert_frames": ([vp, vp, ci, ci, ci, ci, vp, ci, vp], ci),
    "b200pose_infer_frames": ([vp, vp, vp, ci, ci, ci, ci, ci, ci, ctypes.POINTER(ctypes.c_double), ci, ci, cf, ci, vp],
                              ci),
    "b200pose_jpeg_info": ([vp, ctypes.c_longlong, ctypes.POINTER(ci), ctypes.POINTER(ci), ctypes.POINTER(ci)], ci),
    "b200pose_jpeg_info_ex": ([vp, ctypes.c_longlong, ci, ctypes.POINTER(ci), ctypes.POINTER(ci), ctypes.POINTER(ci)], ci),
    "b200pose_net_set_jpeg_progressive": ([vp, ci], ci),
    "b200pose_net_get_jpeg_progressive": ([vp], ci),
    "b200pose_net_decode_jpegs": ([vp, vp, vp, ci, vp, ci, vp], ci),
    "b200pose_infer_jpegs": ([vp, vp, vp, vp, ci, ci, ci, ctypes.POINTER(ctypes.c_double), ci, ci, cf, ci, vp], ci),
    "b200pose_post_jpeg_status": ([vp, ci], ci),
    "b200pose_png_info": ([vp, ctypes.c_longlong, ctypes.POINTER(ci), ctypes.POINTER(ci), ctypes.POINTER(ci)], ci),
    "b200pose_net_decode_pngs": ([vp, vp, vp, ci, vp, ci, vp], ci),
    "b200pose_infer_pngs": ([vp, vp, vp, vp, ci, ci, ci, ctypes.POINTER(ctypes.c_double), ci, ci, cf, ci, vp], ci),
    "b200pose_post_png_status": ([vp, ci], ci),
    "b200pose_jpeg_encode_bound": ([ci, ci, ci], ctypes.c_longlong),
    "b200pose_net_encode_jpegs": ([vp, vp, ci, vp, ci, ci, ci, vp, ctypes.c_longlong, ci, vp, vp], ci),
    "b200pose_png_encode_bound": ([ci, ci], ctypes.c_longlong),
    "b200pose_net_encode_pngs": ([vp, vp, ci, vp, ci, vp, ctypes.c_longlong, ci, vp, vp], ci),
    "b200pose_coco_kpt_eval": ([ci, ci, ci, vp, vp, vp, vp, vp, ci, vp, vp, vp, vp, ci, vp, vp, vp, vp, vp,
                                ctypes.c_longlong, vp], ci),
    "b200pose_ground_truth": ([ci, vp, vp, vp, ci, vp, vp, ci, ci, vp], ci),
    "b200pose_ground_truth_f64": ([ci, vp, vp, vp, ci, vp, vp, ci, ci, vp], ci),
    "b200pose_net_augment": ([vp, vp, ci, ci, vp, vp, ci, vp, vp, ci, vp], ci),
    "b200pose_net_last_forward": ([vp, vp, vp, ci], ci),
    "b200pose_net_stage_losses": ([vp, vp, vp, vp, ci, vp, vp], ci),
    "process_paf": ([ci, ci, ci, vp, ci, ci, ci, vp, ci, ci, ci, vp], ci),
    "get_num_humans": ([], ci),
    "get_part_cid": ([ci, ci], ci),
    "get_score": ([ci], cf),
    "get_part_x": ([ci], ci),
    "get_part_y": ([ci], ci),
    "get_part_score": ([ci], cf),
}

# b200pose_frame (include/b200pose.h 3d): pixel formats and the per-frame descriptor
FRAME_FORMATS = {"bgr": 0, "nv12": 1, "i420": 2}
# JPEG encoding samplings: cv2's IMWRITE_JPEG_SAMPLING_FACTOR values (b200pose_net_encode_jpegs)
JPEG_SAMPLING = {"420": 0x221111, "422": 0x211111, "440": 0x121111, "411": 0x411111, "444": 0x111111}
# cv2.ROTATE_90_CLOCKWISE, cv2.ROTATE_180, cv2.ROTATE_90_COUNTERCLOCKWISE -> degrees clockwise
_CV2_ROTATIONS = {0: 90, 1: 180, 2: 270}


class PostParams(ctypes.Structure):
    """b200pose_post_params (include/b200pose.h section 2): the settings of PAF scoring and the person prune."""
    _fields_ = [("paf_thresh", ctypes.c_float), ("paf_samples", ctypes.c_int), ("paf_min_above", ctypes.c_int),
                ("min_parts", ctypes.c_int), ("min_person_score", ctypes.c_float)]

    def as_dict(self):
        return {name: getattr(self, name) for name, _ in self._fields_}


class Frame(ctypes.Structure):
    _fields_ = [("plane", ctypes.c_void_p * 3), ("pitch", ctypes.c_int * 3), ("h", ctypes.c_int), ("w", ctypes.c_int)]


def rotation_of(rotate_code):
    """Degrees clockwise of a cv2.ROTATE_* code (None: 0) - the `rotate` argument of the frame entry points."""
    if rotate_code is None:
        return 0
    if rotate_code not in _CV2_ROTATIONS:
        raise B200PoseError("unknown cv2 rotate code %r (cv2.ROTATE_90_CLOCKWISE, _180 or _90_COUNTERCLOCKWISE)"
                            % (rotate_code,))
    return _CV2_ROTATIONS[rotate_code]


class B200PoseError(RuntimeError):
    pass


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise B200PoseError("%s is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                            "(there is no CPU/PyTorch fallback for this path)" % LIB_PATH)
    L = ctypes.CDLL(LIB_PATH)
    for name, (args, res) in _SIGNATURES.items():
        fn = getattr(L, name)     # AttributeError here = the library does not export what include/b200pose.h declares
        fn.argtypes = args
        fn.restype = res
    _lib = L
    return L


EXPORTED = list(_SIGNATURES)


def check(rc, what=""):
    if rc != 0:
        msg = lib().b200pose_last_error()
        raise B200PoseError("%s failed (rc=%d): %s" % (what or "b200pose call", rc, msg.decode() if msg else "?"))


def crop_geometry(src_h, src_w, dest_size=368, factor=8):
    """(im_scale, (res_h, res_w), (pad_h, pad_w)) exactly as crop_with_factor (im_transform.py:119-134) computes them.
    Host arithmetic only, but it lives in the library so that there is one implementation."""
    sc = ctypes.c_double()
    v = [ctypes.c_int() for _ in range(4)]
    check(lib().b200pose_crop_geometry(int(src_h), int(src_w), int(dest_size), int(factor), ctypes.byref(sc),
                                       *[ctypes.byref(x) for x in v]), "b200pose_crop_geometry")
    return sc.value, (v[0].value, v[1].value), (v[2].value, v[3].value)


def launch_count():
    return int(lib().b200pose_launch_count())


def openpose_shapes(l2_stages=4, l1_stages=2):
    """The state_dict shapes of OpenPose_Model(l2_stages, l1_stages, 38, 19) in the reference's order, from the
    library's own table (no device needed)."""
    n = lib().b200pose_openpose_num_tensors(int(l2_stages), int(l1_stages))
    if n < 0:
        raise B200PoseError("OpenPose_Model(%r, %r): stages must be l2 >= 1, l1 >= 1, l2 + l1 <= 12"
                            % (l2_stages, l1_stages))
    dims = (ctypes.c_long * 4)()
    out = []
    for i in range(n):
        nd = lib().b200pose_openpose_tensor_shape(int(l2_stages), int(l1_stages), i, dims)
        out.append(tuple(int(d) for d in dims[:nd]))
    return out
