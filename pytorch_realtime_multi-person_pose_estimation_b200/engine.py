"""Batched device-resident engine: rtpose VGG19 forward + fused post-processing behind the C ABI.

This is the new batched entry point SURVEY.md 8(b) asks for (`infer_batch`); the reference-shaped per-image calls
(get_model().forward, get_outputs, paf_to_pose_cpp) are thin wrappers over the same native objects.
"""
import ctypes

import numpy as np

from . import _native as nat

# A ragged batch runs on the canvas of its largest frame, and every layer pays for the whole canvas (DESIGN.md 2.8):
# n * Hc * Wc may exceed the sum of the frames' own H_i * W_i by at most this factor.
RAGGED_WASTE = 1.125


def plan_ragged_batches(shapes, batch_cap, waste=RAGGED_WASTE):
    """Groups frames of padded sizes shapes[i] = (H_i, W_i) into ragged batches of at most batch_cap frames.
    Frames are ordered by orientation (landscape and square first, then portrait) and by size; a batch is closed when the
    next frame would make n * Hc * Wc exceed `waste` times the sum of H_i * W_i, or the orientation changes.  Returns
    lists of frame indices."""
    order = sorted(range(len(shapes)), key=lambda i: (shapes[i][0] > shapes[i][1], shapes[i][0], shapes[i][1], i))
    batches, cur, hc, wc, area = [], [], 0, 0, 0
    for i in order:
        h, w = shapes[i]
        nh, nw, na = max(hc, h), max(wc, w), area + h * w
        if cur and (len(cur) == batch_cap or (shapes[cur[0]][0] > shapes[cur[0]][1]) != (h > w)
                    or (len(cur) + 1) * nh * nw > waste * na):
            batches.append(cur)
            cur, nh, nw, na = [], h, w, h * w
        cur.append(i)
        hc, wc, area = nh, nw, na
    if cur:
        batches.append(cur)
    return batches


def _at(v, i):
    return v[i] if isinstance(v, (list, tuple)) else v


def check_overflow_flags(flags):
    """fp16 mode: binary16 tops out at 65504; an image whose activations went beyond it has inf / NaN maps."""
    bad = [int(i) for i in np.nonzero(np.asarray(flags))[0]]
    if bad:
        raise nat.B200PoseError("fp16 overflow: activations of image(s) %s exceeded the binary16 range (65504); their maps "
                                "are not valid - run them in bf16, bf16x3 or fp32 mode" % bad)


def _plane(a):
    """(array kept alive, pointer, row pitch in bytes, shape, on_device) of one uint8 plane: a numpy array or a torch
    tensor (CUDA: read in place).  Rows may be padded (the pitch is the row stride); within a row the bytes must be
    contiguous, else the plane is copied."""
    if isinstance(a, np.ndarray):
        if a.dtype != np.uint8:
            raise nat.B200PoseError("frames: expected uint8 planes, got %s" % a.dtype)
        if a.ndim not in (2, 3):
            raise nat.B200PoseError("frames: a plane has 2 or 3 dimensions, got shape %s" % (a.shape,))
        if a.strides[-1] != 1 or (a.ndim == 3 and a.strides[1] != a.shape[2]) or a.strides[0] < a.shape[1] * a.strides[1]:
            a = np.ascontiguousarray(a)
        return a, a.ctypes.data, a.strides[0], a.shape, False
    import torch
    if not isinstance(a, torch.Tensor) or a.dtype != torch.uint8:
        raise nat.B200PoseError("frames: expected uint8 numpy arrays or torch tensors, got %r" % (type(a),))
    if not a.is_cuda:
        return _plane(a.numpy())
    if a.dim() not in (2, 3):
        raise nat.B200PoseError("frames: a plane has 2 or 3 dimensions, got shape %s" % (tuple(a.shape),))
    if a.stride(-1) != 1 or (a.dim() == 3 and a.stride(1) != a.shape[2]) or \
            a.stride(0) < a.shape[1] * a.stride(1):
        a = a.contiguous()
    return a, a.data_ptr(), a.stride(0), tuple(a.shape), True


def _frame_planes(frame, fmt):
    """The planes of one frame: BGR (h, w, 3); NV12 / I420 as one packed 2-D (3h/2, w) array (cv2.cvtColor's layout)
    or as a tuple (Y, UV) / (Y, U, V), UV given as (h/2, w) or (h/2, w/2, 2)."""
    if fmt == "bgr":
        return [frame]
    if isinstance(frame, (tuple, list)):
        return list(frame)
    if len(frame.shape) != 2 or frame.shape[0] % 3:
        raise nat.B200PoseError("frames: a packed %s frame is a 2-D (3h/2, w) array, got shape %s"
                                % (fmt.upper(), tuple(frame.shape)))
    h, w = frame.shape[0] * 2 // 3, frame.shape[1]
    if fmt == "nv12":
        return [frame[:h], frame[h:]]
    if not isinstance(frame, np.ndarray):
        frame = frame.contiguous()
    else:
        frame = np.ascontiguousarray(frame)
    flat, q = frame.reshape(-1), (h // 2) * (w // 2)
    return [frame[:h], flat[h * w:h * w + q].reshape(h // 2, w // 2), flat[h * w + q:h * w + 2 * q].reshape(h // 2, w // 2)]


def frame_table(frames, format):
    """frames -> (ctypes array of b200pose_frame, the arrays it points into, on_device, stored sizes [(h, w)]).
    Plane shapes are checked here, so the library never reads past a plane; sizes and pitches are checked there."""
    if format not in nat.FRAME_FORMATS:
        raise nat.B200PoseError("frames: unknown format %r (expected one of %s)" % (format, sorted(nat.FRAME_FORMATS)))
    table = (nat.Frame * max(1, len(frames)))()
    keep, sides, sizes = [], set(), []
    for i, frame in enumerate(frames):
        planes = [_plane(a) for a in _frame_planes(frame, format)]
        want = {"bgr": 1, "nv12": 2, "i420": 3}[format]
        if len(planes) != want:
            raise nat.B200PoseError("frame %d: %s has %d planes, got %d" % (i, format.upper(), want, len(planes)))
        shp = [p[3] for p in planes]
        h, w = shp[0][0], shp[0][1]
        if format == "bgr":
            ok = len(shp[0]) == 3 and shp[0][2] == 3
        elif format == "nv12":
            ok = len(shp[0]) == 2 and tuple(shp[1]) in ((h // 2, w), (h // 2, w // 2, 2))
        else:
            ok = len(shp[0]) == 2 and all(tuple(s) == (h // 2, w // 2) for s in shp[1:])
        if not ok:
            raise nat.B200PoseError("frame %d: plane shapes %s do not form a %s frame" % (i, shp, format.upper()))
        for k, (arr, ptr, pitch, _, dev) in enumerate(planes):
            table[i].plane[k] = ptr
            table[i].pitch[k] = pitch
            keep.append(arr)
            sides.add(dev)
        table[i].h, table[i].w = h, w
        sizes.append((h, w))
    if len(sides) > 1:
        raise nat.B200PoseError("frames: all planes must be host arrays or all CUDA tensors")
    return table, keep, sides == {True}, sizes


def _blob(b):
    """A JPEG stream (bytes, bytearray or a 1-D uint8 numpy array) as a uint8 array whose memory the library reads."""
    a = np.frombuffer(b, np.uint8) if isinstance(b, (bytes, bytearray, memoryview)) else np.ascontiguousarray(b)
    if a.dtype != np.uint8 or a.ndim != 1:
        raise nat.B200PoseError("jpeg: a stream is bytes or a 1-D uint8 array, got %s %s" % (a.dtype, a.shape))
    return a


def jpeg_table(blobs):
    """(stream pointer array, size array, the arrays they point into) of b200pose_net_decode_jpegs / _infer_jpegs."""
    arrs = [_blob(b) for b in blobs]
    ptrs = (ctypes.c_void_p * max(1, len(arrs)))(*[a.ctypes.data for a in arrs])
    sizes = (ctypes.c_longlong * max(1, len(arrs)))(*[a.size for a in arrs])
    return ptrs, sizes, arrs


def jpeg_info(blob):
    """(h, w, supported, reason) of a JPEG stream on the host (b200pose_jpeg_info): the size of the frame
    cv2.imdecode returns, EXIF orientation applied, and whether the device decodes it (reason: why not).  Raises for a
    malformed stream."""
    a = _blob(blob)
    h, w, sup = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    nat.check(nat.lib().b200pose_jpeg_info(ctypes.c_void_p(a.ctypes.data), a.size, ctypes.byref(h), ctypes.byref(w),
                                           ctypes.byref(sup)), "b200pose_jpeg_info")
    reason = "" if sup.value else nat.lib().b200pose_last_error().decode()
    return h.value, w.value, bool(sup.value), reason


def _packed_views(frames):
    """A device tensor whose data pointer starts the frames packed back to back: the first frame itself when the frames
    are contiguous and consecutive (views of one packed buffer, as b200pose_post_draw draws on), else a packed copy."""
    import torch
    if not frames:
        return None
    at = frames[0].data_ptr()
    for f in frames:
        if not f.is_contiguous() or f.data_ptr() != at:
            return torch.cat([f.reshape(-1) for f in frames])
        at += f.numel()
    return frames[0]


def rotated_size(h, w, rotate):
    return (w, h) if rotate in (90, 270) else (h, w)


class NativeNet:
    """Owns a b200pose_net handle on one CUDA device: the rtpose VGG19 network, or OpenPose_Model(l2, l1) for a net
    made by NativeNet.openpose."""

    openpose_stages = None       # (l2_stages, l1_stages) of an OpenPose_Model net

    def __init__(self, device_index, openpose=None):
        self._h = ctypes.c_void_p()
        if openpose is None:
            nat.check(nat.lib().b200pose_net_create(ctypes.byref(self._h), int(device_index)), "b200pose_net_create")
        else:
            l2, l1 = (int(v) for v in openpose)
            nat.check(nat.lib().b200pose_net_create_openpose(ctypes.byref(self._h), int(device_index), l2, l1),
                      "b200pose_net_create_openpose")
            self.openpose_stages = (l2, l1)
        self.device_index = int(device_index)

    @classmethod
    def openpose(cls, device_index=0, l2_stages=4, l1_stages=2):
        """A net of the reference's OpenPose_Model(l2_stages, l1_stages, 38, 19) (lib/network/openpose.py): load its
        state dict with load_state_dict_arrays (or use openpose_engine, which checks the names too)."""
        return cls(device_index, openpose=(l2_stages, l1_stages))

    @property
    def num_tensors(self):
        return nat.NUM_TENSORS if self.openpose_stages is None else len(nat.openpose_shapes(*self.openpose_stages))

    def load_state_dict_arrays(self, arrays):
        """arrays: the net's state_dict tensors as float32 numpy arrays in the reference's order (rtpose: 184)."""
        L = nat.lib()
        if len(arrays) != self.num_tensors:
            what = "rtpose" if self.openpose_stages is None else "OpenPose_Model(%d, %d)" % self.openpose_stages
            raise nat.B200PoseError("%s: expected %d tensors, got %d" % (what, self.num_tensors, len(arrays)))
        for i, a in enumerate(arrays):
            a = np.ascontiguousarray(a, dtype=np.float32)
            nat.check(L.b200pose_net_set_tensor(self._h, i, a.ctypes.data, a.size), "set_tensor(%d)" % i)
        nat.check(L.b200pose_net_finalize(self._h), "b200pose_net_finalize")

    def set_preprocess(self, name):
        """Normalisation fused into the uint8 entry points: 'rtpose' (default), 'vgg', 'inception' or 'ssd'
        (lib/datasets/preprocessing.py; get_outputs' `preprocess` argument)."""
        if name not in nat.PREPROCESS:
            raise nat.B200PoseError("unknown preprocess %r (expected one of %s)" % (name, sorted(nat.PREPROCESS)))
        nat.check(nat.lib().b200pose_net_set_preprocess(self._h, nat.PREPROCESS[name]), "b200pose_net_set_preprocess")

    def set_stages(self, k):
        """Refinement stages every later forward runs: the trunk, stage 1 and stages 2 .. k (1 <= k <= 6, default 6).
        Forwards fill the first 2k of the 12 stage maps; the fused entry points post-process stage k's maps."""
        k = int(k)
        if k != self.__dict__.get("_stages", 6):      # the net's count: every change of it goes through here
            nat.check(nat.lib().b200pose_net_set_stages(self._h, k), "b200pose_net_set_stages")
            self._stages = k

    def forward_ptr(self, in_ptr, in_on_device, n, H, W, mode, out_ptrs, out_on_device, stream):
        arr = (ctypes.c_void_p * 12)(*[ctypes.c_void_p(p) if p else None for p in out_ptrs])
        nat.check(nat.lib().b200pose_net_forward(self._h, ctypes.c_void_p(in_ptr), int(in_on_device), n, H, W, mode,
                                                 arr, int(out_on_device), ctypes.c_void_p(stream)), "b200pose_net_forward")

    def forward_u8_ptr(self, in_ptr, in_on_device, n, H, W, mode, out_ptrs, out_on_device, stream):
        """uint8 HWC BGR frames [n,H,W,3]; rtpose_preprocess is fused into the first convolution."""
        arr = (ctypes.c_void_p * 12)(*[ctypes.c_void_p(p) if p else None for p in out_ptrs])
        nat.check(nat.lib().b200pose_net_forward_u8(self._h, ctypes.c_void_p(in_ptr), int(in_on_device), n, H, W, mode,
                                                    arr, int(out_on_device), ctypes.c_void_p(stream)),
                  "b200pose_net_forward_u8")

    def forward_ragged_u8_ptr(self, in_ptr, in_on_device, shapes, mode, out_ptrs, out_on_device, stream):
        """Ragged batch: uint8 HWC BGR frames of the padded sizes shapes[i] = (H_i, W_i), packed back to back; the
        12 maps come out at the canvas size [n, C, max H_i / 8, max W_i / 8], +0 outside each frame."""
        hw = (ctypes.c_int * (2 * len(shapes)))(*[int(v) for s in shapes for v in s])
        arr = (ctypes.c_void_p * 12)(*[ctypes.c_void_p(p) if p else None for p in out_ptrs])
        nat.check(nat.lib().b200pose_net_forward_ragged_u8(self._h, ctypes.c_void_p(in_ptr), int(in_on_device), len(shapes),
                                                           hw, mode, arr, int(out_on_device), ctypes.c_void_p(stream)),
                  "b200pose_net_forward_ragged_u8")

    def overflow(self, n, stream=0):
        """Per image of the last forward (n = its batch): True if the fp16 mode overflowed binary16 for it.  Waits for
        `stream`.  Always False for the other modes."""
        flags = np.zeros(n, np.int32)
        if nat.lib().b200pose_net_overflow(self._h, flags.ctypes.data, int(n), ctypes.c_void_p(stream)) < 0:
            nat.check(1, "b200pose_net_overflow")
        return flags.astype(bool)

    def check_overflow(self, n, stream=0):
        """Raises B200PoseError naming the images of the last forward whose fp16 values overflowed."""
        check_overflow_flags(self.overflow(n, stream))

    def crop_with_factor(self, images, dest_size=368, factor=8):
        """Device-side crop_with_factor (im_transform.py:119-134) of uint8 BGR frames of one size: [n,h,w,3] or [h,w,3]
        -> (padded frames, im_scale, resized shape) like the reference (which returns them for one image)."""
        images = np.ascontiguousarray(images, dtype=np.uint8)
        single = images.ndim == 3
        if single:
            images = images[None]
        n, sh, sw, c = images.shape
        if c != 3:
            raise nat.B200PoseError("crop_with_factor: expected 3-channel BGR frames")
        scale, (rh, rw), (ph, pw) = nat.crop_geometry(sh, sw, dest_size, factor)
        out = np.empty((n, ph, pw, 3), np.uint8)
        nat.check(nat.lib().b200pose_net_crop_with_factor(self._h, ctypes.c_void_p(images.ctypes.data), 0, n, sh, sw,
                                                          int(dest_size), int(factor), ctypes.c_void_p(out.ctypes.data), 0,
                                                          None), "b200pose_net_crop_with_factor")
        return (out[0] if single else out), scale, (rh, rw, 3)

    def convert_frames(self, frames, format="nv12", rotate=0, stream=0, device=False):
        """Device-side cv2.rotate(cv2.cvtColor(frame, COLOR_YUV2BGR_NV12 / _I420)) of frames as PoseEngine.infer_frames
        takes them: a list of uint8 BGR host arrays [oh, ow, 3], `rotate` degrees clockwise.  device=True: frames of one
        size into a CUDA uint8 tensor [n, oh, ow, 3] instead, written asynchronously on the current stream."""
        table, keep, on_dev, sizes = frame_table(frames, format)
        outs = [rotated_size(h, w, rotate) for h, w in sizes]
        if device:
            import torch
            if len(set(outs)) != 1:
                raise nat.B200PoseError("convert_frames(device=True): the frames must share one size")
            out = torch.empty((len(frames),) + outs[0] + (3,), dtype=torch.uint8, device="cuda:%d" % self.device_index)
            nat.check(nat.lib().b200pose_net_convert_frames(self._h, table, len(frames), nat.FRAME_FORMATS[format],
                                                            int(on_dev), int(rotate), ctypes.c_void_p(out.data_ptr()), 1,
                                                            ctypes.c_void_p(torch.cuda.current_stream(out.device).cuda_stream)),
                      "b200pose_net_convert_frames")
            return out
        flat = np.empty(sum(h * w * 3 for h, w in outs), np.uint8)
        nat.check(nat.lib().b200pose_net_convert_frames(self._h, table, len(frames), nat.FRAME_FORMATS[format],
                                                        int(on_dev), int(rotate), ctypes.c_void_p(flat.ctypes.data), 0,
                                                        ctypes.c_void_p(stream)), "b200pose_net_convert_frames")
        res, at = [], 0
        for h, w in outs:
            res.append(flat[at:at + h * w * 3].reshape(h, w, 3))
            at += h * w * 3
        return res

    def decode_jpegs(self, blobs, device=False, stream=0):
        """cv2.imdecode(blob, cv2.IMREAD_COLOR) of every stream, on the device (b200pose_net_decode_jpegs): a list of
        uint8 HWC BGR numpy frames, or with device=True of CUDA uint8 tensors [h, w, 3] (views of one buffer, written
        on the current stream).  Raises, naming the image, for a stream the device does not decode or whose data is
        damaged."""
        ptrs, sizes, keep = jpeg_table(blobs)
        shapes = [jpeg_info(b)[:2] for b in keep]
        total = sum(h * w * 3 for h, w in shapes)
        if device:
            import torch
            flat = torch.empty(max(1, total), dtype=torch.uint8, device="cuda:%d" % self.device_index)
            ptr, stream = flat.data_ptr(), torch.cuda.current_stream(flat.device).cuda_stream
        else:
            flat = np.empty(max(1, total), np.uint8)
            ptr = flat.ctypes.data
        nat.check(nat.lib().b200pose_net_decode_jpegs(self._h, ptrs, sizes, len(keep), ctypes.c_void_p(ptr), int(device),
                                                      ctypes.c_void_p(stream)), "b200pose_net_decode_jpegs")
        out, at = [], 0
        for h, w in shapes:
            out.append(flat[at:at + h * w * 3].reshape(h, w, 3))
            at += h * w * 3
        return out

    def _frames_to_encode(self, frames, what):
        """The frames of an encode call as (frame pointer, on device, [(h, w)], buffer that keeps the pointer valid):
        a list of uint8 HWC BGR numpy arrays (packed on the host), a CUDA uint8 tensor [n, h, w, 3], or a list of CUDA
        uint8 tensors [h, w, 3] on the net's device (packed unless they are consecutive views of one buffer)."""
        try:
            import torch
        except ImportError:
            torch = None
        dev_in = torch is not None and (isinstance(frames, torch.Tensor) or any(isinstance(f, torch.Tensor) for f in frames))
        if dev_in:
            tensors = [frames] if isinstance(frames, torch.Tensor) else list(frames)
            for f in tensors:
                if not isinstance(f, torch.Tensor) or not f.is_cuda:
                    raise nat.B200PoseError("%s: frames are all numpy arrays or all CUDA tensors" % what)
                if f.device.index != self.device_index:
                    raise nat.B200PoseError("%s: a frame tensor is on %s, the net on cuda:%d"
                                            % (what, f.device, self.device_index))
            if isinstance(frames, torch.Tensor):
                if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[3] != 3:
                    raise nat.B200PoseError("%s: expected a CUDA uint8 tensor [n, h, w, 3]" % what)
                sizes = [tuple(frames.shape[1:3])] * frames.shape[0]
                flat = frames.contiguous()
            else:
                for f in frames:
                    if f.dtype != torch.uint8 or f.dim() != 3 or f.shape[2] != 3:
                        raise nat.B200PoseError("%s: expected a list of CUDA uint8 tensors [h, w, 3]" % what)
                sizes = [tuple(f.shape[:2]) for f in frames]
                flat = _packed_views(frames)
            src = flat.data_ptr() if flat is not None else 0
        else:
            arrs = [np.ascontiguousarray(f) for f in frames]
            for a in arrs:
                if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3:
                    raise nat.B200PoseError("%s: expected uint8 HWC BGR frames" % what)
            sizes = [a.shape[:2] for a in arrs]
            flat = np.concatenate([a.reshape(-1) for a in arrs]) if arrs else None
            src = flat.ctypes.data if flat is not None else 0
        return src, dev_in, sizes, flat

    def _encode(self, frames, what, bound, call, device, stream):
        """The streams of an encode call `what` (the entry point's name without b200pose_net_): bound(h, w) gives
        each frame's capacity, call(src, on_device, hw, n, out, cap, out_on_device, lens, stream) runs the entry point.  A list of bytes, or with device=True of 1-D CUDA uint8
        tensors (views of one buffer, written on the current stream)."""
        src, dev_in, sizes, flat = self._frames_to_encode(frames, what)
        n = len(sizes)
        if n == 0:
            return []
        cap = 0
        for h, w in sizes:
            b = int(bound(int(h), int(w)))
            if b < 0:
                nat.check(1, "b200pose_%s_encode_bound" % what[len("encode_"):-1])
            cap += b
        if dev_in or device:
            import torch
            stream = torch.cuda.current_stream(torch.device("cuda", self.device_index)).cuda_stream
            out = (torch.empty(cap, dtype=torch.uint8, device="cuda:%d" % self.device_index) if device
                   else np.empty(cap, np.uint8))
        else:
            out = np.empty(cap, np.uint8)
        hw = (ctypes.c_int * (2 * n))(*[int(v) for s in sizes for v in s])
        lens = (ctypes.c_longlong * n)()
        nat.check(call(ctypes.c_void_p(src), int(dev_in), hw, n, ctypes.c_void_p(out.data_ptr() if device else out.ctypes.data),
                       cap, int(device), lens, ctypes.c_void_p(stream)), "b200pose_net_" + what)
        total = sum(lens)
        if device:      # the bound-sized buffer goes back to the allocator; the views keep only the streams
            out = out[:total].clone()
        res, at = [], 0
        for k in lens:
            res.append(out[at:at + k] if device else out[at:at + k].tobytes())
            at += k
        return res

    def encode_jpegs(self, frames, quality=95, sampling="420", device=False, stream=0):
        """cv2.imencode('.jpg', frame, [IMWRITE_JPEG_QUALITY, quality, IMWRITE_JPEG_SAMPLING_FACTOR, s])[1] of every
        frame, on the device (b200pose_net_encode_jpegs); sampling one of '420', '422', '440', '411', '444'.  frames: a
        list of uint8 HWC BGR numpy arrays (staged through the device), a CUDA uint8 tensor [n, h, w, 3], or a list of
        CUDA uint8 tensors [h, w, 3] of any sizes.  Returns a list of bytes, or with device=True of 1-D CUDA uint8
        tensors (views of one buffer, written on the current stream)."""
        if sampling not in nat.JPEG_SAMPLING:
            raise nat.B200PoseError("encode_jpegs: unknown sampling %r (one of %s)" % (sampling, sorted(nat.JPEG_SAMPLING)))
        code, L = nat.JPEG_SAMPLING[sampling], nat.lib()
        return self._encode(frames, "encode_jpegs", lambda h, w: L.b200pose_jpeg_encode_bound(h, w, code),
                            lambda src, dev_in, hw, n, out, cap, dev_out, lens, st: L.b200pose_net_encode_jpegs(
                                self._h, src, dev_in, hw, n, int(quality), code, out, cap, dev_out, lens, st),
                            device, stream)

    def encode_pngs(self, frames, device=False, stream=0):
        """cv2.imencode('.png', frame)[1] of every frame, on the device (b200pose_net_encode_pngs).  frames: a list of
        uint8 HWC BGR numpy arrays (staged through the device), a CUDA uint8 tensor [n, h, w, 3], or a list of CUDA
        uint8 tensors [h, w, 3] of any sizes.  Returns a list of bytes, or with device=True of 1-D CUDA uint8 tensors
        (views of one buffer, written on the current stream)."""
        L = nat.lib()
        return self._encode(frames, "encode_pngs", L.b200pose_png_encode_bound,
                            lambda src, dev_in, hw, n, out, cap, dev_out, lens, st: L.b200pose_net_encode_pngs(
                                self._h, src, dev_in, hw, n, out, cap, dev_out, lens, st),
                            device, stream)

    def __del__(self):
        try:
            if self._h:
                nat.lib().b200pose_net_destroy(self._h)
                self._h = None
        except Exception:
            pass


class NativePost:
    """Owns a b200pose_post handle (fused NMS + PAF scoring + matching + assembly)."""

    def __init__(self, device_index, batch_cap=32, peak_cap=1024, human_cap=1024):
        self._h = ctypes.c_void_p()
        nat.check(nat.lib().b200pose_post_create(ctypes.byref(self._h), int(device_index), batch_cap, peak_cap, human_cap),
                  "b200pose_post_create")
        self.batch_cap, self.peak_cap, self.human_cap = batch_cap, peak_cap, human_cap

    def set_params(self, **fields):
        """Settings of PAF scoring and the person prune for the runs submitted from now on (fused runs included):
        paf_thresh, paf_samples, paf_min_above, min_parts, min_person_score (include/b200pose.h section 2).  Fields not
        given take their defaults, so set_params() restores the reference's constants.  A value outside its range
        raises B200PoseError naming the field and leaves the settings unchanged."""
        q = nat.PostParams()
        nat.check(nat.lib().b200pose_post_default_params(ctypes.byref(q)), "b200pose_post_default_params")
        names = [name for name, _ in nat.PostParams._fields_]
        for k, v in fields.items():
            if k not in names:
                raise nat.B200PoseError("set_params: unknown field %r (one of %s)" % (k, ", ".join(names)))
            if isinstance(getattr(q, k), int) and (int(v) != v or not -2 ** 31 <= v < 2 ** 31):   # ctypes would wrap
                raise nat.B200PoseError("set_params: %s must be a 32-bit integer, got %r" % (k, v))
            setattr(q, k, v)
        nat.check(nat.lib().b200pose_post_set_params(self._h, ctypes.byref(q)), "b200pose_post_set_params")

    def params(self):
        """The settings the next run uses, as a dict of set_params' fields."""
        q = nat.PostParams()
        nat.check(nat.lib().b200pose_post_get_params(self._h, ctypes.byref(q)), "b200pose_post_get_params")
        return q.as_dict()

    def set_grids(self, score_blocks=0, sort_blocks=0):
        """Test hook: the grids of the PAF scoring and range sorting kernels for the runs submitted from now on (fused
        runs and debug_sort included); 0 restores a default.  The results never depend on them.  A value outside
        0 .. 65535 raises B200PoseError naming it and leaves the grids unchanged."""
        for name, v in (("score_blocks", score_blocks), ("sort_blocks", sort_blocks)):
            if int(v) != v or not -2 ** 31 <= v < 2 ** 31:      # ctypes would wrap
                raise nat.B200PoseError("set_grids: %s must be a 32-bit integer, got %r" % (name, v))
        nat.check(nat.lib().b200pose_post_set_grids(self._h, int(score_blocks), int(sort_blocks)),
                  "b200pose_post_set_grids")

    def connections(self, img, limb):
        """Test hook: (a int32 [k], b int32 [k], score float32 [k]), the connections the greedy matcher chose for limb
        `limb` of image `img` of the latest run, in its order; a and b index the peaks of the limb's two parts."""
        L = nat.lib()
        a = np.empty(self.peak_cap, np.int32)
        b = np.empty(self.peak_cap, np.int32)
        s = np.empty(self.peak_cap, np.float32)
        k = int(L.b200pose_post_debug_connections(self._h, int(img), int(limb), a.ctypes.data, b.ctypes.data,
                                                   s.ctypes.data, self.peak_cap))
        if k < 0:
            nat.check(1, "b200pose_post_debug_connections")
        return a[:k].copy(), b[:k].copy(), s[:k].copy()

    def run(self, heat_ptr, paf_ptr, on_device, layout, n, h, w, thresh, stream=0):
        nat.check(nat.lib().b200pose_post_run(self._h, ctypes.c_void_p(heat_ptr), ctypes.c_void_p(paf_ptr), int(on_device),
                                              layout, n, h, w, ctypes.c_float(thresh), ctypes.c_void_p(stream)),
                  "b200pose_post_run")

    def flip_merge(self, normal_heat, flipped_heat, normal_paf, flipped_paf, layout=1):
        """Device-side handle_paf_and_heat (evaluate/coco_eval.py:197-242) on host float32 arrays.
        layout 1: heat [n,h,w,19] / paf [n,h,w,38] (or a single image [h,w,C]); layout 0: [n,C,h,w].
        Returns (averaged_paf, averaged_heat) like the reference; the inputs are not modified."""
        arrs = [np.ascontiguousarray(a, dtype=np.float32) for a in (normal_heat, flipped_heat, normal_paf, flipped_paf)]
        single = arrs[0].ndim == 3
        if single:
            arrs = [a[None] for a in arrs]
        if layout == 1:
            n, h, w, ch = arrs[0].shape
            cp = arrs[2].shape[3]
        else:
            n, ch, h, w = arrs[0].shape
            cp = arrs[2].shape[1]
        if ch != 19 or cp != 38 or arrs[1].shape != arrs[0].shape or arrs[3].shape != arrs[2].shape:
            raise nat.B200PoseError("flip_merge: expected heat with 19 and paf with 38 channels, equal shapes")
        out_heat, out_paf = np.empty_like(arrs[0]), np.empty_like(arrs[2])
        nat.check(nat.lib().b200pose_flip_merge(self._h, *[ctypes.c_void_p(a.ctypes.data) for a in arrs], 0, int(layout),
                                                n, h, w, ctypes.c_void_p(out_heat.ctypes.data),
                                                ctypes.c_void_p(out_paf.ctypes.data), None), "b200pose_flip_merge")
        return (out_paf[0], out_heat[0]) if single else (out_paf, out_heat)

    def draw(self, frames_ptr, on_device, n, frame_hw, net_hw, stream=0):
        """Draws the persons of images 0 .. n-1 of the selected run in place on n packed uint8 HWC BGR frames
        (b200pose_post_draw): frame_hw / net_hw are n (h, w) pairs, the frames' sizes and their network inputs'."""
        fh = np.ascontiguousarray(frame_hw, np.int32).reshape(-1)
        nh = np.ascontiguousarray(net_hw, np.int32).reshape(-1)
        if len(fh) != 2 * n or len(nh) != 2 * n:
            raise nat.B200PoseError("draw: frame_hw and net_hw need %d (h, w) pairs" % n)
        nat.check(nat.lib().b200pose_post_draw(self._h, ctypes.c_void_p(frames_ptr), int(on_device), int(n),
                                               ctypes.c_void_p(fh.ctypes.data), ctypes.c_void_p(nh.ctypes.data),
                                               ctypes.c_void_p(stream)), "b200pose_post_draw")

    def sync(self):
        nat.check(nat.lib().b200pose_post_sync(self._h), "b200pose_post_sync")

    def last_ticket(self):
        return int(nat.lib().b200pose_post_last_ticket(self._h))

    def select(self, ticket):
        """Wait for run `ticket` (one of the last two submitted) and make the getters read its results."""
        nat.check(nat.lib().b200pose_post_select(self._h, int(ticket)), "b200pose_post_select")

    def status(self, img):
        return int(nat.lib().b200pose_post_status(self._h, img))

    def status_accum(self, reset=False):
        """OR of the status bits of every image of every run since the last reset (waits for the second stream)."""
        st = int(nat.lib().b200pose_post_status_accum(self._h, int(bool(reset))))
        if st < 0:
            nat.check(1, "b200pose_post_status_accum")
        return st

    def check_status(self, n):
        for i in range(n):
            st = self.status(i)
            if st < 0 or (st & 0xF):
                raise nat.B200PoseError("post-processing capacity exceeded on image %d (status bits %d: 1=peaks>%d per "
                                        "part, 2=candidate pool, 4=rows, 8=humans>%d); raise the caps"
                                        % (i, st & 0xF, self.peak_cap, self.human_cap))

    def overflow(self, img):
        """True if the network overflowed binary16 for frame img of the selected fused fp16 run."""
        v = int(nat.lib().b200pose_post_overflow(self._h, img))
        if v < 0:
            nat.check(1, "b200pose_post_overflow")
        return v == 1

    def jpeg_status(self, img):
        """Status bits of JPEG image img of the selected run (b200pose_post_jpeg_status): 0 when its data was whole."""
        v = int(nat.lib().b200pose_post_jpeg_status(self._h, img))
        if v < 0:
            nat.check(1, "b200pose_post_jpeg_status")
        return v

    def humans(self, img):
        """float32 [k, 73]: score, 18 x (x, y, peak score, peak id | -1)."""
        L = nat.lib()
        k = L.b200pose_post_num_humans(self._h, img)
        if k < 0:
            nat.check(1, "b200pose_post_num_humans")
        out = np.empty((max(k, 1), nat.HUMAN_FLOATS), np.float32)
        got = L.b200pose_post_get_humans(self._h, img, out.ctypes.data, k)
        return out[:got]

    def peaks(self, img):
        """float32 [P, 5]: x, y, score, id, part (the joint_list of paf_to_pose.py:376-378)."""
        cap = 18 * self.peak_cap
        out = np.empty((cap, 5), np.float32)
        got = nat.lib().b200pose_post_get_peaks(self._h, img, out.ctypes.data, cap)
        if got < 0:
            nat.check(1, "b200pose_post_get_peaks")
        return out[:got].copy()

    def __del__(self):
        try:
            if self._h:
                nat.lib().b200pose_post_destroy(self._h)
                self._h = None
        except Exception:
            pass


def post_params_from_cfg(cfg):
    """The post-processing settings of a reference config: cfg.TEST.THRESH_PAF and
    cfg.TEST.NUM_INTERMED_PTS_BETWEEN_KEYPOINTS on top of the defaults (the reference declares both keys but its
    pafprocess ignores them).  paf_min_above keeps its default 6, so fewer than 7 samples need it set explicitly.
    For NativePost.set_params(**d) or PoseEngine(post_params=d)."""
    q = nat.PostParams()
    nat.check(nat.lib().b200pose_post_default_params(ctypes.byref(q)), "b200pose_post_default_params")
    d = q.as_dict()
    d["paf_thresh"] = float(np.float32(cfg.TEST.THRESH_PAF))
    d["paf_samples"] = int(cfg.TEST.NUM_INTERMED_PTS_BETWEEN_KEYPOINTS)
    return d


def humans_to_dicts(rows, width, height):
    """[(score, {part: (x/width, y/height, peak score)})] - the content paf_to_pose_cpp puts into Human objects.
    Conversions are done in bulk (float32 -> Python float, i.e. double, then the divisions in double exactly like the
    reference's `float(x) / W`); the per-person dictionaries are the only Python-level loop left."""
    rows = np.asarray(rows, dtype=np.float32).reshape(-1, nat.HUMAN_FLOATS)
    if rows.shape[0] == 0:
        return []
    body = rows[:, 1:].reshape(-1, 18, 4).astype(np.float64)
    xs = (body[:, :, 0] / width).tolist()
    ys = (body[:, :, 1] / height).tolist()
    ss = body[:, :, 2].tolist()
    present = (body[:, :, 3] >= 0).tolist()
    scores = rows[:, 0].astype(np.float64).tolist()
    out = []
    for k in range(len(scores)):
        pr, x, y, sc = present[k], xs[k], ys[k], ss[k]
        parts = {p: (x[p], y[p], sc[p]) for p in range(18) if pr[p]}
        if parts:
            out.append((scores[k], parts))
    return out


class PoseEngine:
    """Fused batched inference on one GPU: images -> humans, maps never leave the device.  `stages`: the refinement
    stages each submission runs (1 .. 6, default 6); the fused entry points post-process the last one's maps.  On an
    OpenPose_Model net (NativeNet.openpose) the count is the architecture's: `stages` must stay None, and modes fp8 /
    fp16 are refused here.  `post_params`: the
    post-processing settings of the submissions (a dict of NativePost.set_params' fields; None: the reference's
    constants), changed later with set_post_params."""

    stages = 6

    def __init__(self, state_arrays, device_index=0, mode="bf16", batch_cap=32, peak_cap=1024, human_cap=1024, net=None,
                 stages=None, post_params=None):
        if net is None:
            net = NativeNet(device_index)
            net.load_state_dict_arrays(state_arrays)
        self.net = net
        if net.openpose_stages is not None:
            # the stage count is the architecture's: the engine never sets one; fp8 / fp16 do not run on such a net
            what = "OpenPose_Model(%d, %d)" % net.openpose_stages
            if stages is not None:
                raise nat.B200PoseError("%s runs all its stages; stages=%r cannot be set" % (what, stages))
            if mode in ("fp8", "fp16"):
                raise nat.B200PoseError("%s runs modes bf16, bf16x3 and fp32, not %s" % (what, mode))
            self.stages = None
        else:
            self.stages = 6 if stages is None else int(stages)
            self.net.set_stages(self.stages)      # an invalid count fails here, before any submission
        self.post = NativePost(device_index, batch_cap, peak_cap, human_cap)
        if post_params:
            self.post.set_params(**post_params)
        self.mode = nat.MODES[mode]
        self.device_index = device_index
        self._shapes = {}
        self._last = None

    def _net_h(self):
        """The net's handle, set to this engine's stage count: engines may share a net with each other and with the
        module (rtpose_model.pose_engine), so the count is set before every submission (not on an OpenPose_Model net)."""
        if self.net.openpose_stages is None:
            self.net.set_stages(self.stages)
        return self.net._h

    def set_post_params(self, params=None, **fields):
        """Post-processing settings of the following submissions (a dict such as post_params_from_cfg's, and / or
        fields; see NativePost.set_params).  Runs already submitted keep theirs."""
        self.post.set_params(**dict(params or {}, **fields))

    def _remember(self, n, H, W):
        """Shape of the run just submitted, kept per ticket (two runs may be in flight with different batch sizes or
        frame shapes: fetch(ticket=i) must read run i with run i's n and normalise by run i's W / H).  H, W: one size,
        or per frame lists for a ragged batch."""
        t = self.post.last_ticket()
        if self.__dict__.get("_shapes") is None:
            self._shapes = {}
        self._shapes[t] = (n, H, W)
        for old in [k for k in self._shapes if k < t - 1]:
            del self._shapes[old]
        self._last = (n, H, W)
        return t

    def _shape_of(self, ticket):
        if ticket is None:
            return self._last
        if ticket not in (self.__dict__.get("_shapes") or {}):
            raise nat.B200PoseError("ticket %r is not one of the last two runs" % (ticket,))
        return self._shapes[ticket]

    @classmethod
    def from_net(cls, net, mode="bf16", batch_cap=32, peak_cap=1024, human_cap=1024, stages=None, post_params=None):
        """An engine around an existing NativeNet (e.g. the one a get_model() module already packed its weights into)."""
        return cls(None, net.device_index, mode, batch_cap, peak_cap, human_cap, net=net, stages=stages,
                   post_params=post_params)

    def submit_images(self, images, dest_size=368, factor=8, thresh=0.1, flip=False):
        """Asynchronous half of infer_images for frames of ONE shape (a video stream): returns a ticket; the frames must
        stay alive until fetch(ticket=...).  Two submissions may be in flight."""
        batch = np.ascontiguousarray(np.stack(images))
        if batch.dtype != np.uint8 or batch.ndim != 4 or batch.shape[3] != 3:
            raise nat.B200PoseError("submit_images: expected uint8 [h,w,3] frames of one shape")
        if len(batch) > self.post.batch_cap:
            raise nat.B200PoseError("submit_images: %d frames exceed batch_cap %d" % (len(batch), self.post.batch_cap))
        t = self.infer_raw_async_u8(batch.ctypes.data, False, len(batch), batch.shape[1], batch.shape[2], dest_size, factor,
                                    thresh, flip)
        return self._hold(t, batch)

    def _hold(self, t, inputs):
        """Keeps the host inputs of run t alive until its fetch: host staging is read asynchronously."""
        if self.__dict__.get("_alive") is None:
            self._alive = {}
        self._alive[t] = inputs
        for old in [k for k in self._alive if k < t - 1]:
            del self._alive[old]
        return t

    def infer_frames_async(self, frames, format="nv12", rotate=0, dest_size=368, factor=8, thresh=0.1, flip=False,
                           scales=None, stream=0):
        """Video frames as decoders hand them out, converted and rotated on the device ahead of crop_with_factor
        (b200pose_infer_frames): `format` 'nv12', 'i420' or 'bgr'; numpy arrays or CUDA uint8 tensors (read in place);
        4:2:0 frames as one packed 2-D (3h/2, w) array (cv2.cvtColor's layout) or as planes (Y, UV) / (Y, U, V) whose
        row strides are their pitches, so a padded decoder surface needs no copy; BGR as (h, w, 3).  `rotate`: degrees
        clockwise (nat.rotation_of maps cv2.ROTATE_* codes).  Frames of one rotated size run as a uniform batch, mixed
        sizes as a ragged one; scales as for infer_images.  Returns a ticket; host frames are kept alive until the
        fetch.  Person coordinates refer to each rotated frame's padded frame."""
        table, keep, on_dev, sizes = frame_table(frames, format)
        rot = int(rotate)
        arr = None if scales is None else (ctypes.c_double * len(scales))(*[float(s) for s in scales])
        nat.check(nat.lib().b200pose_infer_frames(self._net_h(), self.post._h, table, len(frames),
                                                  nat.FRAME_FORMATS[format], int(on_dev), rot, int(dest_size), int(factor),
                                                  arr, 0 if scales is None else len(scales), self.mode,
                                                  ctypes.c_float(thresh), int(bool(flip)), ctypes.c_void_p(stream)),
                  "b200pose_infer_frames")
        pads = [nat.crop_geometry(*rotated_size(h, w, rot), dest_size, factor)[2] for h, w in sizes]
        if len(set(pads)) == 1:
            t = self._remember(len(frames), pads[0][0], pads[0][1])
        else:
            t = self._remember(len(frames), [p[0] for p in pads], [p[1] for p in pads])
        return self._hold(t, None if on_dev else keep)

    def infer_frames_arrays(self, frames, format="nv12", rotate=0, dest_size=368, factor=8, thresh=0.1, flip=False,
                            scales=None):
        """infer_frames, but per frame the raw person rows (float32 [k, 73], pixel coordinates of the padded frame)."""
        return self.infer_frames(frames, format, rotate, dest_size, factor, thresh, flip, scales, _arrays=True)

    def infer_frames(self, frames, format="nv12", rotate=0, dest_size=368, factor=8, thresh=0.1, flip=False,
                     scales=None, _arrays=False):
        """Blocking infer_frames_async over any number of frames: per-frame human lists in input order.  Frames are
        grouped into batches of at most batch_cap by plan_ragged_batches on their rotated padded sizes, as
        infer_images groups BGR frames."""
        _, _, _, sizes = frame_table(frames, format)
        pads = [nat.crop_geometry(*rotated_size(h, w, int(rotate)), dest_size, factor)[2] for h, w in sizes]
        out = [None] * len(frames)
        for part in plan_ragged_batches(pads, self.post.batch_cap):
            self.infer_frames_async([frames[i] for i in part], format, rotate, dest_size, factor, thresh, flip, scales)
            for i, humans in zip(part, self.fetch_arrays() if _arrays else self.fetch()):
                out[i] = humans.copy() if _arrays else humans
        return out

    def infer_jpegs_async(self, blobs, dest_size=368, factor=8, thresh=0.1, flip=False, scales=None, stream=0):
        """JPEG streams decoded on the device and run as infer_raw_* does on the decoded frames (b200pose_infer_jpegs):
        uniform when every frame has one size, ragged otherwise; scales as for infer_images.  At most batch_cap
        streams, all of which the device decodes (jpeg_info).  Returns a ticket; fetch / fetch_arrays raise, naming the
        images, when an image's entropy-coded data is damaged.  Person coordinates refer to each decoded frame's
        padded frame."""
        ptrs, sizes, keep = jpeg_table(blobs)
        shapes = [jpeg_info(b)[:2] for b in keep]
        arr = None if scales is None else (ctypes.c_double * len(scales))(*[float(s) for s in scales])
        nat.check(nat.lib().b200pose_infer_jpegs(self._net_h(), self.post._h, ptrs, sizes, len(keep), int(dest_size),
                                                 int(factor), arr, 0 if scales is None else len(scales), self.mode,
                                                 ctypes.c_float(thresh), int(bool(flip)), ctypes.c_void_p(stream)),
                  "b200pose_infer_jpegs")
        pads = [nat.crop_geometry(h, w, dest_size, factor)[2] for h, w in shapes]
        if len(set(pads)) == 1:
            t = self._remember(len(keep), pads[0][0], pads[0][1])
        else:
            t = self._remember(len(keep), [p[0] for p in pads], [p[1] for p in pads])
        self._jpeg_runs = {k for k in (self.__dict__.get("_jpeg_runs") or ()) if k >= t - 1} | {t}
        return t

    def check_jpegs(self, n, names=None):
        """Raises naming the images (names[k], default k) of the selected run whose entropy-coded data was damaged."""
        bad = [((names[k] if names else k), s) for k, s in ((k, self.post.jpeg_status(k)) for k in range(n)) if s]
        if bad:
            raise nat.B200PoseError("jpeg: damaged entropy-coded data in image(s) %s (status bits: 1 invalid code, 2 data "
                                    "ends early, 4 data left over, 8 restart markers)" % bad)

    def infer_jpegs_arrays(self, blobs, dest_size=368, factor=8, thresh=0.1, flip=False, scales=None):
        """infer_jpegs, but per image the raw person rows (float32 [k, 73], pixel coordinates of the padded frame)."""
        return self.infer_jpegs(blobs, dest_size, factor, thresh, flip, scales, _arrays=True)

    def infer_jpegs(self, blobs, dest_size=368, factor=8, thresh=0.1, flip=False, scales=None, _arrays=False):
        """infer_images([cv2.imdecode(b, cv2.IMREAD_COLOR) for b in blobs]) with the decoding on the device: per-image
        human lists in input order.  Streams are grouped by plan_ragged_batches on their decoded padded sizes
        (jpeg_info); streams the device does not decode (progressive, CMYK, ...) are decoded by cv2.imdecode and run
        through infer_images - a frame's result does not depend on its batch.  Malformed streams raise, and so do
        streams whose entropy-coded data is damaged, naming the image."""
        infos = []
        for i, b in enumerate(blobs):
            try:
                infos.append(jpeg_info(b))
            except nat.B200PoseError as e:
                raise nat.B200PoseError("infer_jpegs: image %d: %s" % (i, e)) from None
        dev = [i for i, inf in enumerate(infos) if inf[2]]
        out = [None] * len(blobs)
        pads = [nat.crop_geometry(infos[i][0], infos[i][1], dest_size, factor)[2] for i in dev]
        for part in plan_ragged_batches(pads, self.post.batch_cap):
            idx = [dev[k] for k in part]
            self.infer_jpegs_async([blobs[i] for i in idx], dest_size, factor, thresh, flip, scales)
            self.post.sync()
            self.check_jpegs(len(idx), idx)
            for i, humans in zip(idx, self.fetch_arrays() if _arrays else self.fetch()):
                out[i] = humans.copy() if _arrays else humans
        rest = [i for i, inf in enumerate(infos) if not inf[2]]
        if rest:
            import cv2
            frames = [cv2.imdecode(_blob(blobs[i]), cv2.IMREAD_COLOR) for i in rest]
            for i, humans in zip(rest, self.infer_images(frames, dest_size, factor, thresh, flip, scales, _arrays)):
                out[i] = humans
        return out

    def infer_async(self, in_ptr, in_on_device, n, H, W, thresh=0.1, stream=0):
        nat.check(nat.lib().b200pose_infer(self._net_h(), self.post._h, ctypes.c_void_p(in_ptr), int(in_on_device), n, H, W,
                                           self.mode, ctypes.c_float(thresh), ctypes.c_void_p(stream)), "b200pose_infer")
        return self._remember(n, H, W)

    def infer_async_u8(self, in_ptr, in_on_device, n, H, W, thresh=0.1, stream=0):
        """uint8 HWC BGR frames [n,H,W,3] (host pinned or device); preprocessing runs on the device."""
        nat.check(nat.lib().b200pose_infer_u8(self._net_h(), self.post._h, ctypes.c_void_p(in_ptr), int(in_on_device), n, H,
                                              W, self.mode, ctypes.c_float(thresh), ctypes.c_void_p(stream)),
                  "b200pose_infer_u8")
        return self._remember(n, H, W)

    def infer_flip_async(self, in_ptr, in_on_device, n, H, W, thresh=0.1, stream=0):
        """Flip test-time averaging (fp32 NCHW input): frames + device-made mirrored copies as one 2n batch, maps merged
        as handle_paf_and_heat does, post-processing on the averaged maps."""
        nat.check(nat.lib().b200pose_infer_flip(self._net_h(), self.post._h, ctypes.c_void_p(in_ptr), int(in_on_device), n,
                                                H, W, self.mode, ctypes.c_float(thresh), ctypes.c_void_p(stream)),
                  "b200pose_infer_flip")
        return self._remember(n, H, W)

    def infer_flip_async_u8(self, in_ptr, in_on_device, n, H, W, thresh=0.1, stream=0):
        nat.check(nat.lib().b200pose_infer_u8_flip(self._net_h(), self.post._h, ctypes.c_void_p(in_ptr), int(in_on_device),
                                                   n, H, W, self.mode, ctypes.c_float(thresh), ctypes.c_void_p(stream)),
                  "b200pose_infer_u8_flip")
        return self._remember(n, H, W)

    def infer_raw_async_u8(self, in_ptr, in_on_device, n, src_h, src_w, dest_size=368, factor=8, thresh=0.1, flip=False,
                           stream=0):
        """Raw uint8 BGR frames of one size [n,src_h,src_w,3]: crop_with_factor (resize + pad), the network and the
        post-processing all run on the device.  Person coordinates refer to the padded frame."""
        nat.check(nat.lib().b200pose_infer_raw_u8(self._net_h(), self.post._h, ctypes.c_void_p(in_ptr), int(in_on_device), n,
                                                  src_h, src_w, int(dest_size), int(factor), self.mode,
                                                  ctypes.c_float(thresh), int(bool(flip)), ctypes.c_void_p(stream)),
                  "b200pose_infer_raw_u8")
        _, _, (ph, pw) = nat.crop_geometry(src_h, src_w, dest_size, factor)
        return self._remember(n, ph, pw)

    def infer_raw_ragged_async_u8(self, in_ptr, in_on_device, src_shapes, dest_size=368, factor=8, thresh=0.1, flip=False,
                                  stream=0):
        """Raw uint8 BGR frames of different sizes src_shapes[i] = (h_i, w_i), packed back to back, as one ragged batch:
        each frame is cropped to its own padded size and person coordinates refer to that padded frame."""
        n = len(src_shapes)
        hw = (ctypes.c_int * (2 * n))(*[int(v) for s in src_shapes for v in s])
        nat.check(nat.lib().b200pose_infer_raw_u8_ragged(self._net_h(), self.post._h, ctypes.c_void_p(in_ptr), int(in_on_device),
                                                         n, hw, int(dest_size), int(factor), self.mode,
                                                         ctypes.c_float(thresh), int(bool(flip)), ctypes.c_void_p(stream)),
                  "b200pose_infer_raw_u8_ragged")
        pads = [nat.crop_geometry(h, w, dest_size, factor)[2] for h, w in src_shapes]
        return self._remember(n, [p[0] for p in pads], [p[1] for p in pads])

    def infer_raw_multiscale_async_u8(self, in_ptr, in_on_device, n, src_h, src_w, scales, base_size=368, factor=8,
                                      thresh=0.1, flip=False, stream=0):
        """Multi-scale (+ flip) test-time averaging of raw uint8 BGR frames of one size (BASELINE.json configs[4]):
        every scale s runs crop_with_factor(int(base_size * s)) + the network on the device, the maps are resized
        (bicubic) to the grid of base_size, averaged, and post-processed.  Coordinates refer to the padded base frame."""
        arr = (ctypes.c_double * len(scales))(*[float(s) for s in scales])
        nat.check(nat.lib().b200pose_infer_raw_u8_multiscale(self._net_h(), self.post._h, ctypes.c_void_p(in_ptr),
                                                             int(in_on_device), n, src_h, src_w, int(base_size),
                                                             int(factor), arr, len(scales), self.mode,
                                                             ctypes.c_float(thresh), int(bool(flip)),
                                                             ctypes.c_void_p(stream)),
                  "b200pose_infer_raw_u8_multiscale")
        _, _, (ph, pw) = nat.crop_geometry(src_h, src_w, base_size, factor)
        return self._remember(n, ph, pw)

    def infer_raw_multiscale_ragged_async_u8(self, in_ptr, in_on_device, src_shapes, scales, base_size=368, factor=8,
                                             thresh=0.1, flip=False, stream=0):
        """Multi-scale (+ flip) test-time averaging of raw uint8 BGR frames of different sizes src_shapes[i] = (h_i, w_i),
        packed back to back: every scale runs as one ragged batch, and person coordinates refer to each frame's own
        padded base frame."""
        n = len(src_shapes)
        hw = (ctypes.c_int * (2 * n))(*[int(v) for s in src_shapes for v in s])
        arr = (ctypes.c_double * len(scales))(*[float(s) for s in scales])
        nat.check(nat.lib().b200pose_infer_raw_u8_multiscale_ragged(self._net_h(), self.post._h, ctypes.c_void_p(in_ptr),
                                                                    int(in_on_device), n, hw, int(base_size), int(factor),
                                                                    arr, len(scales), self.mode, ctypes.c_float(thresh),
                                                                    int(bool(flip)), ctypes.c_void_p(stream)),
                  "b200pose_infer_raw_u8_multiscale_ragged")
        pads = [nat.crop_geometry(h, w, base_size, factor)[2] for h, w in src_shapes]
        return self._remember(n, [p[0] for p in pads], [p[1] for p in pads])

    def infer_images_arrays(self, images, dest_size=368, factor=8, thresh=0.1, flip=False, scales=None):
        """infer_images, but per image the raw person rows (float32 [k, 73], pixel coordinates of the padded frame)."""
        return self.infer_images(images, dest_size, factor, thresh, flip, scales, _arrays=True)

    def infer_images(self, images, dest_size=368, factor=8, thresh=0.1, flip=False, scales=None, _arrays=False):
        """images: a list of raw uint8 BGR frames of arbitrary (mixed) sizes, as cv2.imread returns them.  Returns per-image
        human lists in input order, coordinates normalised to the padded frame like paf_to_pose_cpp's.
        The frames run as ragged batches of at most batch_cap frames of different sizes (plan_ragged_batches on the
        padded sizes at dest_size; a batch of one source size takes the uniform entry point).  scales: e.g.
        (0.5, 1.0, 1.5, 2.0) for multi-scale test-time averaging around dest_size; every scale of a batch runs as one
        device batch."""
        for im in images:
            if im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3:
                raise nat.B200PoseError("infer_images: expected uint8 [h,w,3] frames")
        pads = [nat.crop_geometry(im.shape[0], im.shape[1], dest_size, factor)[2] for im in images]
        groups = plan_ragged_batches(pads, self.post.batch_cap)
        out = [None] * len(images)
        for part in groups:
            shapes = [images[i].shape[:2] for i in part]
            if len(set(shapes)) == 1:
                batch = np.ascontiguousarray(np.stack([images[i] for i in part]))
                self._keep = batch
                sh, sw = shapes[0]
                if scales is None:
                    self.infer_raw_async_u8(batch.ctypes.data, False, len(part), sh, sw, dest_size, factor, thresh, flip)
                else:
                    self.infer_raw_multiscale_async_u8(batch.ctypes.data, False, len(part), sh, sw, scales, dest_size,
                                                       factor, thresh, flip)
            else:
                batch = np.concatenate([np.ascontiguousarray(images[i]).ravel() for i in part])
                self._keep = batch
                if scales is None:
                    self.infer_raw_ragged_async_u8(batch.ctypes.data, False, shapes, dest_size, factor, thresh, flip)
                else:
                    self.infer_raw_multiscale_ragged_async_u8(batch.ctypes.data, False, shapes, scales, dest_size, factor,
                                                              thresh, flip)
            for i, humans in zip(part, self.fetch_arrays() if _arrays else self.fetch()):
                out[i] = humans.copy() if _arrays else humans
        return out

    def fetch(self, check=True, ticket=None):
        """Results of run `ticket` (default: the latest).  Up to two runs may be in flight: submit i+1, then fetch i."""
        n, H, W = self._shape_of(ticket)
        if ticket is None:
            self.post.sync()
        else:
            self.post.select(ticket)
        self._check_overflow(n)
        self._check_jpeg_run(ticket, n)
        if check:
            self.post.check_status(n)
        return [humans_to_dicts(self.post.humans(i), _at(W, i), _at(H, i)) for i in range(n)]

    def _check_jpeg_run(self, ticket, n):
        """A run made from JPEG streams (infer_jpegs_async) raises, whatever `check` says, when an image's entropy-coded
        data was damaged: its persons are never handed back in silence."""
        t = self.post.last_ticket() if ticket is None else ticket
        if t in (self.__dict__.get("_jpeg_runs") or ()):
            self.check_jpegs(n)

    def _check_overflow(self, n):
        if self.mode == nat.MODE_FP16:      # whatever `check` says: overflowed maps are never handed back in silence
            check_overflow_flags([self.post.overflow(i) for i in range(n)])

    def fetch_arrays(self, check=True, ticket=None):
        """Like fetch() but without building Python objects: per image a float32 array [k, 73] with rows
        (score, 18 x (x, y, peak score, peak id | -1)), x / y in pixels of the (padded) network input."""
        n, H, W = self._shape_of(ticket)
        if ticket is None:
            self.post.sync()
        else:
            self.post.select(ticket)
        self._check_overflow(n)
        self._check_jpeg_run(ticket, n)
        if check:
            self.post.check_status(n)
        return [self.post.humans(i) for i in range(n)]

    def encode_jpegs(self, frames, quality=95, sampling="420", device=False, stream=0):
        """NativeNet.encode_jpegs on this engine's device: cv2.imencode('.jpg', ...) of every frame, on the GPU."""
        return self.net.encode_jpegs(frames, quality, sampling, device, stream)

    def encode_pngs(self, frames, device=False, stream=0):
        """NativeNet.encode_pngs on this engine's device: cv2.imencode('.png', frame) of every frame, on the GPU."""
        return self.net.encode_pngs(frames, device, stream)

    def draw_humans(self, frames, ticket=None, dest_size=368, factor=8, net_sizes=None):
        """draw_humans(frame, humans_from_rows(rows, net_w, net_h)) for every frame of run `ticket` (default: the
        latest), on the device, in place like draw_humans(imgcopy=False): `frames` a list of uint8 HWC BGR numpy arrays
        (staged through the device; sizes may differ) or a CUDA uint8 tensor [n, h, w, 3] (drawn asynchronously on the
        current stream).  net_sizes: per frame the (h, w) of the padded network input its coordinates are in; default
        each frame's crop_geometry(h, w, dest_size, factor).  Returns `frames`."""
        if ticket is None:
            self.post.sync()
        else:
            self.post.select(ticket)
        try:
            import torch
            is_tensor = isinstance(frames, torch.Tensor)
        except ImportError:
            is_tensor = False
        if is_tensor:
            if not frames.is_cuda or frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[3] != 3:
                raise nat.B200PoseError("draw_humans: expected a CUDA uint8 tensor [n, h, w, 3]")
            if not frames.is_contiguous():
                raise nat.B200PoseError("draw_humans: the frame tensor must be contiguous (it is drawn in place)")
            sizes = [tuple(frames.shape[1:3])] * frames.shape[0]
        else:
            for f in frames:
                if not isinstance(f, np.ndarray) or f.dtype != np.uint8 or f.ndim != 3 or f.shape[2] != 3:
                    raise nat.B200PoseError("draw_humans: expected uint8 HWC BGR frames")
            sizes = [f.shape[:2] for f in frames]
        n = len(sizes)
        if n == 0:
            return frames
        if net_sizes is None:
            net_sizes = [nat.crop_geometry(h, w, dest_size, factor)[2] for h, w in sizes]
        if is_tensor:
            self.post.draw(frames.data_ptr(), True, n, sizes, net_sizes, torch.cuda.current_stream(frames.device).cuda_stream)
            return frames
        flat = np.concatenate([np.ascontiguousarray(f).reshape(-1) for f in frames])
        self.post.draw(flat.ctypes.data, False, n, sizes, net_sizes)
        at = 0
        for f in frames:
            f[...] = flat[at:at + f.size].reshape(f.shape)
            at += f.size
        return frames

    def infer_batch(self, images, thresh=0.1, flip=False):
        """images: uint8 numpy [n,H,W,3] (BGR frames, preprocessing fused on the device), float32 numpy [n,3,H,W]
        (already preprocessed, host) or a CUDA float tensor.  Returns per-image human lists.
        flip=True: left/right flip test-time averaging on the device (handle_paf_and_heat semantics)."""
        run_u8 = self.infer_flip_async_u8 if flip else self.infer_async_u8
        run_f32 = self.infer_flip_async if flip else self.infer_async
        if isinstance(images, np.ndarray) and images.dtype == np.uint8:
            images = np.ascontiguousarray(images)
            n, H, W, _ = images.shape          # [n,H,W,3] BGR, already cropped/padded to multiples of 8
            self._keep = images
            run_u8(images.ctypes.data, False, n, H, W, thresh)
        elif isinstance(images, np.ndarray):
            images = np.ascontiguousarray(images, dtype=np.float32)
            n, _, H, W = images.shape
            self._keep = images
            run_f32(images.ctypes.data, False, n, H, W, thresh)
        else:
            import torch
            if not images.is_cuda:
                raise nat.B200PoseError("torch inputs must live on the GPU (no CPU fallback)")
            images = images.contiguous().float()
            n, _, H, W = images.shape
            self._keep = images
            run_f32(images.data_ptr(), True, n, H, W, thresh, torch.cuda.current_stream().cuda_stream)
        return self.fetch()


def openpose_state_dict_keys(l2_stages=4, l1_stages=2):
    """The state_dict keys of the reference's OpenPose_Model(l2_stages, l1_stages) (lib/network/openpose.py), in order:
    feature_extractor (make_vgg19_block's Sequential: conv / ReLU / pool entries, PReLU after conv4_2, conv4_3_CPM and
    conv4_4_CPM), then l2_stages.{i} and l1_stages.{i} (StageBlock: Mconv{b}_{j}.Mconv / .MPrelu, Mconv6, Mconv7)."""
    keys, idx = [], 0
    for name in ("1_1", "1_2", "P", "2_1", "2_2", "P", "3_1", "3_2", "3_3", "3_4", "P", "4_1", "4_2", "4_3", "4_4"):
        if name == "P":
            idx += 1
            continue
        keys += ["feature_extractor.%d.weight" % idx, "feature_extractor.%d.bias" % idx]
        if name in ("4_2", "4_3", "4_4"):
            keys.append("feature_extractor.%d.weight" % (idx + 1))
        idx += 2
    for branch, count in (("l2_stages", l2_stages), ("l1_stages", l1_stages)):
        for i in range(count):
            for blk in ["Mconv%d_%d" % (b, j) for b in range(1, 6) for j in range(3)] + ["Mconv6"]:
                p = "%s.%d.%s." % (branch, i, blk)
                keys += [p + "Mconv.weight", p + "Mconv.bias", p + "MPrelu.weight"]
            keys += ["%s.%d.Mconv7.weight" % (branch, i), "%s.%d.Mconv7.bias" % (branch, i)]
    return keys


def openpose_engine(state_dict, l2_stages=4, l1_stages=2, device_index=0, mode="bf16", **engine_kwargs):
    """A PoseEngine running the reference's OpenPose_Model(l2_stages, l1_stages, 38, 19) with `state_dict` (its
    state_dict(), or any mapping of the same keys, in the same order, to tensors or arrays).  Every key and shape is
    checked against the model's - names from openpose_state_dict_keys, shapes from the library's table - and the first
    mismatch is named.  Modes bf16, bf16x3 and fp32; engine_kwargs as for PoseEngine (batch_cap, post_params, ...)."""
    keys = openpose_state_dict_keys(l2_stages, l1_stages)
    shapes = nat.openpose_shapes(l2_stages, l1_stages)
    what = "OpenPose_Model(%d, %d)" % (l2_stages, l1_stages)
    items = list(state_dict.items())
    arrays = []
    for i, want in enumerate(keys):
        if i >= len(items):
            raise nat.B200PoseError("%s state_dict: entry %d %r is missing (%d entries given, %d expected)"
                                    % (what, i, want, len(items), len(keys)))
        k, v = items[i]
        if k != want:
            raise nat.B200PoseError("%s state_dict: entry %d is %r, expected %r" % (what, i, k, want))
        a = v.detach().cpu().numpy() if hasattr(v, "detach") else np.asarray(v)
        if tuple(a.shape) != shapes[i]:
            raise nat.B200PoseError("%s state_dict: %r has shape %s, expected %s" % (what, k, tuple(a.shape), shapes[i]))
        arrays.append(np.ascontiguousarray(a, dtype=np.float32))
    if len(items) > len(keys):
        raise nat.B200PoseError("%s state_dict: unexpected entry %d %r (%d expected)" % (what, len(keys), items[len(keys)][0],
                                                                                      len(keys)))
    net = NativeNet.openpose(device_index, l2_stages, l1_stages)
    net.load_state_dict_arrays(arrays)
    return PoseEngine.from_net(net, mode=mode, **engine_kwargs)
