"""Drop-in for /root/reference/lib/network/rtpose_vgg.py on the inference path.

`get_model('vgg19')` returns an nn.Module whose state_dict has the reference's 184 keys/shapes
(model0.{0,2,5,...}, model{1..6}_{1,2}.{0,2,...}; rtpose_vgg.py:69-127, 140-156), so
`model.load_state_dict(torch.load(w))`, `.cuda()`, `.float()`, `.eval()` and `torch.nn.DataParallel(model)`
(demo/picture_demo.py:45-49) work unchanged.  `forward` (rtpose_vgg.py:158-198) does NOT run nn.Conv2d: it hands
the input's device pointer to libb200pose.so, which runs the hand-written sm_90a kernels, and returns
`((paf, heat), saved_for_loss[12])` as CUDA fp32 NCHW tensors.

Precision: `model.precision = 'bf16x3'` (default: split-precision operands on the wgmma tensor cores with K-chunked
fp32 accumulation - maps within 1.4e-4 of the reference's fp32 network at 368x368, inside its 1e-3 tolerance), `'bf16'`
(the fast mode of the batched engine and the benchmark: ~4.5x faster, maps within ~8e-2) or `'fp32'` (CUDA cores,
bit-identical to the oracle's fp32 network); the environment variable B200POSE_MODE sets the default.
"""
import os
import threading

import torch
import torch.nn as nn

from ... import _native as nat
from ...engine import NativeNet

_TRUNK = [(3, 64), (64, 64), "P", (64, 128), (128, 128), "P", (128, 256), (256, 256), (256, 256), (256, 256), "P",
          (256, 512), (512, 512), (512, 256), (256, 128)]


def _stage_spec(stage, out_ch):
    if stage == 1:
        return [(128, 128, 3)] * 3 + [(128, 512, 1), (512, out_ch, 1)]
    return [(185, 128, 7)] + [(128, 128, 7)] * 4 + [(128, 128, 1), (128, out_ch, 1)]


def _make_trunk():
    layers = []
    for item in _TRUNK:
        if item == "P":
            layers.append(nn.MaxPool2d(2, 2, 0))
        else:
            layers += [nn.Conv2d(item[0], item[1], 3, 1, 1), nn.ReLU(inplace=True)]
    return nn.Sequential(*layers)


def _make_branch(spec):
    layers = []
    for i, (cin, cout, k) in enumerate(spec):
        layers.append(nn.Conv2d(cin, cout, k, 1, k // 2))
        if i != len(spec) - 1:          # the last conv of a branch has no ReLU (rtpose_vgg.py:30-35)
            layers.append(nn.ReLU(inplace=True))
    return nn.Sequential(*layers)


class rtpose_model(nn.Module):
    """Parameter container with the reference layout + native forward."""

    def __init__(self):
        super().__init__()
        self.model0 = _make_trunk()
        for s in range(1, 7):
            setattr(self, "model%d_1" % s, _make_branch(_stage_spec(s, 38)))
        for s in range(1, 7):
            setattr(self, "model%d_2" % s, _make_branch(_stage_spec(s, 19)))
        self.precision = os.environ.get("B200POSE_MODE", "bf16x3")
        self._engines = {}     # device index -> (signature, NativeNet); shared by DataParallel replicas
        self._lock = threading.Lock()
        # DataParallel replicas are shallow copies with EMPTY `_parameters` (torch/nn/parallel/replicate.py): plain
        # attributes like this box travel with the copy, so a replica finds the module that owns the weights.  (A list,
        # not the module itself: nn.Module.__setattr__ would register it as a child of itself.)
        self._master = [self]
        for m in self.modules():   # same init as rtpose_vgg.py:200-222
            if isinstance(m, nn.Conv2d):
                nn.init.normal_(m.weight, std=0.01)
                nn.init.constant_(m.bias, 0.0)

    def _signature(self):
        # every one of the 184 tensors: an in-place edit (or a load_state_dict) of ANY of them bumps its version
        return tuple((p.data_ptr(), p._version) for p in self.state_dict(keep_vars=True).values())

    def _engine(self, device):
        """The native net of `device`, (re)packed from the weights of the module that owns them.  Called on the master
        or on a DataParallel replica (whose own parameters()/state_dict() are empty); replicas run in threads."""
        master = self._master[0]
        idx = device.index if device.index is not None else torch.cuda.current_device()
        with master._lock:
            sig = master._signature()
            if len(sig) != nat.NUM_TENSORS:
                raise nat.B200PoseError("rtpose_model: expected %d weight tensors, found %d" % (nat.NUM_TENSORS, len(sig)))
            cached = master._engines.get(idx)
            if cached is None or cached[0] != sig:
                net = cached[1] if cached is not None else NativeNet(idx)
                arrays = [p.detach().to(torch.float32).cpu().contiguous().numpy()
                          for p in master.state_dict(keep_vars=True).values()]
                net.load_state_dict_arrays(arrays)
                master._engines[idx] = (sig, net)
            return master._engines[idx][1]

    def __deepcopy__(self, memo):
        # the copy owns its own weights, engines and lock (a lock cannot be deep-copied)
        import copy
        new = self.__class__.__new__(self.__class__)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            if k in ("_engines", "_lock", "_master", "_pose_engines"):
                continue
            new.__dict__[k] = copy.deepcopy(v, memo)
        new.__dict__["_engines"] = {}
        new.__dict__["_lock"] = threading.Lock()
        new.__dict__["_master"] = [new]
        return new

    def __getstate__(self):
        st = self.__dict__.copy()
        for k in ("_engines", "_lock", "_master", "_pose_engines"):
            st.pop(k, None)
        return st

    def __setstate__(self, st):
        self.__dict__.update(st)
        self._engines = {}
        self._lock = threading.Lock()
        self._master = [self]

    def maps_from_frame(self, img, preprocess, dest_size, factor):
        """The device-side body of get_outputs (evaluate/coco_eval.py:80-114) for one raw uint8 BGR frame: the frame
        goes to the GPU as bytes, crop_with_factor (bilinear resize + zero padding, bit-identical to cv2's) and the
        `preprocess` normalisation run there, fused into the first convolution's load, and only the two final maps come
        back.  Returns (paf [1,38,h,w], heat [1,19,h,w]) CUDA tensors and im_scale."""
        import ctypes
        import numpy as np
        master = self._master[0]
        device = next(master.parameters()).device
        if device.type != "cuda":
            raise nat.B200PoseError("the model must be on a CUDA device (model.cuda()): this build has no CPU fallback")
        if self.precision not in nat.MODES:
            raise ValueError("precision must be one of %s" % list(nat.MODES))
        net = self._engine(device)
        net.set_preprocess(preprocess)
        img = np.ascontiguousarray(img)
        sh, sw = img.shape[:2]
        scale, _, (ph, pw) = nat.crop_geometry(sh, sw, dest_size, factor)
        with torch.cuda.device(device):
            stream = torch.cuda.current_stream().cuda_stream
            frame = torch.empty((1, ph, pw, 3), dtype=torch.uint8, device=device)
            nat.check(nat.lib().b200pose_net_crop_with_factor(net._h, ctypes.c_void_p(img.ctypes.data), 0, 1, sh, sw,
                                                              int(dest_size), int(factor), ctypes.c_void_p(frame.data_ptr()),
                                                              1, ctypes.c_void_p(stream)), "b200pose_net_crop_with_factor")
            paf = torch.empty((1, 38, ph // 8, pw // 8), dtype=torch.float32, device=device)
            heat = torch.empty((1, 19, ph // 8, pw // 8), dtype=torch.float32, device=device)
            net.forward_u8_ptr(frame.data_ptr(), True, 1, ph, pw, nat.MODES[self.precision],
                               [0] * 10 + [paf.data_ptr(), heat.data_ptr()], True, stream)
        return paf, heat, scale

    def pose_engine(self, batch_cap=32, peak_cap=2048, human_cap=2048):
        """The batched fused engine (network + post-processing, maps never leave the device) around this module's native
        net and weights; cached per (device, precision, capacities).  evaluate.coco_eval.run_eval and the streaming
        front-ends use it."""
        from ...engine import PoseEngine
        master = self._master[0]
        device = next(master.parameters()).device
        if device.type != "cuda":
            raise nat.B200PoseError("the model must be on a CUDA device (model.cuda()): this build has no CPU fallback")
        net = self._engine(device)
        idx = device.index if device.index is not None else torch.cuda.current_device()
        key = (idx, self.precision, batch_cap, peak_cap, human_cap)
        with master._lock:
            cache = master.__dict__.setdefault("_pose_engines", {})
            if key not in cache:
                cache[key] = PoseEngine.from_net(net, self.precision, batch_cap, peak_cap, human_cap)
            return cache[key]

    def forward(self, x):
        if not x.is_cuda:
            raise nat.B200PoseError("rtpose_model.forward needs a CUDA tensor: this build has no CPU fallback")
        if self.precision not in nat.MODES:
            raise ValueError("precision must be one of %s" % list(nat.MODES))
        x = x.contiguous().to(torch.float32)
        n, c, H, W = x.shape
        if c != 3 or H % 8 or W % 8:
            raise ValueError("expected [N,3,H,W] with H, W multiples of 8, got %s" % (tuple(x.shape),))
        net = self._engine(x.device)
        h, w = H // 8, W // 8
        saved = [torch.empty((n, 38 if i % 2 == 0 else 19, h, w), dtype=torch.float32, device=x.device)
                 for i in range(12)]
        with torch.cuda.device(x.device):
            stream = torch.cuda.current_stream().cuda_stream
            net.forward_ptr(x.data_ptr(), True, n, H, W, nat.MODES[self.precision], [t.data_ptr() for t in saved], True,
                            stream)
        return (saved[-2], saved[-1]), saved


def get_model(trunk='vgg19'):
    """rtpose_vgg.py:60.  Only the VGG19 trunk exists on this path (BASELINE.json north_star)."""
    if trunk != 'vgg19':
        raise NotImplementedError("only trunk='vgg19' is built for the H100 path")
    return rtpose_model()


def use_vgg(model):
    """rtpose_vgg.py:235-251 downloads ImageNet VGG19 weights; there is no network here."""
    raise RuntimeError("use_vgg() needs network access (torchvision VGG19 weights); load a checkpoint instead")
