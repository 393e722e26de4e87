"""Pipelined capture -> infer -> draw loop for video files and cameras (SURVEY.md 8f rank 4).

The reference's front-ends (/root/reference/video_demo.py:85-125, demo/web_demo.py:51-71) read a frame, call
get_outputs + paf_to_pose_cpp, draw, and only then read the next frame.  Here frames are grouped into batches and two
batches are kept in flight: while the GPU works on batch i+1 (upload, crop_with_factor, network, post-processing - the
fused engine), the host decodes the next frames and draws batch i.  The drawing itself is the reference's draw_humans, or its device
restatement (draw='device' / 'cuda', DESIGN.md 2.12).
"""
import numpy as np

from .lib.utils.common import draw_humans
from .lib.utils.paf_to_pose import humans_from_rows
from . import _native as nat
from . import engine


def frames_of(capture, rotate_code=None, limit=None):
    """Frames of a cv2.VideoCapture-like object until it runs dry (optionally rotated, as video_demo.py:27-45 does)."""
    import cv2
    k = 0
    while limit is None or k < limit:
        ok, frame = capture.read()
        if not ok or frame is None:
            return
        if rotate_code is not None:
            frame = cv2.rotate(frame, rotate_code)
        yield frame
        k += 1


class PoseStream:
    """for frame, humans, drawn in PoseStream(model, frames, batch=8): ...

    model: a module from lib.network.rtpose_vgg.get_model() (bare or DataParallel-wrapped) on a CUDA device, or a
    PoseEngine (e.g. engine.openpose_engine's, to run OpenPose_Model); the stream then runs on that engine's net and
    post-processing, and submits batches of at most its batch_cap frames.
    frames: any iterator of uint8 BGR frames of ONE shape.  batch=1 minimises latency (camera), larger batches raise
    throughput (files).  `draw=False` skips the rendering.  draw=True draws with the reference's draw_humans on the
    host; draw='device' yields the same numpy frames drawn on the GPU (PoseEngine.draw_humans); draw='cuda' yields the
    drawn frames as CUDA uint8 tensors [h, w, 3] and downloads nothing but the person rows.
    format 'nv12' / 'i420' (frames as PoseEngine.infer_frames_async takes them, e.g. decoder surfaces already on the GPU)
    and rotate (degrees clockwise; nat.rotation_of maps cv2.ROTATE_* codes): the frames are converted and rotated on
    the device; with draw=True or 'device' each batch is also converted back to host BGR for the drawing, and the
    converted frame is the one yielded; with draw='cuda' it is converted into a device tensor instead."""

    def __init__(self, model, frames, batch=8, preprocess='rtpose', dest_size=368, factor=8, thresh=0.1, draw=True,
                 format='bgr', rotate=None):
        if isinstance(model, engine.PoseEngine):
            self.engine = model
            batch = min(max(1, int(batch)), model.post.batch_cap)
        else:
            core = getattr(model, "module", model)
            if not hasattr(core, "pose_engine"):
                raise nat.B200PoseError("PoseStream needs a model from lib.network.rtpose_vgg.get_model() or a PoseEngine")
            self.engine = core.pose_engine(batch_cap=max(1, int(batch)))
        self.engine.net.set_preprocess(preprocess)
        self.frames, self.batch = iter(frames), max(1, int(batch))
        if draw not in (True, False, 'device', 'cuda'):
            raise nat.B200PoseError("PoseStream: draw must be True, False, 'device' or 'cuda', got %r" % (draw,))
        self.dest_size, self.factor, self.thresh, self.draw = dest_size, factor, thresh, draw
        self.format, self.rotate = format, int(rotate or 0)

    def _next_batch(self):
        out = []
        for frame in self.frames:
            out.append(frame)
            if len(out) == self.batch:
                break
        return out

    def _finish(self, ticket, batch, size):
        rows = self.engine.fetch_arrays(ticket=ticket)
        _, _, (ph, pw) = nat.crop_geometry(size[0], size[1], self.dest_size, self.factor)
        if self.draw == 'device':
            drawn = self.engine.draw_humans([f.copy() for f in batch], ticket=ticket, net_sizes=[(ph, pw)] * len(batch))
        elif self.draw == 'cuda':
            drawn = self._device_batch(batch)
            self.engine.draw_humans(drawn, ticket=ticket, net_sizes=[(ph, pw)] * len(batch))
        for i, (frame, r) in enumerate(zip(batch, rows)):
            humans = humans_from_rows(r, pw, ph)
            # draw_humans scales by the ORIGINAL frame size, like the reference front-ends (coordinates are normalised by
            # the padded network input, padding included - the same small offset the reference has)
            if self.draw is True:
                yield frame, humans, draw_humans(frame, humans, imgcopy=True)
            else:
                yield frame, humans, (drawn[i] if self.draw else None)

    def _device_batch(self, batch):
        """draw='cuda': the frames to draw on as one CUDA tensor [n, h, w, 3] (a copy: the yielded frames stay as
        they are)."""
        import torch
        if isinstance(batch, torch.Tensor):
            return batch.clone()
        dev = "cuda:%d" % self.engine.net.device_index
        if all(isinstance(f, torch.Tensor) for f in batch):
            return torch.stack(list(batch)).to(dev)
        return torch.from_numpy(np.stack(batch)).to(dev)

    def __iter__(self):
        pending = None
        while True:
            batch = self._next_batch()
            if batch and self.format == 'bgr' and not self.rotate:
                if any(f.shape != batch[0].shape for f in batch):
                    raise nat.B200PoseError("PoseStream: the frames of a stream must share one shape")
                ticket = self.engine.submit_images(batch, self.dest_size, self.factor, self.thresh)
                size = batch[0].shape[:2]
            elif batch:
                sizes = {engine.rotated_size(h, w, self.rotate) for h, w in engine.frame_table(batch, self.format)[3]}
                if len(sizes) != 1:
                    raise nat.B200PoseError("PoseStream: the frames of a stream must share one shape")
                size = sizes.pop()
                # host BGR frames to draw on: one more conversion launch and its download, before the submission so
                # that its synchronisation waits only for the batch already in flight
                if self.draw == 'cuda':
                    shown = self.engine.net.convert_frames(batch, self.format, self.rotate, device=True)
                elif self.draw:
                    shown = self.engine.net.convert_frames(batch, self.format, self.rotate)
                else:
                    shown = batch
                ticket = self.engine.infer_frames_async(batch, self.format, self.rotate, self.dest_size, self.factor,
                                                        self.thresh)
                batch = shown
            if pending is not None:
                yield from self._finish(*pending)
            if len(batch) == 0:
                return
            pending = (ticket, batch, size)
