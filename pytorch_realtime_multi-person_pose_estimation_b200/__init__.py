"""H100-native OpenPose (rtpose VGG19) inference path.

The compute lives in libb200pose.so (hand-written sm_90a CUDA, C ABI in include/b200pose.h); this package is the
host-side mirror of the reference's Python interface for that path (lib.network.rtpose_vgg.get_model,
evaluate.coco_eval.get_outputs, lib.utils.paf_to_pose.paf_to_pose_cpp, lib.pafprocess) plus the batched engine.
There is no CPU fallback: importing works anywhere, running requires an H100 and the built library.
"""
from . import _native  # noqa: F401
