"""Import-compatibility module for /root/reference/lib/network/openpose.py.

evaluate/evaluation.py:6 imports `OpenPose_Model` and `use_vgg` from here but only ever builds the rtpose VGG19 model
(evaluation.py:19-20; the OpenPose_Model line is commented out).  The dense-block `OpenPose_Model` family is a
different network and is outside the H100 hot path (SURVEY.md section 8 scope table), so constructing it fails loudly
instead of silently falling back to a PyTorch implementation."""
from .rtpose_vgg import use_vgg  # noqa: F401  (openpose.py:212 defines the same helper)


class OpenPose_Model:
    def __init__(self, *args, **kwargs):
        raise NotImplementedError("OpenPose_Model (lib/network/openpose.py:111) is not part of the H100 inference path; "
                                  "use lib.network.rtpose_vgg.get_model('vgg19')")
