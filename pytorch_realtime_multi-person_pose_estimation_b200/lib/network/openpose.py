"""Import-compatibility module for /root/reference/lib/network/openpose.py.

evaluate/evaluation.py:6 imports `OpenPose_Model` and `use_vgg` from here but only ever builds the rtpose VGG19 model
(evaluation.py:19-20; the OpenPose_Model line is commented out).  The dense-block `OpenPose_Model` network itself runs on
the device through engine.openpose_engine / NativeNet.openpose (DESIGN.md 2.11).  The nn.Module stays a stub that fails
loudly: no reference script could use it, since its forward returns (paf, heat) tuples where get_outputs
(coco_eval.py:110-112) expects tensors."""
from .rtpose_vgg import use_vgg  # noqa: F401  (openpose.py:212 defines the same helper)


class OpenPose_Model:
    def __init__(self, *args, **kwargs):
        raise NotImplementedError("OpenPose_Model (lib/network/openpose.py:111) is not available as a module: load its "
                                  "state_dict with engine.openpose_engine(state_dict, l2_stages, l1_stages) to run it "
                                  "on the device, or use lib.network.rtpose_vgg.get_model('vgg19')")
