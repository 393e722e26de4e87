"""GPU (-m gpu): run_eval's batched loop writes the visualisations named .jpg / .jpeg on the device (persons drawn on
the uploaded frames, encoded from the same buffer, DESIGN.md 2.14): over a directory of JPEG images of mixed sizes and
orientations, several ragged batches per pass, its files are byte for byte those of the per-image loop
(get_outputs + paf_to_pose_cpp + draw_humans + cv2.imwrite), with the same COCO records."""
import json
import sys
import types

import numpy as np
import pytest
import torch

from conftest import pkg_module

pytestmark = pytest.mark.gpu


def _model(he_sd):
    from lib.network.rtpose_vgg import get_model
    model = get_model("vgg19")
    model.load_state_dict(he_sd)
    model = model.cuda().float().eval()
    model.precision = "bf16"
    return model


class Opaque(torch.nn.Module):
    """Hides the device fast paths: coco_eval then runs the reference's own per-image sequence through the same net."""

    def __init__(self, inner):
        super().__init__()
        self.inner = inner

    def forward(self, x):
        return self.inner(x)


def test_batched_jpeg_visualisations_equal_the_per_image_loop(built, he_sd, monkeypatch, tmp_path):
    import cv2
    ev = pkg_module("evaluate.coco_eval")
    img_dir = tmp_path / "img"
    img_dir.mkdir()
    rs = np.random.RandomState(8)
    shapes = [(120, 160), (200, 230), (160, 120), (368, 368), (200, 230), (97, 64), (120, 160), (230, 200)]
    names = ["im%d.%s" % (i, ("jpg", "jpeg", "JPG", "png")[i % 4]) for i in range(len(shapes))]
    for name, (h, w) in zip(names, shapes):
        cv2.imwrite(str(img_dir / name), rs.randint(0, 256, (h, w, 3)).astype(np.uint8))
    seen = {}

    class COCO:
        def __init__(self, anno): pass
        def getCatIds(self, catNms): return [1]
        def getImgIds(self, catIds): return list(range(len(names)))
        def loadImgs(self, i): return [{"file_name": names[i]}]
        def loadRes(self, path): seen["results"] = json.load(open(path)); return "dt"

    class COCOeval:
        def __init__(self, gt, dt, kind): self.params = types.SimpleNamespace(imgIds=None); self.stats = [0.25]
        def evaluate(self): pass
        def accumulate(self): pass
        def summarize(self): pass
    for name, attrs in (("pycocotools", {}), ("pycocotools.coco", {"COCO": COCO}), ("pycocotools.cocoeval", {"COCOeval": COCOeval})):
        m = types.ModuleType(name)
        m.__dict__.update(attrs)
        monkeypatch.setitem(sys.modules, name, m)
    monkeypatch.chdir(tmp_path)
    monkeypatch.setattr(ev, "EVAL_BATCH", 5)          # several passes, several ragged batches per pass
    calls = []
    write_vis_device = ev.write_vis_device
    monkeypatch.setattr(ev, "write_vis_device", lambda *a: calls.append(len(a[5])) or write_vis_device(*a))
    model = _model(he_sd)
    out = {}
    for tag, mdl in (("batched", model), ("serial", Opaque(model))):
        vis = tmp_path / ("vis_" + tag)
        vis.mkdir()
        with torch.no_grad():
            assert ev.run_eval(str(img_dir), "anno.json", str(vis), model=mdl, preprocess="vgg") == 0.25
        out[tag] = (seen["results"], {n: (vis / n).read_bytes() for n in names})
    assert sum(calls) == sum(1 for n in names if not n.endswith("png")) and len(calls) >= 2
    assert len(out["batched"][0]) > 20
    assert out["batched"][0] == out["serial"][0]
    for n in names:
        assert out["batched"][1][n] == out["serial"][1][n], n
