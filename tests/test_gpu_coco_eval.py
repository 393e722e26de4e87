"""GPU (-m gpu): COCO keypoint evaluation on the device (DESIGN.md 2.16) against the oracle (oracle/coco_kpt_eval.py):
precision and recall identical and the ten stats equal on the hand cases, on seeded val2017-sized evaluations (constant
and tied scores) and on a two-category file, with the exported OKS within 4 ulp; four launches per call at any size;
refusals that name their argument and leave no CUDA error behind; run_eval and evaluation.main end to end without
pycocotools."""
import json
import os
import sys

import numpy as np
import pytest

import coco_eval_check as ce
from conftest import pkg_module

pytestmark = pytest.mark.gpu


def _device_equals_oracle(gt, rs, ids):
    eng = pkg_module("engine")
    ev = ce.oracle(gt, rs, ids)
    ce.assert_margins(ev)
    got = eng.coco_keypoint_eval(gt, rs, ids, export_oks=True)
    assert np.array_equal(got.precision, ev.precision)
    assert np.array_equal(got.recall, ev.recall)
    assert np.array_equal(got.stats, ev.stats), (got.stats, ev.stats)
    assert sorted(got.oks) == sorted(k for k, v in ev.ious.items() if len(v))
    assert max([ce.ulps(got.oks[k], ev.ious[k]) for k in got.oks] + [0]) <= 4
    return got, ev


@pytest.mark.parametrize("name", sorted(ce.hand_cases()))
def test_device_equals_oracle_on_hand_cases(built, name):
    _device_equals_oracle(*ce.hand_cases()[name])


@pytest.mark.parametrize("seed,scores", [(11, "const"), (12, "ties"), (13, "const")])
def test_device_equals_oracle_at_val2017_scale(built, seed, scores):
    gt, rs, ids = ce.scenario(seed, scores=scores)
    got, ev = _device_equals_oracle(gt, rs, ids)
    assert len(rs) >= 25000 and len(gt["annotations"]) == 11000 and np.any(ev.precision > 0)
    print("seed %d %s: stats %s" % (seed, scores, np.round(got.stats, 4).tolist()))
    got.summarize()


def test_device_equals_oracle_on_two_categories(built):
    gt, rs, ids = ce.scenario(21, n_images=1500, n_person=900, n_gts=3500, n_dets=8000, scores="ties", cats=(1, 7))
    got, _ = _device_equals_oracle(gt, rs, ids)
    assert got.precision.shape == (10, 101, 2, 3, 1) and got.cat_ids == [1, 7]


def test_launch_count_is_fixed(built):
    nat, eng = pkg_module("_native"), pkg_module("engine")
    counts = []
    for n_images, n_person, n_gts, n_dets in ((10, 8, 20, 40), (5000, 2700, 11000, 25000)):
        gt, rs, ids = ce.scenario(31, n_images, n_person, n_gts, n_dets)
        before = nat.launch_count()
        eng.coco_keypoint_eval(gt, rs, ids)
        counts.append(nat.launch_count() - before)
    assert counts == [4, 4], counts


def test_refusals_name_their_argument(built):
    import torch
    nat, eng = pkg_module("_native"), pkg_module("engine")
    gt, rs, ids = ce.hand_cases()["perfect"]

    def bad(gt2, rs2, pattern):
        with pytest.raises(nat.B200PoseError, match=pattern):
            eng.coco_keypoint_eval(gt2, rs2, ids)

    a0 = gt["annotations"][0]
    bad(dict(gt, annotations=[dict(a0, id=0)] + gt["annotations"][1:]), rs, r"gt_id\[0\] is 0")
    bad(dict(gt, annotations=gt["annotations"] + [dict(a0)]), rs, r"gt_id\[\d+\] = 1 repeats an earlier gt")
    bad(gt, [dict(rs[0], score=float("nan"))] + rs[1:], r"dt_score\[0\] is not finite")
    bad(gt, [dict(rs[0], score=float("inf"))] + rs[1:], r"dt_score\[0\] is not finite")
    kp = list(rs[0]["keypoints"])
    kp[4] = float("nan")
    bad(gt, [dict(rs[0], keypoints=kp)] + rs[1:], "dt_kpt of detection 0 is not finite")
    bad(dict(gt, annotations=[dict(a0, area=float("inf"))] + gt["annotations"][1:]), rs, "gt_box of gt 0 is not finite")
    bad(gt, rs + [rs[0]] * 1025, r"unit_dt0: unit 0 has 1027 detections")
    bad(gt, [dict(rs[0], keypoints=kp[:48])], "keypoints has 48 values")
    bad(gt, [], "results is empty")
    torch.cuda.synchronize()
    assert torch.cuda.current_stream().query()
    got = eng.coco_keypoint_eval(gt, rs, ids)       # the library still works after every refusal
    assert np.allclose(got.stats, 1.0, rtol=0, atol=1e-12)


def _synthetic_coco(tmp_path, rs, n=40):
    """n JPEG images of mixed sizes (noise) and a person_keypoints file whose persons are generated."""
    import cv2
    img_dir = tmp_path / "val"
    img_dir.mkdir()
    images, anns = [], []
    for i in range(n):
        h, w = [(120, 160), (200, 230), (160, 120), (240, 240), (97, 64)][i % 5]
        iid = 1000 + 7 * i
        name = "%012d.jpg" % iid
        cv2.imwrite(str(img_dir / name), rs.randint(0, 256, (h, w, 3)).astype(np.uint8))
        images.append({"id": iid, "file_name": name, "height": h, "width": w})
        for j in range(i % 3):
            k = ce.skeleton(rs.uniform(20, w - 20), rs.uniform(20, h - 20), rs.uniform(4, 12))
            k[:, 2] = rs.choice([0, 2], 17, p=[.3, .7])
            anns.append(ce.ann(len(anns) + 1, iid, k, [k[:, 0].min(), k[:, 1].min(), 30, 40], rs.uniform(200, 3000)))
    anno = tmp_path / "person_keypoints.json"
    anno.write_text(json.dumps({"images": images, "annotations": anns,
                                "categories": [{"id": 1, "name": "person"}]}))
    return img_dir, anno


def test_run_eval_and_evaluation_main_without_pycocotools(built, he_sd, monkeypatch, tmp_path):
    import torch
    ev_mod = pkg_module("evaluate.coco_eval")
    evaluation = pkg_module("evaluate.evaluation")
    monkeypatch.setitem(sys.modules, "pycocotools", None)
    monkeypatch.chdir(tmp_path)
    img_dir, anno = _synthetic_coco(tmp_path, np.random.RandomState(4))
    records = []
    append_result = ev_mod.append_result
    monkeypatch.setattr(ev_mod, "append_result", lambda *a: append_result(*a) or records.append(list(a[3])))
    from lib.network.rtpose_vgg import get_model
    model = get_model("vgg19")
    model.load_state_dict(he_sd)
    model = model.cuda().float().eval()
    vis = tmp_path / "vis"
    vis.mkdir()
    with torch.no_grad():
        ap = ev_mod.run_eval(str(img_dir), str(anno), str(vis), model=model, preprocess="vgg")
    gt = json.loads(anno.read_text())
    ids = sorted({a["image_id"] for a in gt["annotations"]})      # run_eval's images: those with a person
    names = sorted(im["file_name"] for im in gt["images"] if im["id"] in ids)
    assert sorted(os.listdir(vis)) == names and not (tmp_path / "results.json").exists()
    out = records[-1]
    assert out, "the synthetic weights found no person"
    want = ce.oracle(gt, out, ids).stats[0]
    print("run_eval: %d records over %d images, AP %r" % (len(out), len(ids), ap))
    assert ap == want
    # evaluation.main, unmodified, on the same set with a Lightning-style checkpoint of the same weights
    ckpt = tmp_path / "ckpt.pth"
    torch.save({"state_dict": {"model." + k: v for k, v in he_sd.items()}}, str(ckpt))
    vis2 = tmp_path / "vis2"
    vis2.mkdir()
    got = evaluation.main(["--weight", str(ckpt), "--image-dir", str(img_dir), "--anno-file", str(anno),
                           "--vis-dir", str(vis2), "--preprocess", "vgg"])
    assert got == ap and sorted(os.listdir(vis2)) == names
