"""CPU: COCO keypoint evaluation (DESIGN.md 2.16) - the oracle (oracle/coco_kpt_eval.py, pycocotools' COCOeval for
keypoints restated) on hand-computable cases, and csrc/coco_eval_core.h compiled for the host, split the way the kernels
run it, against the oracle: precision and recall identical, OKS within 4 ulp, on the hand cases and on seeded
datasets; numpy's summation order; loadRes's refusals; the kernels' resource use."""
import os
import subprocess

import numpy as np
import pytest

import coco_eval_check as ce
from conftest import pkg_module


@pytest.fixture(scope="module")
def core(tmp_path_factory):
    return ce.compile_core(str(tmp_path_factory.mktemp("coco_eval") / "libcocoevalcore.so"))


@pytest.fixture(scope="module")
def cases():
    return ce.hand_cases()


def _one(stats):
    """1.0 up to the mean's rounding (a mean of 1010 ones need not be exactly 1)."""
    return np.allclose(stats, 1.0, rtol=0, atol=1e-12)


def _oracle(cases, name):
    return ce.oracle(*cases[name])


def test_params_are_numpys():
    from oracle import coco_kpt_eval as ok
    eng = pkg_module("engine")
    assert eng.COCO_IOU_THRS[8] == 0.8999999999999999 and np.array_equal(eng.COCO_IOU_THRS, ok.IOU_THRS)
    assert np.array_equal(eng.COCO_REC_THRS, ok.REC_THRS) and eng.COCO_REC_THRS[7] == np.linspace(0, 1, 101)[7]


def test_sum_order_is_numpys(core):
    rs = np.random.RandomState(3)
    for trial in range(4000):
        n = rs.randint(1, 18)
        a = rs.choice([1e16, 1.0, -1e16, 3.3, 1e-17], n) if trial % 2 else np.exp(-rs.exponential(3, n))
        a = np.ascontiguousarray(a, np.float64)
        assert core.core_sum(a.ctypes.data, n) == np.sum(a), (n, a)
    assert np.sum([1e16, 1, 1, 1, 1, 1, 1, 1, 1, -1e16, 1, 1]) == 10.0


def test_perfect_detections_give_every_stat_one(cases):
    assert _one(_oracle(cases, "perfect").stats)


def test_one_detection_at_a_known_oks(cases):
    from oracle import coco_kpt_eval as ok
    gt, rs, ids = cases["known_oks"]
    ev = ce.oracle(gt, rs, ids)
    g = np.array(gt["annotations"][0]["keypoints"]).reshape(17, 3)
    e = 36.0 / ((ok.SIGMAS * 2) ** 2) / (20000 + np.spacing(1)) / 2      # every part 6 px off in x
    oks = np.sum(np.exp(-e)) / 17
    assert np.all(g[:, 2] > 0) and abs(ev.ious[1, 1][0, 0] - oks) < 1e-15
    want = np.where(ok.IOU_THRS <= oks, 1.0, 0.0)
    assert np.array_equal(ev.precision[:, :, 0, 0, 0], np.repeat(want[:, None], 101, 1) / (1 + np.spacing(1)))
    assert 0 < ev.stats[0] < 1 and ev.stats[1] == ev.precision[0, :, 0, 0, 0].mean()


def test_crowd_gt_is_matched_many_times(cases):
    ev = _oracle(cases, "crowd")
    assert np.all(ev.precision[:, :, 0, 0, 0] == 1 / (1 + np.spacing(1)))      # the three detections on the crowd gt are ignored, not fp


def test_gt_without_keypoints_uses_the_enlarged_box(cases):
    ev = _oracle(cases, "no_keypoints")
    m = ev.ious[1, 1]          # detections by score: inside the enlarged box, outside it, the perfect one
    assert m[0, 1] == 1.0 and 0 < m[1, 1] < 1
    x0, x1, y0, y1 = 280 - 40, 280 + 80, 150 - 100, 150 + 200
    from oracle import coco_kpt_eval as ok
    d = np.array(cases["no_keypoints"][1][2]["keypoints"]).reshape(17, 3)
    dx = np.maximum(0, x0 - d[:, 0]) + np.maximum(0, d[:, 0] - x1)
    dy = np.maximum(0, y0 - d[:, 1]) + np.maximum(0, d[:, 1] - y1)
    e = (dx ** 2 + dy ** 2) / ((ok.SIGMAS * 2) ** 2) / (2500 + np.spacing(1)) / 2
    assert m[1, 1] == np.sum(np.exp(-e)) / 17 and m[1, 1] < 0.5
    # by score: the detection inside the box matches the ignored gt (ignored), the outside one is fp, the perfect one tp
    assert np.all(ev.precision[:, :, 0, 0, 0] == 1 / (2 + np.spacing(1)))


def test_area_bounds_are_inclusive(cases):
    ev = _oracle(cases, "area_bounds")
    assert _one(ev.stats)      # 32^2 is medium, 96^2 medium and large


def test_truncation_after_sorting(cases):
    ev = _oracle(cases, "truncation")
    assert ev.stats[0] == 0.0 and ev.stats[5] == 0.0


def test_no_gt_in_a_range_gives_minus_one(cases):
    ev = _oracle(cases, "empty_range")
    assert np.all(ev.precision[:, :, 0, 1, 0] == -1) and np.all(ev.recall[:, 0, 1, 0] == -1)
    assert ev.stats[3] == -1 and ev.stats[8] == -1 and _one(ev.stats[0])


def test_tied_oks_goes_to_the_last_gt(cases):
    ev = _oracle(cases, "tie_last")
    m = ev.ious[1, 1]
    assert m[0, 0] == m[0, 1] and m[1, 0] == 1.0 and m[1, 1] < 0.5
    assert _one(ev.stats[1])      # A took gt 2, so B matched gt 1 at IoU .5


def test_equal_scores_rank_by_image_id_then_list_order(cases):
    ev = _oracle(cases, "equal_scores")
    # global order: image 3's fp, its tp, then image 5's tp, fp, tp
    tp = np.cumsum([0, 1, 1, 0, 1])
    fp = np.cumsum([1, 0, 0, 1, 0])
    pr = tp / (tp + fp + np.spacing(1))
    assert ev.precision[0, 100, 0, 0, 0] == pr[-1] and ev.recall[0, 0, 0, 0] == 1.0
    assert ev.precision[0, 0, 0, 0, 0] == max(pr)


def test_detection_area_spans_the_zero_parts(cases, core):
    gt, rs, ids = cases["zero_parts"]
    d = np.ascontiguousarray(np.array(rs[1]["keypoints"]).reshape(17, 3), np.float64)
    assert core.core_dt_area(d.ctypes.data) == (d[:, 0].max() - 0) * (d[:, 1].max() - 0)
    ev = ce.oracle(gt, rs, ids)
    assert _one(ev.stats[3]) and abs(ev.stats[0] - 0.5) < 1e-12      # medium: the far detection is large, so ignored


def test_results_outside_img_ids_are_left_out_outside_the_file_refused(cases):
    nat = pkg_module("_native")
    eng = pkg_module("engine")
    assert _one(_oracle(cases, "outside_img_ids").stats[[0, 5]])
    gt, rs, ids = cases["outside_img_ids"]
    with pytest.raises(nat.B200PoseError, match=r"results\[1\]: image_id 7 is not in the gt file"):
        eng.coco_pack(gt, [rs[0], dict(rs[1], image_id=7)], ids)
    with pytest.raises(AssertionError):
        ce.oracle(gt, [rs[0], dict(rs[1], image_id=7)], ids)
    with pytest.raises(nat.B200PoseError, match="results is empty"):
        eng.coco_pack(gt, [], ids)
    with pytest.raises(nat.B200PoseError, match="keypoints has 50 values"):
        eng.coco_pack(gt, [dict(rs[0], keypoints=rs[0]["keypoints"][:50])], ids)


@pytest.mark.parametrize("name", sorted(ce.hand_cases()))
def test_core_equals_oracle_on_hand_cases(core, cases, name):
    gt, rs, ids = cases[name]
    ev = ce.oracle(gt, rs, ids)
    ce.assert_margins(ev)
    prec, rec, oks = ce.core_eval(core, gt, rs, ids)
    assert np.array_equal(prec, ev.precision) and np.array_equal(rec, ev.recall)
    assert sorted(oks) == sorted(k for k, v in ev.ious.items() if len(v))
    assert max([ce.ulps(oks[k], ev.ious[k]) for k in oks] + [0]) <= 4


@pytest.mark.parametrize("seed,scores,cats", [(1, "const", (1,)), (2, "ties", (1,)), (3, "ties", (1, 4))])
def test_core_equals_oracle_on_random_units(core, seed, scores, cats):
    gt, rs, ids = ce.scenario(seed, n_images=300, n_person=160, n_gts=650, n_dets=1500, scores=scores, cats=cats)
    ev = ce.oracle(gt, rs, ids)
    ce.assert_margins(ev)
    prec, rec, oks = ce.core_eval(core, gt, rs, ids)
    assert np.array_equal(prec, ev.precision) and np.array_equal(rec, ev.recall)
    assert max(ce.ulps(oks[k], ev.ious[k]) for k in oks) <= 4
    assert np.any(ev.precision > 0)


def test_permuting_image_blocks_keeps_precision(core):
    gt, rs, ids = ce.scenario(5, n_images=200, n_person=120, n_gts=400, n_dets=900, scores="ties")
    by_img = {}
    for r in rs:
        by_img.setdefault(r["image_id"], []).append(r)
    keys = list(by_img)
    np.random.RandomState(0).shuffle(keys)
    perm = [r for k in keys for r in by_img[k]]
    a, b = ce.oracle(gt, rs, ids), ce.oracle(gt, perm, ids)
    assert np.array_equal(a.precision, b.precision) and np.array_equal(a.stats, b.stats)
    assert np.array_equal(ce.core_eval(core, gt, perm, ids)[0], a.precision)


def test_coco_eval_kernels_do_not_spill(built):
    import __graft_entry__ as g
    nvcc = os.environ.get("NVCC", "nvcc")
    r = subprocess.run([nvcc] + g.NVCC_FLAGS + ["-Xptxas", "-v", "-c", os.path.join(g.CSRC, "coco_eval.cu"),
                        "-o", os.devnull], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=True)
    blocks = r.stdout.split("Compiling entry function")[1:]
    names = [b.split("'")[1] for b in blocks]
    assert len(blocks) == 4 and all("coco" in n for n in names), names
    for b in blocks:
        assert "0 bytes spill stores, 0 bytes spill loads" in b, b


def test_c_abi_declares_the_call():
    nat = pkg_module("_native")
    from conftest import ROOT
    assert "b200pose_coco_kpt_eval" in nat.EXPORTED
    assert "int b200pose_coco_kpt_eval(" in open(os.path.join(ROOT, "include", "b200pose.h")).read()
