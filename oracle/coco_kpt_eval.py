"""Float64 numpy restatement of pycocotools 2.0's COCOeval(cocoGt, cocoDt, 'keypoints') with default Params:
loadRes for keypoint results, _prepare, computeOks, evaluateImg, accumulate and summarize, written from their
documented semantics (DESIGN.md 2.16) in pycocotools' own loop structure.  Used by the tests and tools/bench_coco_eval.py
as the reference for engine.coco_keypoint_eval; nothing in the package imports it."""
import copy
from collections import defaultdict

import numpy as np

IOU_THRS = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
REC_THRS = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
MAX_DETS = 20
AREA_RNG = [[0 ** 2, 1e5 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
AREA_LBL = ['all', 'medium', 'large']
SIGMAS = np.array([.26, .25, .25, .35, .35, .79, .79, .72, .72, .62, .62, 1.07, 1.07, .87, .87, .89, .89]) / 10.0


def load_res(gt, results):
    """COCO.loadRes for keypoint results: box over all 17 x and y values, area, id = index + 1."""
    anns = copy.deepcopy(list(results))
    assert type(anns) == list
    if not anns:
        raise IndexError("loadRes: empty result list")
    img_ids = {im['id'] for im in gt['images']}
    if not {a['image_id'] for a in anns} <= img_ids:
        raise AssertionError("Results do not correspond to current coco set")
    for i, ann in enumerate(anns):
        s = ann['keypoints']
        x, y = s[0::3], s[1::3]
        x0, x1, y0, y1 = np.min(x), np.max(x), np.min(y), np.max(y)
        ann['area'] = (x1 - x0) * (y1 - y0)
        ann['id'] = i + 1
        ann['bbox'] = [x0, y0, x1 - x0, y1 - y0]
    return anns


class Eval:
    """evaluate() + accumulate() + summarize() of one evaluation; the attributes follow COCOeval's."""

    def __init__(self, gt, results, img_ids):
        self.gt = gt
        self.dts_all = load_res(gt, results)
        self.img_ids = list(np.unique(img_ids))
        self.cat_ids = sorted(c['id'] for c in gt['categories'])
        self.evaluate()
        self.accumulate()
        self.summarize()

    def _prepare(self):
        cats = set(self.cat_ids)
        by_img = defaultdict(list)
        for ann in self.gt['annotations']:
            by_img[ann['image_id']].append(ann)
        gts = [g for i in self.img_ids for g in by_img.get(i, []) if g['category_id'] in cats]
        dt_by_img = defaultdict(list)
        for d in self.dts_all:
            dt_by_img[d['image_id']].append(d)
        dts = [d for i in self.img_ids for d in dt_by_img.get(i, []) if d['category_id'] in cats]
        self._gts, self._dts = defaultdict(list), defaultdict(list)
        for g in gts:
            g = dict(g)
            g['ignore'] = 'iscrowd' in g and g['iscrowd']
            g['ignore'] = (g['num_keypoints'] == 0) or g['ignore']
            self._gts[g['image_id'], g['category_id']].append(g)
        for d in dts:
            self._dts[d['image_id'], d['category_id']].append(d)

    def compute_oks(self, img_id, cat_id):
        gts, dts = self._gts[img_id, cat_id], self._dts[img_id, cat_id]
        inds = np.argsort([-d['score'] for d in dts], kind='mergesort')
        dts = [dts[i] for i in inds][:MAX_DETS]
        if len(gts) == 0 or len(dts) == 0:
            return []
        ious = np.zeros((len(dts), len(gts)))
        var = (SIGMAS * 2) ** 2
        k = len(SIGMAS)
        for j, gt in enumerate(gts):
            g = np.array(gt['keypoints'], np.float64)
            xg, yg, vg = g[0::3], g[1::3], g[2::3]
            k1 = np.count_nonzero(vg > 0)
            bb = gt['bbox']
            x0, x1 = bb[0] - bb[2], bb[0] + bb[2] * 2
            y0, y1 = bb[1] - bb[3], bb[1] + bb[3] * 2
            for i, dt in enumerate(dts):
                d = np.array(dt['keypoints'], np.float64)
                xd, yd = d[0::3], d[1::3]
                if k1 > 0:
                    dx, dy = xd - xg, yd - yg
                else:
                    z = np.zeros(k)
                    dx = np.max((z, x0 - xd), axis=0) + np.max((z, xd - x1), axis=0)
                    dy = np.max((z, y0 - yd), axis=0) + np.max((z, yd - y1), axis=0)
                e = (dx ** 2 + dy ** 2) / var / (gt['area'] + np.spacing(1)) / 2
                if k1 > 0:
                    e = e[vg > 0]
                ious[i, j] = np.sum(np.exp(-e)) / e.shape[0]
        return ious

    def evaluate_img(self, img_id, cat_id, a_rng):
        gt, dt = self._gts[img_id, cat_id], self._dts[img_id, cat_id]
        if len(gt) == 0 and len(dt) == 0:
            return None
        for g in gt:
            g['_ignore'] = 1 if (g['ignore'] or g['area'] < a_rng[0] or g['area'] > a_rng[1]) else 0
        gtind = np.argsort([g['_ignore'] for g in gt], kind='mergesort')
        gt = [gt[i] for i in gtind]
        dtind = np.argsort([-d['score'] for d in dt], kind='mergesort')
        dt = [dt[i] for i in dtind[0:MAX_DETS]]
        iscrowd = [int(o.get('iscrowd', 0)) for o in gt]
        ious = self.ious[img_id, cat_id]
        ious = ious[:, gtind] if len(ious) > 0 else ious
        T, G, D = len(IOU_THRS), len(gt), len(dt)
        gtm, dtm = np.zeros((T, G)), np.zeros((T, D))
        gt_ig = np.array([g['_ignore'] for g in gt])
        dt_ig = np.zeros((T, D))
        if not len(ious) == 0:
            for tind, t in enumerate(IOU_THRS):
                for dind, d in enumerate(dt):
                    iou = min([t, 1 - 1e-10])
                    m = -1
                    for gind, g in enumerate(gt):
                        if gtm[tind, gind] > 0 and not iscrowd[gind]:
                            continue
                        if m > -1 and gt_ig[m] == 0 and gt_ig[gind] == 1:
                            break
                        if ious[dind, gind] < iou:
                            continue
                        iou = ious[dind, gind]
                        m = gind
                    if m == -1:
                        continue
                    dt_ig[tind, dind] = gt_ig[m]
                    dtm[tind, dind] = gt[m]['id']
                    gtm[tind, m] = d['id']
        a = np.array([d['area'] < a_rng[0] or d['area'] > a_rng[1] for d in dt]).reshape((1, len(dt)))
        dt_ig = np.logical_or(dt_ig, np.logical_and(dtm == 0, np.repeat(a, T, 0)))
        return {'dtMatches': dtm, 'dtScores': [d['score'] for d in dt], 'gtIgnore': gt_ig, 'dtIgnore': dt_ig}

    def evaluate(self):
        self._prepare()
        self.ious = {(i, c): self.compute_oks(i, c) for i in self.img_ids for c in self.cat_ids}
        self.eval_imgs = [self.evaluate_img(i, c, a) for c in self.cat_ids for a in AREA_RNG for i in self.img_ids]

    def accumulate(self):
        T, R, K, A, M = len(IOU_THRS), len(REC_THRS), len(self.cat_ids), len(AREA_RNG), 1
        precision = -np.ones((T, R, K, A, M))
        recall = -np.ones((T, K, A, M))
        I0, A0 = len(self.img_ids), len(AREA_RNG)
        for k in range(K):
            for a in range(A):
                E = [self.eval_imgs[k * A0 * I0 + a * I0 + i] for i in range(I0)]
                E = [e for e in E if e is not None]
                if len(E) == 0:
                    continue
                dt_scores = np.concatenate([e['dtScores'][0:MAX_DETS] for e in E])
                inds = np.argsort(-dt_scores, kind='mergesort')
                dtm = np.concatenate([e['dtMatches'][:, 0:MAX_DETS] for e in E], axis=1)[:, inds]
                dt_ig = np.concatenate([e['dtIgnore'][:, 0:MAX_DETS] for e in E], axis=1)[:, inds]
                gt_ig = np.concatenate([e['gtIgnore'] for e in E])
                npig = np.count_nonzero(gt_ig == 0)
                if npig == 0:
                    continue
                tps = np.logical_and(dtm, np.logical_not(dt_ig))
                fps = np.logical_and(np.logical_not(dtm), np.logical_not(dt_ig))
                tp_sum = np.cumsum(tps, axis=1).astype(dtype=np.float64)
                fp_sum = np.cumsum(fps, axis=1).astype(dtype=np.float64)
                for t, (tp, fp) in enumerate(zip(tp_sum, fp_sum)):
                    tp, fp = np.array(tp), np.array(fp)
                    nd = len(tp)
                    rc = tp / npig
                    pr = tp / (fp + tp + np.spacing(1))
                    q = np.zeros((R,))
                    recall[t, k, a, 0] = rc[-1] if nd else 0
                    pr, q = pr.tolist(), q.tolist()
                    for i in range(nd - 1, 0, -1):
                        if pr[i] > pr[i - 1]:
                            pr[i - 1] = pr[i]
                    inds_r = np.searchsorted(rc, REC_THRS, side='left')
                    try:
                        for ri, pi in enumerate(inds_r):
                            q[ri] = pr[pi]
                    except IndexError:
                        pass
                    precision[t, :, k, a, 0] = np.array(q)
        self.precision, self.recall = precision, recall

    def summarize(self):
        self.stats, self.lines = summarize(self.precision, self.recall)


def summarize(precision, recall):
    """COCOeval._summarizeKps: (stats [10], the 10 printed lines)."""
    i_str = ' {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} ] = {:0.3f}'

    def one(ap, iou_thr=None, area='all'):
        aind = [i for i, lbl in enumerate(AREA_LBL) if lbl == area]
        s = precision if ap else recall
        if iou_thr is not None:
            s = s[np.where(iou_thr == IOU_THRS)[0]]
        s = s[:, :, :, aind, 0] if ap else s[:, :, aind, 0]
        mean_s = -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
        iou = '{:0.2f}:{:0.2f}'.format(IOU_THRS[0], IOU_THRS[-1]) if iou_thr is None else '{:0.2f}'.format(iou_thr)
        line = i_str.format('Average Precision' if ap else 'Average Recall', '(AP)' if ap else '(AR)', iou, area,
                            MAX_DETS, mean_s)
        return mean_s, line

    out = [one(ap, thr, area) for ap in (1, 0) for thr, area in ((None, 'all'), (.5, 'all'), (.75, 'all'),
                                                                  (None, 'medium'), (None, 'large'))]
    return np.array([s for s, _ in out], np.float64), [line for _, line in out]
