// Host build of the COCO keypoint evaluation core (csrc/coco_eval_core.h), split the way the kernels of coco_eval.cu
// run it: per unit the score ranks, the kept detections and the OKS block; per (unit, area range, threshold) the
// matching, each detection taking the best of the two candidate scans; per category the global order by rank
// counting; per (category, area range, threshold) the precision / recall walk.  The arguments are those of
// b200pose_coco_kpt_eval without the device.  COCO_EVAL_CORE overrides the header's path, so that a test can compile a
// copy with a planted mistake.
#ifndef COCO_EVAL_CORE
#define COCO_EVAL_CORE "../../pytorch_realtime_multi-person_pose_estimation_b200/csrc/coco_eval_core.h"
#endif
#include COCO_EVAL_CORE

#include <algorithm>
#include <vector>

using namespace b2p;

extern "C" double core_oks(const double* g, const double* box, const double* d) { return coco_oks(g, box, d); }
extern "C" double core_dt_area(const double* d) { return coco_dt_area(d); }
extern "C" double core_sum(const double* v, int n) { return coco_sum(v, n); }

// precision [10][101][n_cats][3], recall [10][n_cats][3], oks: the units' OKS blocks back to back (as the device
// exports them), state [3][10][kept] (kCocoTp / kCocoFp / kCocoIgnored per kept detection).  Returns the kept count.
extern "C" int core_eval(int n_units, int n_cats, const int* unit_cat, const int* unit_gt0, const int* unit_dt0,
                         const double* gt_kpt, const double* gt_box, const unsigned char* gt_crowd,
                         const unsigned char* gt_ignore, const double* dt_kpt, const double* dt_score, const double* thr,
                         double* precision, double* recall, double* oks, unsigned char* state_out) {
    // OKS per unit
    std::vector<int> cat_k0(n_cats + 1, 0), k_cat;
    std::vector<double> k_score, k_area;
    std::vector<long long> o0(n_units), k0(n_units);
    long long on = 0;
    for (int u = 0; u < n_units; ++u) {
        const int d0 = unit_dt0[u], nd = unit_dt0[u + 1] - d0, g0 = unit_gt0[u], ng = unit_gt0[u + 1] - g0;
        const int nk = std::min(nd, kCocoMaxDets);
        std::vector<int> kept(nk);
        for (int i = 0; i < nd; ++i) {
            const int r = coco_rank(dt_score + d0, nd, i);
            if (r < kCocoMaxDets) kept[r] = i;
        }
        k0[u] = (long long)k_score.size();
        o0[u] = on;
        for (int r = 0; r < nk; ++r) {
            k_score.push_back(dt_score[d0 + kept[r]]);
            k_area.push_back(coco_dt_area(dt_kpt + (size_t)kCocoKpt * (d0 + kept[r])));
            k_cat.push_back(unit_cat[u]);
            for (int g = 0; g < ng; ++g)
                oks[on++] = coco_oks(gt_kpt + (size_t)kCocoKpt * (g0 + g), gt_box + 5 * (size_t)(g0 + g),
                                     dt_kpt + (size_t)kCocoKpt * (d0 + kept[r]));
        }
        cat_k0[unit_cat[u] + 1] = (int)k_score.size();
    }
    for (int c = 1; c <= n_cats; ++c) cat_k0[c] = std::max(cat_k0[c], cat_k0[c - 1]);
    const int kept = (int)k_score.size();
    // matching per (unit, area range, threshold)
    std::vector<int> npig(n_cats * kCocoAreas, 0);
    std::vector<unsigned char> state((size_t)kCocoAreas * kCocoIouThrs * kept);
    for (int u = 0; u < n_units; ++u) {
        const int g0 = unit_gt0[u], ng = unit_gt0[u + 1] - g0, nk = std::min(unit_dt0[u + 1] - unit_dt0[u], kCocoMaxDets);
        for (int a = 0; a < kCocoAreas; ++a) {
            std::vector<bool> ig(ng);
            for (int g = 0; g < ng; ++g) {
                ig[g] = gt_ignore[g0 + g] || coco_area_out(gt_box[5 * (size_t)(g0 + g) + 4], a);
                npig[unit_cat[u] * kCocoAreas + a] += !ig[g];
            }
            for (int t = 0; t < kCocoIouThrs; ++t) {
                const double floor = coco_iou_floor(thr[t]);
                std::vector<bool> matched(ng, false);
                for (int r = 0; r < nk; ++r) {
                    double on_ = -1.0, oi = -1.0;
                    int gn = -1, gi = -1;
                    for (int g = 0; g < ng; ++g) {
                        if (matched[g] && !gt_crowd[g0 + g]) continue;
                        const double o = oks[o0[u] + (long long)r * ng + g];
                        if (o < floor) continue;
                        if (ig[g]) {
                            if (coco_better(o, g, oi, gi)) oi = o, gi = g;
                        } else if (coco_better(o, g, on_, gn)) {
                            on_ = o, gn = g;
                        }
                    }
                    const int m = gn >= 0 ? gn : gi;
                    if (m >= 0) matched[m] = true;
                    state[((size_t)a * kCocoIouThrs + t) * kept + k0[u] + r] =
                        (unsigned char)coco_dt_state(m >= 0, gn < 0, k_area[k0[u] + r], a);
                }
            }
        }
    }
    // global order per category
    std::vector<int> order(kept);
    for (int i = 0; i < kept; ++i) {
        const int jb = cat_k0[k_cat[i]], je = cat_k0[k_cat[i] + 1];
        order[jb + coco_rank(k_score.data() + jb, je - jb, i - jb)] = i;
    }
    // accumulation per (category, area range, threshold)
    for (int c = 0; c < n_cats; ++c)
        for (int a = 0; a < kCocoAreas; ++a)
            for (int t = 0; t < kCocoIouThrs; ++t) {
                double* prec = precision + ((size_t)t * kCocoRecThrs * n_cats + c) * kCocoAreas + a;
                const size_t ps = (size_t)n_cats * kCocoAreas;
                double& rec = recall[((size_t)t * n_cats + c) * kCocoAreas + a];
                const int np = npig[c * kCocoAreas + a];
                if (np == 0) {
                    for (int r = 0; r < kCocoRecThrs; ++r) prec[r * ps] = -1.0;
                    rec = -1.0;
                    continue;
                }
                double seg[kCocoRecThrs] = {0};
                long long tp = 0, fp = 0;
                rec = 0.0;
                for (int i = cat_k0[c]; i < cat_k0[c + 1]; ++i) {
                    const int s = state[((size_t)a * kCocoIouThrs + t) * kept + order[i]];
                    tp += s == kCocoTp;
                    fp += s == kCocoFp;
                    double rc, pr;
                    coco_pr(tp, fp, np, &rc, &pr);
                    const int q = coco_rec_count(thr + kCocoIouThrs, rc);
                    if (q > 0) seg[q - 1] = std::max(seg[q - 1], pr);
                    rec = rc;
                }
                double run = 0.0;
                for (int r = kCocoRecThrs - 1; r >= 0; --r) prec[r * ps] = run = std::max(run, seg[r]);
            }
    if (state_out) std::copy(state.begin(), state.end(), state_out);
    return kept;
}
