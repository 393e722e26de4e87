// TEST INFRASTRUCTURE: host-only driver around csrc/post_core.h with run-time post-processing settings (PostParams,
// the instantiation the generic kernels run) or the compile-time defaults (DefaultPostParams, the default kernels), so
// both can be checked against the parameterised oracle and the reference compiled with other constants.
// Build: g++ -O2 -ffp-contract=off -std=c++17 -shared -fPIC post_params_host.cpp -o build/libpostparams_host.so
#include <algorithm>
#include <vector>

#include "../../pytorch_realtime_multi-person_pose_estimation_b200/csrc/post_core.h"

using namespace b2p;

static const int LIMB_PARTS[19][2] = B2P_LIMB_TABLES;
static const int LIMB_PAF[19][2] = B2P_LIMB_PAF_TABLES;

static std::vector<float> g_out;            // per human: score, then 18 x (x, y, peak score, cid)  (cid < 0 = missing)
static std::vector<float> g_cand, g_conn;   // (limb, a index, b index, score): sorted candidates, connections

template <class Prm>
static int process(int n_peaks, const float* peaks, int h_up, const float* paf, long sc, long sy, long sx, int shift,
                   const Prm& prm) {
    std::vector<int> px[18], py[18];
    std::vector<float> ps[18];
    for (int i = 0; i < n_peaks; ++i) {
        const int part = (int)peaks[i * 5 + 4];
        px[part].push_back((int)peaks[i * 5 + 0]);
        py[part].push_back((int)peaks[i * 5 + 1]);
        ps[part].push_back(peaks[i * 5 + 2]);
    }
    int part_base[19];
    part_base[0] = 0;
    for (int p = 0; p < 18; ++p) part_base[p + 1] = part_base[p] + (int)px[p].size();
    std::vector<float> peak_score(n_peaks + 1);
    std::vector<int> peak_x(n_peaks + 1), peak_y(n_peaks + 1);
    for (int p = 0; p < 18; ++p)
        for (size_t i = 0; i < px[p].size(); ++i) {
            peak_score[part_base[p] + i] = ps[p][i];
            peak_x[part_base[p] + i] = px[p][i];
            peak_y[part_base[p] + i] = py[p][i];
        }
    const PafView pv{paf, sc, sy, sx, shift};
    std::vector<int> ca[19], cb[19];
    std::vector<float> cs[19];
    g_cand.clear();
    g_conn.clear();
    int total_conn = 0;
    for (int l = 0; l < 19; ++l) {
        const int pa = LIMB_PARTS[l][0], pb = LIMB_PARTS[l][1];
        const int na = (int)px[pa].size(), nb = (int)px[pb].size();
        if (na == 0 || nb == 0) continue;
        std::vector<uint64_t> keys;
        for (int a = 0; a < na; ++a)
            for (int b = 0; b < nb; ++b) {
                float s;
                if (pair_score_t(pv, LIMB_PAF[l][0], LIMB_PAF[l][1], px[pa][a], py[pa][a], px[pb][b], py[pb][b], h_up,
                                 prm, &s))
                    keys.push_back(cand_key(s, (uint32_t)(a * nb + b)));
            }
        par_std_sort_host(keys.data(), (int)keys.size(), 512, 512, 512, 64);   // the device's sort configuration
        for (uint64_t k : keys)
            g_cand.insert(g_cand.end(), {(float)l, (float)((uint32_t)k / nb), (float)((uint32_t)k % nb), key_score(k)});
        const int maxc = na < nb ? na : nb;
        std::vector<uint32_t> ua((na + 31) / 32, 0), ub((nb + 31) / 32, 0);
        ca[l].resize(maxc); cb[l].resize(maxc); cs[l].resize(maxc);
        const int nc = greedy_match(keys.data(), (int)keys.size(), nb, ua.data(), ub.data(), maxc, ca[l].data(),
                                    cb[l].data(), cs[l].data());
        ca[l].resize(nc); cb[l].resize(nc); cs[l].resize(nc);
        for (int c = 0; c < nc; ++c) g_conn.insert(g_conn.end(), {(float)l, (float)ca[l][c], (float)cb[l][c], cs[l][c]});
        total_conn += nc;
    }
    std::vector<float> rows((size_t)(total_conn + 1) * kRowFloats);
    std::vector<uint8_t> alive(total_conn + 1, 0), list_n(n_peaks + 1, 0);
    std::vector<int32_t> lists((size_t)(n_peaks + 1) * kListCap);
    Assembler as;
    as.rows = rows.data(); as.alive = alive.data(); as.lists = lists.data(); as.list_n = list_n.data();
    as.part_base = part_base; as.peak_score = peak_score.data();
    as.row_cap = total_conn + 1; as.nrows = 0; as.degraded = 0; as.overflow = 0;
    for (int l = 0; l < 19; ++l)
        for (size_t c = 0; c < ca[l].size(); ++c)
            as.add_connection(l, LIMB_PARTS[l][0], LIMB_PARTS[l][1], part_base[LIMB_PARTS[l][0]] + ca[l][c],
                              part_base[LIMB_PARTS[l][1]] + cb[l][c], cs[l][c]);
    g_out.clear();
    int nh = 0;
    for (int r = 0; r < as.nrows; ++r) {
        if (!as.keep(r, prm)) continue;
        const float* row = rows.data() + r * kRowFloats;
        g_out.push_back(f_div(row[18], row[19]));
        for (int p = 0; p < 18; ++p) {
            const int cid = (int)row[p];
            if (cid < 0) { g_out.insert(g_out.end(), {0.f, 0.f, 0.f, -1.f}); continue; }
            g_out.insert(g_out.end(), {(float)peak_x[cid], (float)peak_y[cid], peak_score[cid], (float)cid});
        }
        ++nh;
    }
    return nh;
}

// prm: the run-time settings (the generic kernels' instantiation), or null for the compile-time defaults
extern "C" int params_process(int n_peaks, const float* peaks, int h_up, const float* paf, long sc, long sy, long sx,
                              int shift, const PostParams* prm) {
    return prm ? process(n_peaks, peaks, h_up, paf, sc, sy, sx, shift, *prm)
               : process(n_peaks, peaks, h_up, paf, sc, sy, sx, shift, DefaultPostParams{});
}
extern "C" const float* params_result() { return g_out.data(); }
extern "C" long params_num_cands() { return (long)g_cand.size() / 4; }
extern "C" const float* params_cands() { return g_cand.data(); }
extern "C" long params_num_conns() { return (long)g_conn.size() / 4; }
extern "C" const float* params_conns() { return g_conn.data(); }
extern "C" int params_check(const PostParams* prm, char* msg, int cap) { return post_params_check(*prm, msg, cap) ? 1 : 0; }
