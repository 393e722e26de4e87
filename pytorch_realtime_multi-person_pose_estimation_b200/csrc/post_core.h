// Sequential-exact cores of the fused post-processing, shared between device code (postprocess.cu) and a
// host-only unit test (tests/cuda/test_post_core.cpp, compiled with g++).  They restate, operation for
// operation, /root/reference/lib/pafprocess/pafprocess.cpp:
//   pair_score()      :57-94 + get_paf_vectors :220-238 + roundpaf :240-242
//   sort_candidates() :97   (std::sort, libstdc++ introsort - reproduces its order for exactly-equal scores)
//   greedy_match()    :98-124
//   Assembler         :127-191 (person assembly / merge / prune) with O(1) row lookup instead of a linear scan
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define B2P_HD __host__ __device__ __forceinline__
#else
#define B2P_HD inline
#include <math.h>
#endif
#include <stdio.h>

namespace b2p {

constexpr int kNumPart = 18;
constexpr int kNumLimb = 19;
constexpr int kStepPaf = 10;          // pafprocess.h:13
constexpr int kRowFloats = 20;        // 18 part ids, [18] score sum, [19] part count
#define B2P_LIMB_TABLES                                                                                            \
    { {1, 2}, {1, 5}, {2, 3}, {3, 4}, {5, 6}, {6, 7}, {1, 8}, {8, 9}, {9, 10}, {1, 11}, {11, 12}, {12, 13}, {1, 0}, \
      {0, 14}, {14, 16}, {0, 15}, {15, 17}, {2, 16}, {5, 17} }
#define B2P_LIMB_PAF_TABLES                                                                                    \
    { {12, 13}, {20, 21}, {14, 15}, {16, 17}, {22, 23}, {24, 25}, {0, 1}, {2, 3}, {4, 5}, {6, 7}, {8, 9},     \
      {10, 11}, {28, 29}, {30, 31}, {34, 35}, {32, 33}, {36, 37}, {18, 19}, {26, 27} }

// ---- exact IEEE single ops (no FMA contraction on either side)
#if defined(__CUDA_ARCH__)
B2P_HD float f_mul(float a, float b) { return __fmul_rn(a, b); }
B2P_HD float f_add(float a, float b) { return __fadd_rn(a, b); }
B2P_HD float f_div(float a, float b) { return __fdiv_rn(a, b); }
B2P_HD float f_sqrt(float a) { return __fsqrt_rn(a); }
#else
B2P_HD float f_mul(float a, float b) { volatile float r = a * b; return r; }
B2P_HD float f_add(float a, float b) { volatile float r = a + b; return r; }
B2P_HD float f_div(float a, float b) { volatile float r = a / b; return r; }
B2P_HD float f_sqrt(float a) { return sqrtf(a); }
#endif

// PAF accessor: value of channel c at UPSAMPLED pixel (y, x) = base[c*sc + (y>>shift)*sy + (x>>shift)*sx].
// shift=3 reads the low-res map in place of the x8 nearest-neighbour copy the reference materialises
// (paf_to_pose.py:382-383); shift=0 serves the legacy process_paf() call that is handed the upsampled HWC array.
struct PafView {
    const float* base;
    long sc, sy, sx;
    int shift;
    B2P_HD float at(int c, int y, int x) const { return base[c * sc + (long)(y >> shift) * sy + (long)(x >> shift) * sx]; }
};

// Up-sampled coordinate -> low-resolution index at an integer factor f: cv2.resize(INTER_NEAREST) by f reads source
// pixel x // f (checked for f = 1 .. 16).  A shift when f is a power of two, a division otherwise.
struct UpIndex {
    int f, shift;     // shift < 0: divide by f
    B2P_HD int operator()(int v) const { return shift >= 0 ? v >> shift : v / f; }
};
inline UpIndex up_index(int f) {
    int sh = 0;
    while ((1 << sh) < f) ++sh;
    return UpIndex{f, (1 << sh) == f ? sh : -1};
}
// PafView at any factor (the kernels of default runs keep PafView and its shift of 3)
struct PafViewF {
    const float* base;
    long sc, sy, sx;
    UpIndex up;
    B2P_HD float at(int c, int y, int x) const { return base[c * sc + (long)up(y) * sy + (long)up(x) * sx]; }
};

// roundpaf (pafprocess.cpp:240-242) is `(int)(v + 0.5)` evaluated in DOUBLE.  For 0 <= v <= 16384 the single-precision
// form gives the same integer for every float except v = 0x1.fffffep-2 (largest float below 0.5, where v + 0.5f rounds
// up to 1.0f) - checked exhaustively over all 1.18e9 floats of that range - so one compare keeps it exact while avoiding
// the FP64 conversion pipe (20 conversions per candidate pair).
B2P_HD int round_half_up(float v) { return v == 0x1.fffffep-2f ? 0 : (int)f_add(v, 0.5f); }

// The five settings of pair scoring and the prune, pafprocess.h:7-13.  PostParams carries them at run time (kernel
// arguments by value, so every run keeps the values it was submitted with); DefaultPostParams is the reference's
// constants as compile-time values, the instantiation every default run executes, with the sample loop fully unrolled.
struct PostParams {
    float paf_thresh;        // THRESH_VECTOR_SCORE: a PAF sample counts if vec . paf > paf_thresh
    int paf_samples;         // STEP_PAF: samples along a candidate limb, 1 .. kMaxPafSamples
    int paf_min_above;       // THRESH_VECTOR_CNT1: keep a pair iff more than this many samples count
    int min_parts;           // THRESH_PART_CNT: drop a person with fewer parts
    float min_person_score;  // THRESH_HUMAN_SCORE: drop a person whose score / parts is lower
};
struct DefaultPostParams {
    static constexpr float paf_thresh = 0.05f;
    static constexpr int paf_samples = kStepPaf;
    static constexpr int paf_min_above = 6;
    static constexpr int min_parts = 4;
    static constexpr float min_person_score = 0.3f;
};
constexpr int kMaxPafSamples = 64;

// Range check of run-time settings (host): true if valid, else false with the first field out of range, its value and
// its range in msg.
inline bool post_params_check(const PostParams& q, char* msg, int cap) {
    if (!isfinite(q.paf_thresh)) return snprintf(msg, cap, "paf_thresh must be finite, got %g", (double)q.paf_thresh), false;
    if (q.paf_samples < 1 || q.paf_samples > kMaxPafSamples)
        return snprintf(msg, cap, "paf_samples must be 1 .. %d, got %d", kMaxPafSamples, q.paf_samples), false;
    if (q.paf_min_above < -1 || q.paf_min_above > q.paf_samples)
        return snprintf(msg, cap, "paf_min_above must be -1 .. paf_samples (%d), got %d", q.paf_samples, q.paf_min_above),
               false;
    if (q.min_parts < 0 || q.min_parts > kNumPart)
        return snprintf(msg, cap, "min_parts must be 0 .. %d, got %d", kNumPart, q.min_parts), false;
    if (!isfinite(q.min_person_score))
        return snprintf(msg, cap, "min_person_score must be finite, got %g", (double)q.min_person_score), false;
    return true;
}

// Scores one (a, b) peak pair of a limb.  Returns true and the candidate score if it passes both criteria.
// `Paf` is any accessor with `float at(int c, int y, int x) const` (PafView, or the shared-memory planes of the scoring
// kernel); `Prm` is PostParams or DefaultPostParams.  Restated from pafprocess.cpp:57-94 operation for operation, with
// two EXACT simplifications of its double precision parts (both proven below and pinned by the host tests against the
// compiled reference):
//   * `norm < 1e-12` (double):  norm = sqrt(dx^2 + dy^2) of integer dx, dy is 0 or >= 1, so the test is `norm == 0`.
//   * the length penalty  pen = 0.5*h_up/norm - 1.0 (double), crit2 = (float)((double)(scores/n) + min(pen, 0)):
//     q = fl(0.5*h_up/norm) < 1  <=>  norm > 0.5*h_up, because 1 - 0.5*h_up/norm is either <= 0 or >= 2^-25 (norm is a
//     float, 0.5*h_up a multiple of 0.5 below 2^24), far from the 2^-54 rounding boundary below 1; and q - 1.0 is exact
//     (Sterbenz).  So without penalty crit2 is (float)(double)(scores/n) = scores/n itself, and the double expression
//     is evaluated only for pairs longer than half the image height.
// Neither argument depends on the settings.  The penalty argument involves only norm and h_up.  round_half_up is exact
// for 0 <= v <= 16384, and v = fl(a + fl(i * fl(d / n))), 0 <= i < n, lies within a few ulps of the segment between the
// two peaks' coordinates a and a + d for every sample count n: it is in that range whenever the peaks are, and every
// sample lands on a pixel between the two peaks, inside the map.  The thresholds only enter the compares
// `s > paf_thresh` (float) and `crit1 > paf_min_above` (int), which the reference makes in the same types.
template <class Paf, class Prm>
B2P_HD bool pair_score_t(const Paf& paf, int c1, int c2, int ax, int ay, int bx, int by, int h_up, const Prm& prm,
                         float* score_out) {
    const int dxi = bx - ax, dyi = by - ay;
    float vx = (float)dxi, vy = (float)dyi;
    const float norm = f_sqrt(f_add(f_mul(vx, vx), f_mul(vy, vy)));
    if (!(norm > 0.f)) return false;
    vx = f_div(vx, norm);
    vy = f_div(vy, norm);
    const int n = prm.paf_samples;
    const float step_x = f_div((float)dxi, (float)n);
    const float step_y = f_div((float)dyi, (float)n);
    float scores = 0.0f;
    int crit1 = 0;
    // unrolled for the compile-time count; a run-time count (PostParams) keeps a rolled loop of at most kMaxPafSamples
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (int i = 0; i < n; ++i) {
        const int lx = round_half_up(f_add((float)ax, f_mul((float)i, step_x)));
        const int ly = round_half_up(f_add((float)ay, f_mul((float)i, step_y)));
        const float s = f_add(f_mul(vx, paf.at(c1, ly, lx)), f_mul(vy, paf.at(c2, ly, lx)));
        scores = f_add(scores, s);
        if (s > prm.paf_thresh) crit1 += 1;
    }
    if (crit1 <= prm.paf_min_above) return false;
    float crit2 = f_div(scores, (float)n);
    if (norm > 0.5f * (float)h_up) {
        const double pen = 0.5 * h_up / (double)norm - 1.0;
        crit2 = (float)((double)crit2 + pen);
    }
    if (crit2 > 0.f) {
        *score_out = crit2;
        return true;
    }
    return false;
}
B2P_HD bool pair_score(const PafView& paf, int c1, int c2, int ax, int ay, int bx, int by, int h_up, float* score_out) {
    return pair_score_t(paf, c1, c2, ax, ay, bx, by, h_up, DefaultPostParams{}, score_out);
}

// Candidate key: high 32 bits = ~bits(score) (score > 0, so ascending key == descending score), low 32 bits =
// pair index a*nb+b (the order the reference generates candidates in).
B2P_HD uint64_t cand_key(float score, uint32_t pair) {
#if defined(__CUDA_ARCH__)
    const uint32_t b = __float_as_uint(score);
#else
    union { float f; uint32_t u; } cv; cv.f = score; const uint32_t b = cv.u;
#endif
    return ((uint64_t)(~b) << 32) | pair;
}
B2P_HD float key_score(uint64_t k) {
    const uint32_t b = ~(uint32_t)(k >> 32);
#if defined(__CUDA_ARCH__)
    return __uint_as_float(b);
#else
    union { float f; uint32_t u; } cv; cv.u = b; return cv.f;
#endif
}
// comp_candidate(a, b) = a.score > b.score  (pafprocess.cpp:244-246)
#define B2P_COMP(a, b) ((uint32_t)((a) >> 32) < (uint32_t)((b) >> 32))

// libstdc++ std::sort on keys given in generation order; only needed when equal scores exist (a stable parallel
// sort gives the same permutation otherwise).  Iterative form of __introsort_loop + __final_insertion_sort.
B2P_HD void seq_unguarded_linear_insert(uint64_t* v, long last) {
    const uint64_t val = v[last];
    long next = last - 1;
    while (B2P_COMP(val, v[next])) { v[last] = v[next]; last = next; --next; }
    v[last] = val;
}
B2P_HD void seq_insertion_sort(uint64_t* v, long first, long last) {
    if (first == last) return;
    for (long i = first + 1; i != last; ++i) {
        if (B2P_COMP(v[i], v[first])) {
            const uint64_t val = v[i];
            for (long j = i; j > first; --j) v[j] = v[j - 1];
            v[first] = val;
        } else
            seq_unguarded_linear_insert(v, i);
    }
}
B2P_HD void seq_adjust_heap(uint64_t* f, long hole, long len, uint64_t value) {
    const long top = hole;
    long child = hole;
    while (child < (len - 1) / 2) {
        child = 2 * (child + 1);
        if (B2P_COMP(f[child], f[child - 1])) child--;
        f[hole] = f[child];
        hole = child;
    }
    if ((len & 1) == 0 && child == (len - 2) / 2) {
        child = 2 * (child + 1);
        f[hole] = f[child - 1];
        hole = child - 1;
    }
    long parent = (hole - 1) / 2;
    while (hole > top && B2P_COMP(f[parent], value)) { f[hole] = f[parent]; hole = parent; parent = (hole - 1) / 2; }
    f[hole] = value;
}
B2P_HD void seq_heap_sort(uint64_t* v, long first, long last) {
    uint64_t* f = v + first;
    long len = last - first;
    if (len >= 2)
        for (long parent = (len - 2) / 2;; --parent) {
            seq_adjust_heap(f, parent, len, f[parent]);
            if (parent == 0) break;
        }
    while (len > 1) {
        --len;
        const uint64_t value = f[len];
        f[len] = f[0];
        seq_adjust_heap(f, 0, len, value);
    }
}
B2P_HD void seq_std_sort(uint64_t* v, int n) {
    if (n <= 0) return;
    int lg = 0;
    for (int m = n; m > 1; m >>= 1) ++lg;
    // explicit stack replaces the recursion on the right part
    long st_first[64], st_last[64];
    int st_depth[64], sp = 0;
    st_first[0] = 0; st_last[0] = n; st_depth[0] = 2 * lg; sp = 1;
    while (sp > 0) {
        --sp;
        long first = st_first[sp], last = st_last[sp];
        int depth = st_depth[sp];
        while (last - first > 16) {
            if (depth == 0) { seq_heap_sort(v, first, last); break; }
            --depth;
            const long mid = first + (last - first) / 2;
            const long a = first + 1, b = mid, c = last - 1;
            long m;
            if (B2P_COMP(v[a], v[b])) m = B2P_COMP(v[b], v[c]) ? b : (B2P_COMP(v[a], v[c]) ? c : a);
            else m = B2P_COMP(v[a], v[c]) ? a : (B2P_COMP(v[b], v[c]) ? c : b);
            { const uint64_t t = v[first]; v[first] = v[m]; v[m] = t; }
            long lo = first + 1, hi = last;
            for (;;) {
                while (B2P_COMP(v[lo], v[first])) ++lo;
                --hi;
                while (B2P_COMP(v[first], v[hi])) --hi;
                if (!(lo < hi)) break;
                const uint64_t t = v[lo]; v[lo] = v[hi]; v[hi] = t;
                ++lo;
            }
            // recurse on [lo, last) first (as libstdc++ does), then loop on [first, lo): order of the two
            // sub-sorts does not change the result since they touch disjoint ranges.
            if (sp < 64) { st_first[sp] = lo; st_last[sp] = last; st_depth[sp] = depth; ++sp; }
            last = lo;
        }
    }
    if (n > 16) {
        seq_insertion_sort(v, 0, 16);
        for (long i = 16; i != n; ++i) seq_unguarded_linear_insert(v, i);
    } else
        seq_insertion_sort(v, 0, n);
}

// Sequential exact introsort of the sub-range v[first, last) with depth budget `depth` (= what the recursive
// __introsort_loop call on that range does, followed by the part of __final_insertion_sort that falls into it).
// One thread; the device runs 32 of these side by side, one small range per lane.
B2P_HD void seq_sort_range(uint64_t* v, long first, long last, int depth) {
    long sf[24], sl[24];
    int sd[24], sp = 1;
    sf[0] = first; sl[0] = last; sd[0] = depth;
    while (sp > 0) {
        --sp;
        long f = sf[sp], l = sl[sp];
        int d = sd[sp];
        bool heap_sorted = false;
        while (l - f > 16) {
            if (d == 0) { seq_heap_sort(v, f, l); heap_sorted = true; break; }
            --d;
            const long a = f + 1, b = f + (l - f) / 2, c = l - 1;
            long m;
            if (B2P_COMP(v[a], v[b])) m = B2P_COMP(v[b], v[c]) ? b : (B2P_COMP(v[a], v[c]) ? c : a);
            else m = B2P_COMP(v[a], v[c]) ? a : (B2P_COMP(v[b], v[c]) ? c : b);
            { const uint64_t t = v[f]; v[f] = v[m]; v[m] = t; }
            const uint32_t pivot = (uint32_t)(v[f] >> 32);
            long lo = f + 1, hi = l;
            for (;;) {
                while ((uint32_t)(v[lo] >> 32) < pivot) ++lo;
                --hi;
                while (pivot < (uint32_t)(v[hi] >> 32)) --hi;
                if (!(lo < hi)) break;
                const uint64_t t = v[lo]; v[lo] = v[hi]; v[hi] = t;
                ++lo;
            }
            if (l - lo > 16 && sp < 24) { sf[sp] = lo; sl[sp] = l; sd[sp] = d; ++sp; }
            else if (l - lo > 1) {
                if (l - lo > 16) seq_std_sort(v + lo, (int)(l - lo));   // stack exhausted: unreachable for ranges <= 2^24
                else for (long i = lo + 1; i < l; ++i) {                 // leaf: stable insertion sort
                    const uint64_t val = v[i];
                    long j = i;
                    while (j > lo && B2P_COMP(val, v[j - 1])) { v[j] = v[j - 1]; --j; }
                    v[j] = val;
                }
            }
            l = lo;
        }
        if (!heap_sorted)
            for (long i = f + 1; i < l; ++i) {
                const uint64_t val = v[i];
                long j = i;
                while (j > f && B2P_COMP(val, v[j - 1])) { v[j] = v[j - 1]; --j; }
                v[j] = val;
            }
    }
}

// ---------------------------------------------------------------- warp-parallel exact std::sort
// One partition step of libstdc++'s introsort (__unguarded_partition_pivot: median-of-3 of first+1 / mid / last-1
// moved to `first`, then the Hoare loop `while (comp(*lo, pivot)) ++lo; --hi; while (comp(pivot, *hi)) --hi;
// if (!(lo < hi)) return lo; swap; ++lo`), executed by ONE WARP on 32-element chunks: the k-th position where the
// sequential `lo` scan would stop is paired with the k-th position where the `hi` scan would stop, so the swaps -
// and therefore the final order of elements with EQUAL keys - are exactly those of the sequential algorithm.
// On the host (tests) the per-lane parts run as loops.  All lanes must call it with identical arguments.
#if defined(__CUDA_ARCH__)
#define B2P_LANE() ((int)(threadIdx.x & 31))
#define B2P_SYNCWARP() __syncwarp()
#else
#define B2P_LANE() 0
#define B2P_SYNCWARP()
#endif

B2P_HD int nth_set_bit(uint32_t m, int k) {   // position of the (k+1)-th set bit, k < popc(m)
#if defined(__CUDA_ARCH__)
    return (int)__fns(m, 0, k + 1);
#else
    for (int i = 0; i < 32; ++i)
        if ((m >> i) & 1u) { if (k == 0) return i; --k; }
    return -1;
#endif
}
B2P_HD int popc32(uint32_t m) {
#if defined(__CUDA_ARCH__)
    return __popc(m);
#else
    return __builtin_popcount(m);
#endif
}
B2P_HD uint32_t low_bits(long n) { return n <= 0 ? 0u : (n >= 32 ? 0xffffffffu : ((1u << n) - 1u)); }

// stop mask for the ascending scan over positions [c, c+32): bit j <=> !(comp(v[c+j], pivot)) i.e. key >= pivot key
B2P_HD uint32_t chunk_mask_lo(const uint64_t* v, long c, long last, uint32_t pivot) {
#if defined(__CUDA_ARCH__)
    const long p = c + B2P_LANE();
    const bool stop = (p < last) && ((uint32_t)(v[p] >> 32) >= pivot);
    return __ballot_sync(0xffffffffu, stop);
#else
    uint32_t m = 0;
    for (int j = 0; j < 32; ++j) { const long p = c + j; if (p < last && (uint32_t)(v[p] >> 32) >= pivot) m |= 1u << j; }
    return m;
#endif
}
// stop mask for the descending scan over positions c-1, c-2, ..: bit j <=> position c-1-j, !(comp(pivot, v[p]))
B2P_HD uint32_t chunk_mask_hi(const uint64_t* v, long c, long first, uint32_t pivot) {
#if defined(__CUDA_ARCH__)
    const long p = c - 1 - B2P_LANE();
    const bool stop = (p >= first) && ((uint32_t)(v[p] >> 32) <= pivot);
    return __ballot_sync(0xffffffffu, stop);
#else
    uint32_t m = 0;
    for (int j = 0; j < 32; ++j) { const long p = c - 1 - j; if (p >= first && (uint32_t)(v[p] >> 32) <= pivot) m |= 1u << j; }
    return m;
#endif
}

// wscr: 64 bytes of per-warp shared scratch on the device (rank -> lane tables); unused on the host.
B2P_HD long warp_partition(uint64_t* v, long first, long last, unsigned char* wscr = nullptr) {
    if (B2P_LANE() == 0) {   // __move_median_to_first(first, first+1, mid, last-1)
        const long a = first + 1, b = first + (last - first) / 2, c = last - 1;
        long m;
        if (B2P_COMP(v[a], v[b])) m = B2P_COMP(v[b], v[c]) ? b : (B2P_COMP(v[a], v[c]) ? c : a);
        else m = B2P_COMP(v[a], v[c]) ? a : (B2P_COMP(v[b], v[c]) ? c : b);
        const uint64_t t = v[first]; v[first] = v[m]; v[m] = t;
    }
    B2P_SYNCWARP();
    const uint32_t pivot = (uint32_t)(v[first] >> 32);
    long cA = first + 1, cB = last;          // chunk A = [cA, cA+32), chunk B = positions cB-1 .. cB-32
    uint32_t rawA = chunk_mask_lo(v, cA, last, pivot);
    uint32_t rawB = chunk_mask_hi(v, cB, first, pivot);
    long lo_limit = last;    // once a swap happened: the position of the last swapped `hi` (holds a lo-stop value now)
    long hi_limit = first;   // v[first] == pivot stops the hi scan; later: position of the last swapped `lo`
    for (;;) {
        // effective stop masks in the CURRENT array state (rawA/rawB were loaded before the latest swaps)
        uint32_t effA = rawA & low_bits(lo_limit - cA);
        if (lo_limit < last && lo_limit >= cA && lo_limit < cA + 32) effA |= 1u << (lo_limit - cA);
        uint32_t effB = rawB & low_bits(cB - 1 - hi_limit);
        if (cB - 1 - hi_limit >= 0 && cB - 1 - hi_limit < 32) effB |= 1u << (cB - 1 - hi_limit);
        if (effA == 0) { cA += 32; rawA = chunk_mask_lo(v, cA, last, pivot); continue; }
        if (effB == 0) { cB -= 32; rawB = chunk_mask_hi(v, cB, first, pivot); continue; }
        const int pa = popc32(effA), pb = popc32(effB), m = pa < pb ? pa : pb;
        int kp = 0;              // number of leading pairs with lo_k < hi_k
        long lo_k = 0, hi_k = 0; // of pair kp (the first failing one) or garbage if kp == m
        long last_lo = 0, last_hi = 0;
#if defined(__CUDA_ARCH__)
        int ja_last, jb_last;    // bit positions of the m-th stops
        {
            // k-th set bit of each mask for lane k: the lane sitting on a set bit knows its rank (popc below it) and
            // publishes its index at table[rank]  (__fns would cost ~100 instructions per call)
            const int k = B2P_LANE();
            const uint32_t below = (1u << k) - 1u;
            if ((effA >> k) & 1u) wscr[__popc(effA & below)] = (unsigned char)k;
            if ((effB >> k) & 1u) wscr[32 + __popc(effB & below)] = (unsigned char)k;
            __syncwarp();
            long mylo = 0, myhi = 0;
            bool ok = false;
            if (k < m) {
                mylo = cA + wscr[k];
                myhi = cB - 1 - wscr[32 + k];
                ok = mylo < myhi;
            }
            ja_last = wscr[m - 1];
            jb_last = wscr[32 + m - 1];
            const uint32_t okm = __ballot_sync(0xffffffffu, ok);
            kp = __popc(okm);     // ok is monotone in k: lo_k increases, hi_k decreases
            if (ok) { const uint64_t t = v[mylo]; v[mylo] = v[myhi]; v[myhi] = t; }
            const int src_fail = kp < m ? kp : 0, src_last = kp > 0 ? kp - 1 : 0;
            lo_k = __shfl_sync(0xffffffffu, mylo, src_fail);
            hi_k = __shfl_sync(0xffffffffu, myhi, src_fail);
            last_lo = __shfl_sync(0xffffffffu, mylo, src_last);
            last_hi = __shfl_sync(0xffffffffu, myhi, src_last);
            __syncwarp();
        }
#else
        for (int k = 0; k < m; ++k) {
            const long mylo = cA + nth_set_bit(effA, k), myhi = cB - 1 - nth_set_bit(effB, k);
            if (!(mylo < myhi)) { lo_k = mylo; hi_k = myhi; break; }
            const uint64_t t = v[mylo]; v[mylo] = v[myhi]; v[myhi] = t;
            last_lo = mylo; last_hi = myhi;
            ++kp;
        }
#endif
        if (kp > 0) { lo_limit = last_hi; hi_limit = last_lo; }
        if (kp < m) {
            (void)hi_k;
            // sequential loop breaks here with lo at the next lo-stop of the current state
            return (kp > 0 && last_hi < lo_k) ? last_hi : lo_k;
        }
        // all m pairs swapped: the scans have passed the consumed stops
#if defined(__CUDA_ARCH__)
        rawA &= ~low_bits(ja_last + 1);
        rawB &= ~low_bits(jb_last + 1);
#else
        rawA &= ~low_bits(nth_set_bit(effA, m - 1) + 1);
        rawB &= ~low_bits(nth_set_bit(effB, m - 1) + 1);
#endif
    }
}

// ---------------------------------------------------------------- block-parallel exact partition (big ranges)
// Same pairing rule as warp_partition, evaluated by ranks instead of by scanning: with lo-stops (key >= pivot) ranked
// from the left and hi-stops (key <= pivot) ranked from the right over [first+1, last), the sequential Hoare loop
// swaps lo-stop #k with hi-stop #k for k = 1..K, K = number of k with posA[k] < posB[k] (monotone), and returns
// min(posA[K+1], posB[K]).  T cooperating threads each own a contiguous slice; phases are separated by block
// barriers on the device and by plain loops on the host (tests).
struct BlockPartState {
    long first, last;
    uint32_t pivot;
    long per;
    int totA, totB, K;
    long cut;
};
B2P_HD void bp_prepare(BlockPartState& st, uint64_t* v, long first, long last, int T) {   // one thread
    const long a = first + 1, b = first + (last - first) / 2, c = last - 1;
    long m;
    if (B2P_COMP(v[a], v[b])) m = B2P_COMP(v[b], v[c]) ? b : (B2P_COMP(v[a], v[c]) ? c : a);
    else m = B2P_COMP(v[a], v[c]) ? a : (B2P_COMP(v[b], v[c]) ? c : b);
    const uint64_t t = v[first]; v[first] = v[m]; v[m] = t;
    st.first = first; st.last = last;
    st.pivot = (uint32_t)(v[first] >> 32);
    st.per = (last - first - 1 + T - 1) / T;
}
B2P_HD void bp_slice(const BlockPartState& st, int tid, long* s, long* e) {
    long b = st.first + 1 + (long)tid * st.per;
    if (b > st.last) b = st.last;
    long en = b + st.per;
    if (en > st.last) en = st.last;
    *s = b; *e = en;
}
B2P_HD void bp_count(const BlockPartState& st, const uint64_t* v, int tid, int* cA, int* cB) {
    long s, e;
    bp_slice(st, tid, &s, &e);
    int a = 0, b = 0;
    long p = s;
    for (; p + 4 <= e; p += 4) {     // four independent loads in flight (the slices live in L2 / HBM)
        const uint32_t k0 = (uint32_t)(v[p] >> 32), k1 = (uint32_t)(v[p + 1] >> 32);
        const uint32_t k2 = (uint32_t)(v[p + 2] >> 32), k3 = (uint32_t)(v[p + 3] >> 32);
        a += (k0 >= st.pivot) + (k1 >= st.pivot) + (k2 >= st.pivot) + (k3 >= st.pivot);
        b += (k0 <= st.pivot) + (k1 <= st.pivot) + (k2 <= st.pivot) + (k3 <= st.pivot);
    }
    for (; p < e; ++p) {
        const uint32_t k = (uint32_t)(v[p] >> 32);
        a += (k >= st.pivot);
        b += (k <= st.pivot);
    }
    *cA = a; *cB = b;
}
// offA: lo-stops before this slice; b_right: hi-stops after this slice.  posA/posB are 1-based rank -> position
// tables; positions are stored relative to st.first in PosT (int32 for global-memory ranges, uint16 for the
// shared-memory ranges of <= 65535 keys).
template <class PosT>
B2P_HD void bp_scatter(const BlockPartState& st, const uint64_t* v, int tid, int offA, int b_right, PosT* posA,
                       PosT* posB) {
    long s, e;
    bp_slice(st, tid, &s, &e);
    const long f = st.first;
    int a = offA;
    long p = s;
    for (; p + 4 <= e; p += 4) {
        const uint32_t k0 = (uint32_t)(v[p] >> 32), k1 = (uint32_t)(v[p + 1] >> 32);
        const uint32_t k2 = (uint32_t)(v[p + 2] >> 32), k3 = (uint32_t)(v[p + 3] >> 32);
        if (k0 >= st.pivot) posA[++a] = (PosT)(p - f);
        if (k1 >= st.pivot) posA[++a] = (PosT)(p + 1 - f);
        if (k2 >= st.pivot) posA[++a] = (PosT)(p + 2 - f);
        if (k3 >= st.pivot) posA[++a] = (PosT)(p + 3 - f);
    }
    for (; p < e; ++p)
        if ((uint32_t)(v[p] >> 32) >= st.pivot) posA[++a] = (PosT)(p - f);
    int b = b_right;
    p = e - 1;
    for (; p - 3 >= s; p -= 4) {
        const uint32_t k0 = (uint32_t)(v[p] >> 32), k1 = (uint32_t)(v[p - 1] >> 32);
        const uint32_t k2 = (uint32_t)(v[p - 2] >> 32), k3 = (uint32_t)(v[p - 3] >> 32);
        if (k0 <= st.pivot) posB[++b] = (PosT)(p - f);
        if (k1 <= st.pivot) posB[++b] = (PosT)(p - 1 - f);
        if (k2 <= st.pivot) posB[++b] = (PosT)(p - 2 - f);
        if (k3 <= st.pivot) posB[++b] = (PosT)(p - 3 - f);
    }
    for (; p >= s; --p)
        if ((uint32_t)(v[p] >> 32) <= st.pivot) posB[++b] = (PosT)(p - f);
}
template <class PosT>
B2P_HD int bp_count_swaps(const BlockPartState& st, int tid, int T, const PosT* posA, const PosT* posB) {
    const int lim = st.totA < st.totB ? st.totA : st.totB;
    int c = 0;
    for (int k = 1 + tid; k <= lim; k += T) c += (posA[k] < posB[k]);
    return c;
}
template <class PosT>
B2P_HD void bp_swap(const BlockPartState& st, uint64_t* v, int tid, int T, const PosT* posA, const PosT* posB) {
    for (int k = 1 + tid; k <= st.K; k += T) {
        const long ia = st.first + posA[k], ib = st.first + posB[k];
        const uint64_t t = v[ia]; v[ia] = v[ib]; v[ib] = t;
    }
}
template <class PosT>
B2P_HD long bp_cut(const BlockPartState& st, const PosT* posA, const PosT* posB) {
    const long a_next = (st.K + 1 <= st.totA) ? st.first + posA[st.K + 1] : st.last;
    return (st.K > 0 && st.first + posB[st.K] < a_next) ? st.first + posB[st.K] : a_next;
}

#if !defined(__CUDA_ARCH__)
// host emulation of one block partition with T virtual threads (tests)
template <class PosT>
inline long block_partition_host(uint64_t* v, long first, long last, int T, PosT* posA, PosT* posB) {
    BlockPartState st;
    bp_prepare(st, v, first, last, T);
    int* cA = new int[T]; int* cB = new int[T];
    for (int t = 0; t < T; ++t) bp_count(st, v, t, &cA[t], &cB[t]);
    int totA = 0, totB = 0;
    for (int t = 0; t < T; ++t) { totA += cA[t]; totB += cB[t]; }
    st.totA = totA; st.totB = totB;
    int offA = 0, left = 0;
    for (int t = 0; t < T; ++t) {
        bp_scatter(st, v, t, offA, totB - left - cB[t], posA, posB);
        offA += cA[t]; left += cB[t];
    }
    int K = 0;
    for (int t = 0; t < T; ++t) K += bp_count_swaps(st, t, T, posA, posB);
    st.K = K;
    for (int t = 0; t < T; ++t) bp_swap(st, v, t, T, posA, posB);
    delete[] cA; delete[] cB;
    return bp_cut(st, posA, posB);
}
#endif

// stable insertion sort of a leaf (<= 16 elements) = what __final_insertion_sort does inside one introsort leaf
B2P_HD void leaf_insertion_sort(uint64_t* v, long first, long last) {
    for (long i = first + 1; i < last; ++i) {
        const uint64_t val = v[i];
        long j = i;
        while (j > first && B2P_COMP(val, v[j - 1])) { v[j] = v[j - 1]; --j; }
        v[j] = val;
    }
}

#if !defined(__CUDA_ARCH__)
// host reference driver of the parallel formulation (tests): same partition routine, explicit stack
// big: ranges above it use the rank-based partition with T virtual threads and int32 tables; warp_rank: ranges of
// <= warp_rank keys use the rank-based partition with 32 lanes and uint16 tables of 512 entries (the device warp
// phase); everything else uses the chunked warp_partition.
inline void par_std_sort_host(uint64_t* v, int n, int big = 1 << 30, int T = 512, int warp_rank = 0, int seq_small = 0) {
    if (n <= 1) return;
    int32_t* posA = new int32_t[n + 2];
    int32_t* posB = new int32_t[n + 2];
    uint16_t tabA[512], tabB[512];
    int lg = 0;
    for (int m = n; m > 1; m >>= 1) ++lg;
    long sf[128], sl[128];
    int sd[128], sp = 0;
    sf[0] = 0; sl[0] = n; sd[0] = 2 * lg; sp = 1;
    while (sp > 0) {
        --sp;
        long first = sf[sp], last = sl[sp];
        int depth = sd[sp];
        bool heap_sorted = false;
        while (last - first > 16) {
            if (last - first <= seq_small) { seq_sort_range(v, first, last, depth); heap_sorted = true; break; }
            if (depth == 0) { seq_heap_sort(v, first, last); heap_sorted = true; break; }
            --depth;
            const long cut = (last - first > big) ? block_partition_host(v, first, last, T, posA, posB)
                             : (last - first <= warp_rank) ? block_partition_host(v, first, last, 32, tabA, tabB)
                                                           : warp_partition(v, first, last);
            if (last - cut > 16) { sf[sp] = cut; sl[sp] = last; sd[sp] = depth; ++sp; }
            else if (seq_small) seq_sort_range(v, cut, last, depth);
            else leaf_insertion_sort(v, cut, last);
            last = cut;
        }
        if (!heap_sorted) { if (seq_small) seq_sort_range(v, first, last, depth); else leaf_insertion_sort(v, first, last); }
    }
    delete[] posA; delete[] posB;
}
#endif

// Greedy one-to-one assignment over sorted candidates.  used_a/used_b: zeroed bitmaps.  Writes accepted
// connections (a index, b index, score) in acceptance order; returns their number.
B2P_HD int greedy_match(const uint64_t* keys, int n, int nb, uint32_t* used_a, uint32_t* used_b, int max_conn,
                        int* conn_a, int* conn_b, float* conn_s) {
    int nc = 0;
    for (int i = 0; i < n && nc < max_conn; ++i) {
        const uint32_t pair = (uint32_t)keys[i];
        const int a = pair / nb, b = pair % nb;
        if ((used_a[a >> 5] >> (a & 31)) & 1u) continue;
        if ((used_b[b >> 5] >> (b & 31)) & 1u) continue;
        used_a[a >> 5] |= 1u << (a & 31);
        used_b[b >> 5] |= 1u << (b & 31);
        conn_a[nc] = a;
        conn_b[nc] = b;
        conn_s[nc] = key_score(keys[i]);
        ++nc;
    }
    return nc;
}

// ---------------------------------------------------------------- person assembly
// Rows ("subset" in the reference) are float[20].  `rows` has capacity row_cap; erased rows are flagged dead and
// skipped (= vector::erase order).  For O(1) lookup every peak id keeps the list of alive rows holding it in its
// own part's slot (capacity kListCap; a longer list flips `degraded`, after which lookups scan all rows).
constexpr int kListCap = 4;

struct Assembler {
    float* rows;            // [row_cap][20]
    uint8_t* alive;         // [row_cap]
    int32_t* lists;         // [n_peaks][kListCap]
    uint8_t* list_n;        // [n_peaks]
    const int* part_base;   // [19] first peak id of each part (prefix sum of counts), [18] = total
    const float* peak_score;// [n_peaks] by id
    int row_cap, nrows, degraded, overflow;

    B2P_HD bool valid_id(float v, int part) const {
        return v >= (float)part_base[part] && v < (float)part_base[part + 1];
    }
    B2P_HD void list_add(int id, int r) {
        int n = list_n[id];
        if (n >= kListCap) { degraded = 1; return; }
        lists[id * kListCap + n] = r;
        list_n[id] = (uint8_t)(n + 1);
    }
    B2P_HD void list_remove(int id, int r) {
        int n = list_n[id];
        for (int i = 0; i < n; ++i)
            if (lists[id * kListCap + i] == r) {
                lists[id * kListCap + i] = lists[id * kListCap + n - 1];
                list_n[id] = (uint8_t)(n - 1);
                return;
            }
    }
    B2P_HD void set_slot(int r, int part, float nv) {
        const float old = rows[r * kRowFloats + part];
        if (valid_id(old, part)) list_remove((int)old, r);
        rows[r * kRowFloats + part] = nv;
        if (valid_id(nv, part)) list_add((int)nv, r);
    }
    // rows holding cid1 at p1 or cid2 at p2: count + two lowest row indices
    B2P_HD void lookup(int p1, int cid1, int p2, int cid2, int* found, int* s1, int* s2) const {
        int f = 0, a = 0x7fffffff, b = 0x7fffffff;
        if (!degraded) {
            for (int pass = 0; pass < 2; ++pass) {
                const int id = pass ? cid2 : cid1;
                const int other_p = pass ? p1 : p2;
                const int other_id = pass ? cid1 : cid2;
                const int n = list_n[id];
                for (int i = 0; i < n; ++i) {
                    const int r = lists[id * kListCap + i];
                    // a row matching on both slots is counted once (in pass 0)
                    if (pass == 1 && rows[r * kRowFloats + other_p] == (float)other_id) continue;
                    ++f;
                    if (r < a) { b = a; a = r; } else if (r < b) b = r;
                }
            }
        } else {
            for (int r = 0; r < nrows; ++r) {
                if (!alive[r]) continue;
                if (rows[r * kRowFloats + p1] == (float)cid1 || rows[r * kRowFloats + p2] == (float)cid2) {
                    ++f;
                    if (r < a) { b = a; a = r; } else if (r < b) b = r;
                }
            }
        }
        *found = f; *s1 = a; *s2 = b;
    }
    // one connection of limb `limb` (parts p1 -> p2), pafprocess.cpp:133-184
    B2P_HD void add_connection(int limb, int p1, int p2, int cid1, int cid2, float cscore) {
        int found, s1, s2;
        lookup(p1, cid1, p2, cid2, &found, &s1, &s2);
        if (found == 1) {
            float* r1 = rows + s1 * kRowFloats;
            if (r1[p2] != (float)cid2) {
                set_slot(s1, p2, (float)cid2);
                r1[19] = f_add(r1[19], 1.f);
                r1[18] = f_add(r1[18], f_add(peak_score[cid2], cscore));
            }
        } else if (found == 2) {
            float* r1 = rows + s1 * kRowFloats;
            float* r2 = rows + s2 * kRowFloats;
            int membership = 0;
            for (int k = 0; k < 18; ++k)
                if (r1[k] > 0 && r2[k] > 0) membership = 2;
            if (membership == 0) {
                for (int k = 0; k < 18; ++k) {
                    const float nv = f_add(r1[k], f_add(r2[k], 1.f));
                    if (valid_id(r2[k], k)) list_remove((int)r2[k], s2);
                    set_slot(s1, k, nv);
                }
                r1[19] = f_add(r1[19], r2[19]);
                r1[18] = f_add(r1[18], r2[18]);
                r1[18] = f_add(r1[18], cscore);
                alive[s2] = 0;
            } else {
                set_slot(s1, p2, (float)cid2);
                r1[19] = f_add(r1[19], 1.f);
                r1[18] = f_add(r1[18], f_add(peak_score[cid2], cscore));
            }
        } else if (found == 0 && limb < 18) {
            if (nrows >= row_cap) { overflow = 1; return; }
            float* row = rows + nrows * kRowFloats;
            for (int k = 0; k < kRowFloats; ++k) row[k] = -1.f;
            alive[nrows] = 1;
            set_slot(nrows, p1, (float)cid1);
            set_slot(nrows, p2, (float)cid2);
            row[19] = 2.f;
            row[18] = f_add(f_add(peak_score[cid1], peak_score[cid2]), cscore);
            ++nrows;
        }
    }
    // prune (pafprocess.cpp:187-191): keep rows with count >= min_parts and score/count >= min_person_score (the
    // reference's float compares; its int THRESH_PART_CNT converts to float)
    template <class Prm>
    B2P_HD bool keep(int r, const Prm& prm) const {
        if (!alive[r]) return false;
        const float* row = rows + r * kRowFloats;
        return !(row[19] < (float)prm.min_parts || f_div(row[18], row[19]) < prm.min_person_score);
    }
    B2P_HD bool keep(int r) const { return keep(r, DefaultPostParams{}); }
};

}  // namespace b2p
