/* ORACLE (test infrastructure only - never linked into the product library).
 *
 * Plain-C restatement of the reference's only native component,
 *   /root/reference/lib/pafprocess/pafprocess.cpp:22-246  (constants: pafprocess.h:6-24).
 * Same arithmetic, operation for operation (float vs double promotions included); written independently
 * (flat arrays, alive flags instead of vector::erase).  Pinned against the compiled, unmodified reference
 * source (oracle/_ref/libpafprocess_ref.so, built by oracle/Makefile) in tests/test_oracle_pafprocess.py.
 *
 * std::sort's handling of exactly-equal scores is reproduced by restating libstdc++'s introsort (see below).
 *
 * Build: gcc -O2 -ffp-contract=off -shared -fPIC pafprocess_port.c -o libpafprocess_port.so -lm
 */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#define NUM_PART 18
#define NUM_LIMB 19
#define STEP_PAF 10
static const float THRESH_VECTOR_SCORE = 0.05f; /* pafprocess.h:7 */
static const int THRESH_VECTOR_CNT1 = 6;        /* pafprocess.h:8 */
static const int THRESH_PART_CNT = 4;           /* pafprocess.h:9 */
static const float THRESH_HUMAN_SCORE = 0.3f;   /* pafprocess.h:10 */

/* pafprocess.h:16-24 */
static const int LIMB_PAF_CH[NUM_LIMB][2] = {{12, 13}, {20, 21}, {14, 15}, {16, 17}, {22, 23}, {24, 25}, {0, 1},
                                             {2, 3},   {4, 5},   {6, 7},   {8, 9},   {10, 11}, {28, 29}, {30, 31},
                                             {34, 35}, {32, 33}, {36, 37}, {18, 19}, {26, 27}};
static const int LIMB_PARTS[NUM_LIMB][2] = {{1, 2},   {1, 5},   {2, 3},  {3, 4},  {5, 6},   {6, 7},  {1, 8},
                                            {8, 9},   {9, 10},  {1, 11}, {11, 12}, {12, 13}, {1, 0},  {0, 14},
                                            {14, 16}, {0, 15},  {15, 17}, {2, 16}, {5, 17}};

typedef struct { int x, y; float score; int id; } Peak;
typedef struct { int idx1, idx2; float score; } Cand;
typedef struct { int cid1, cid2; float score; int pid1, pid2; } Conn;

/* results kept between calls, like the reference's file-scope globals (pafprocess.cpp:12-13) */
static float* g_rows = NULL;  /* [n_rows][20] */
static int g_nrows = 0;
static Peak* g_line = NULL;
static int g_nline = 0;
/* the connections of the last port_process_paf call per limb, in the order the greedy loop chose them (getters only) */
static Conn* g_conn[NUM_LIMB];
static int g_nconn[NUM_LIMB];

/* std::sort(candidates.begin(), candidates.end(), comp_candidate) (pafprocess.cpp:97, comp = a.score > b.score).
 * The order of candidates with EXACTLY equal score is whatever the standard library's algorithm leaves; such
 * ties occur in practice (two heat-map peaks refined to the same pixel), so the published libstdc++ algorithm
 * (bits/stl_algo.h: __introsort_loop, median-of-3 __unguarded_partition_pivot, threshold 16,
 * __final_insertion_sort; heap-sort fallback when the depth limit 2*floor(log2 n) is exhausted) is restated. */
#define COMP(a, b) ((a).score > (b).score)
static void swap_c(Cand* a, Cand* b) { Cand t = *a; *a = *b; *b = t; }
static void unguarded_linear_insert(Cand* last) {
    Cand val = *last;
    Cand* next = last - 1;
    while (COMP(val, *next)) { *last = *next; last = next; --next; }
    *last = val;
}
static void insertion_sort(Cand* first, Cand* last) {
    if (first == last) return;
    for (Cand* i = first + 1; i != last; ++i) {
        if (COMP(*i, *first)) {
            Cand val = *i;
            memmove(first + 1, first, (size_t)(i - first) * sizeof(Cand));
            *first = val;
        } else
            unguarded_linear_insert(i);
    }
}
static void adjust_heap(Cand* first, long hole, long len, Cand value) {   /* std::__adjust_heap + __push_heap */
    const long top = hole;
    long child = hole;
    while (child < (len - 1) / 2) {
        child = 2 * (child + 1);
        if (COMP(first[child], first[child - 1])) child--;
        first[hole] = first[child];
        hole = child;
    }
    if ((len & 1) == 0 && child == (len - 2) / 2) {
        child = 2 * (child + 1);
        first[hole] = first[child - 1];
        hole = child - 1;
    }
    long parent = (hole - 1) / 2;
    while (hole > top && COMP(first[parent], value)) {
        first[hole] = first[parent];
        hole = parent;
        parent = (hole - 1) / 2;
    }
    first[hole] = value;
}
static void heap_sort(Cand* first, Cand* last) {   /* std::__partial_sort(first, last, last) */
    const long len = last - first;
    if (len >= 2)
        for (long parent = (len - 2) / 2;; --parent) {
            adjust_heap(first, parent, len, first[parent]);
            if (parent == 0) break;
        }
    while (last - first > 1) {
        --last;
        Cand value = *last;
        *last = *first;
        adjust_heap(first, 0, last - first, value);
    }
}
static void introsort_loop(Cand* first, Cand* last, int depth_limit) {
    while (last - first > 16) {
        if (depth_limit == 0) { heap_sort(first, last); return; }
        --depth_limit;
        Cand* mid = first + (last - first) / 2;
        Cand *a = first + 1, *b = mid, *c = last - 1;   /* __move_median_to_first(first, a, b, c) */
        if (COMP(*a, *b)) {
            if (COMP(*b, *c)) swap_c(first, b);
            else if (COMP(*a, *c)) swap_c(first, c);
            else swap_c(first, a);
        } else if (COMP(*a, *c)) swap_c(first, a);
        else if (COMP(*b, *c)) swap_c(first, c);
        else swap_c(first, b);
        Cand *lo = first + 1, *hi = last;               /* __unguarded_partition(first+1, last, pivot=first) */
        for (;;) {
            while (COMP(*lo, *first)) ++lo;
            --hi;
            while (COMP(*first, *hi)) --hi;
            if (!(lo < hi)) break;
            swap_c(lo, hi);
            ++lo;
        }
        introsort_loop(lo, last, depth_limit);
        last = lo;
    }
}
static void std_sort_desc(Cand* first, int n) {
    if (n <= 0) return;
    Cand* last = first + n;
    int lg = 0;
    for (int m = n; m > 1; m >>= 1) ++lg;
    introsort_loop(first, last, 2 * lg);
    if (n > 16) {
        insertion_sort(first, first + 16);
        for (Cand* i = first + 16; i != last; ++i) unguarded_linear_insert(i);
    } else
        insertion_sort(first, last);
}

int port_process_paf(int p1, int p2, int p3, const float* peaks, int h1, int h2, int h3, const float* heatmap, int f1,
                     int f2, int f3, const float* pafmap) {
    (void)h2; (void)h3; (void)heatmap; (void)f1;
    const int total = p1 * p2;
    Peak* by_part[NUM_PART];
    int n_part[NUM_PART];
    memset(n_part, 0, sizeof(n_part));
    for (int p = 0; p < NUM_PART; ++p) by_part[p] = (Peak*)malloc(sizeof(Peak) * (total > 0 ? total : 1));
    int peak_cnt = 0;
    for (int img = 0; img < p1; ++img)
        for (int k = 0; k < p2; ++k) {            /* pafprocess.cpp:26-36 */
            const float* r = peaks + (size_t)p3 * (k + (size_t)p2 * img);
            Peak pk;
            pk.id = peak_cnt++;
            pk.x = (int)r[0];
            pk.y = (int)r[1];
            pk.score = r[2];
            int part = (int)r[4];
            by_part[part][n_part[part]++] = pk;
        }
    free(g_line);
    g_line = (Peak*)malloc(sizeof(Peak) * (total > 0 ? total : 1));
    g_nline = 0;
    for (int p = 0; p < NUM_PART; ++p)            /* pafprocess.cpp:38-43 */
        for (int i = 0; i < n_part[p]; ++i) g_line[g_nline++] = by_part[p][i];

    Conn* conns[NUM_LIMB];
    int n_conn[NUM_LIMB];
    for (int l = 0; l < NUM_LIMB; ++l) {          /* pafprocess.cpp:47-125 */
        conns[l] = NULL;
        n_conn[l] = 0;
        const Peak* A = by_part[LIMB_PARTS[l][0]];
        const Peak* B = by_part[LIMB_PARTS[l][1]];
        const int na = n_part[LIMB_PARTS[l][0]], nb = n_part[LIMB_PARTS[l][1]];
        if (na == 0 || nb == 0) continue;
        Cand* cands = (Cand*)malloc(sizeof(Cand) * (size_t)na * nb);
        int nc = 0;
        for (int a = 0; a < na; ++a)
            for (int b = 0; b < nb; ++b) {
                float vx = (float)(B[b].x - A[a].x);
                float vy = (float)(B[b].y - A[a].y);
                float norm = sqrtf(vx * vx + vy * vy);             /* :63 */
                if (norm < 1e-12) continue;                        /* :66 */
                vx = vx / norm;
                vy = vy / norm;
                const float step_x = (B[b].x - A[a].x) / (float)STEP_PAF;   /* :224-225 */
                const float step_y = (B[b].y - A[a].y) / (float)STEP_PAF;
                float scores = 0.0f;
                int crit1 = 0;
                for (int i = 0; i < STEP_PAF; ++i) {
                    int lx = (int)((double)(A[a].x + i * step_x) + 0.5);    /* roundpaf, :240-242 */
                    int ly = (int)((double)(A[a].y + i * step_y) + 0.5);
                    float px = pafmap[LIMB_PAF_CH[l][0] + (size_t)f3 * (lx + (size_t)f2 * ly)];
                    float py = pafmap[LIMB_PAF_CH[l][1] + (size_t)f3 * (lx + (size_t)f2 * ly)];
                    float s = vx * px + vy * py;
                    scores += s;
                    if (s > THRESH_VECTOR_SCORE) crit1 += 1;
                }
                double pen = 0.5 * h1 / norm - 1.0;                /* :83 (double arithmetic) */
                float crit2 = (float)((double)(scores / STEP_PAF) + (pen < 0.0 ? pen : 0.0));
                if (crit1 > THRESH_VECTOR_CNT1 && crit2 > 0) {
                    cands[nc].idx1 = a;
                    cands[nc].idx2 = b;
                    cands[nc].score = crit2;
                    ++nc;
                }
            }
        std_sort_desc(cands, nc);                                  /* :97 */
        conns[l] = (Conn*)malloc(sizeof(Conn) * (size_t)(na < nb ? na : nb));
        char* used_a = (char*)calloc(na, 1);
        char* used_b = (char*)calloc(nb, 1);
        for (int c = 0; c < nc; ++c) {                             /* :98-124 */
            if (used_a[cands[c].idx1] || used_b[cands[c].idx2]) continue;
            used_a[cands[c].idx1] = 1;
            used_b[cands[c].idx2] = 1;
            Conn cn;
            cn.pid1 = cands[c].idx1;
            cn.pid2 = cands[c].idx2;
            cn.score = cands[c].score;
            cn.cid1 = A[cands[c].idx1].id;
            cn.cid2 = B[cands[c].idx2].id;
            conns[l][n_conn[l]++] = cn;
        }
        free(used_a); free(used_b); free(cands);
    }

    /* person assembly, pafprocess.cpp:127-185.  rows live in a flat array; erased rows are flagged dead and
     * skipped, which preserves the relative order vector::erase/push_back would give. */
    int cap = 1;
    for (int l = 0; l < NUM_LIMB; ++l) cap += n_conn[l];
    float* rows = (float*)malloc(sizeof(float) * 20 * cap);
    char* alive = (char*)calloc(cap, 1);
    int nrows = 0;
    for (int l = 0; l < NUM_LIMB; ++l) {
        const int p1i = LIMB_PARTS[l][0], p2i = LIMB_PARTS[l][1];
        for (int c = 0; c < n_conn[l]; ++c) {
            const Conn cn = conns[l][c];
            int found = 0, s1 = 0, s2 = 0;
            for (int r = 0; r < nrows; ++r) {
                if (!alive[r]) continue;
                if (rows[r * 20 + p1i] == cn.cid1 || rows[r * 20 + p2i] == cn.cid2) {
                    if (found == 0) s1 = r;
                    if (found == 1) s2 = r;
                    found += 1;
                }
            }
            if (found == 1) {
                if (rows[s1 * 20 + p2i] != cn.cid2) {
                    rows[s1 * 20 + p2i] = cn.cid2;
                    rows[s1 * 20 + 19] += 1;
                    rows[s1 * 20 + 18] += g_line[cn.cid2].score + cn.score;
                }
            } else if (found == 2) {
                int membership = 0;
                for (int k = 0; k < 18; ++k)
                    if (rows[s1 * 20 + k] > 0 && rows[s2 * 20 + k] > 0) membership = 2;   /* "> 0" as in :155 */
                if (membership == 0) {
                    for (int k = 0; k < 18; ++k) rows[s1 * 20 + k] += (rows[s2 * 20 + k] + 1);
                    rows[s1 * 20 + 19] += rows[s2 * 20 + 19];
                    rows[s1 * 20 + 18] += rows[s2 * 20 + 18];
                    rows[s1 * 20 + 18] += cn.score;
                    alive[s2] = 0;
                } else {
                    rows[s1 * 20 + p2i] = cn.cid2;
                    rows[s1 * 20 + 19] += 1;
                    rows[s1 * 20 + 18] += g_line[cn.cid2].score + cn.score;
                }
            } else if (found == 0 && l < 18) {
                float* row = rows + 20 * nrows;
                for (int k = 0; k < 20; ++k) row[k] = -1;
                row[p1i] = cn.cid1;
                row[p2i] = cn.cid2;
                row[19] = 2;
                row[18] = g_line[cn.cid1].score + g_line[cn.cid2].score + cn.score;
                alive[nrows++] = 1;
            }
        }
    }
    /* prune, pafprocess.cpp:187-191 */
    free(g_rows);
    g_rows = (float*)malloc(sizeof(float) * 20 * (nrows > 0 ? nrows : 1));
    g_nrows = 0;
    for (int r = 0; r < nrows; ++r) {
        if (!alive[r]) continue;
        if (rows[r * 20 + 19] < THRESH_PART_CNT || rows[r * 20 + 18] / rows[r * 20 + 19] < THRESH_HUMAN_SCORE) continue;
        memcpy(g_rows + 20 * g_nrows++, rows + 20 * r, sizeof(float) * 20);
    }
    free(rows); free(alive);
    for (int l = 0; l < NUM_LIMB; ++l) {         /* kept for the connection getters */
        free(g_conn[l]);
        g_conn[l] = conns[l];
        g_nconn[l] = n_conn[l];
    }
    for (int p = 0; p < NUM_PART; ++p) free(by_part[p]);
    return 0;
}

int port_get_num_humans(void) { return g_nrows; }
int port_get_part_cid(int human, int part) { return (int)g_rows[human * 20 + part]; }
float port_get_score(int human) { return g_rows[human * 20 + 18] / g_rows[human * 20 + 19]; }
int port_get_part_x(int cid) { return g_line[cid].x; }
int port_get_part_y(int cid) { return g_line[cid].y; }
float port_get_part_score(int cid) { return g_line[cid].score; }
/* connection k of limb `limb` (pafprocess.cpp:113-119): peak indices within the limb's two parts and the score */
int port_get_num_connections(int limb) { return g_nconn[limb]; }
void port_get_connection(int limb, int k, int* a, int* b, float* score) {
    *a = g_conn[limb][k].pid1;
    *b = g_conn[limb][k].pid2;
    *score = g_conn[limb][k].score;
}
