/* ORACLE (test infrastructure only - never linked into the product library).
 *
 * pafprocess with its five compile-time constants (the reference's pafprocess.h:7-13) as arguments.  It reuses the
 * sort, the tables and the result globals of the plain-C port, which this file includes unchanged, so the port's
 * getters read the results of either entry point:
 *   port_process_paf         the reference's constants (pafprocess_port.c, unchanged)
 *   port_process_paf_params  the same algorithm with THRESH_VECTOR_SCORE, STEP_PAF, THRESH_VECTOR_CNT1,
 *                            THRESH_PART_CNT and THRESH_HUMAN_SCORE taken from `prm`
 * Every expression keeps the reference's types: the sample test and the count compare `>` in float / int, the
 * sample step and the mean are float divisions by (float)STEP_PAF, the prune compares floats with the int part count
 * converted to float (pafprocess.cpp:57-94, 187-191, 220-242).
 *
 * Build: gcc -O2 -ffp-contract=off -shared -fPIC pafprocess_params.c -o libpafprocess_params.so -lm
 */
#include "pafprocess_port.c"

typedef struct {
    float paf_thresh;        /* THRESH_VECTOR_SCORE */
    int paf_samples;         /* STEP_PAF */
    int paf_min_above;       /* THRESH_VECTOR_CNT1 */
    int min_parts;           /* THRESH_PART_CNT */
    float min_person_score;  /* THRESH_HUMAN_SCORE */
} PortParams;

/* the candidates (after the sort) and connections of the last call, as (limb, a index, b index, score) float quads */
static float* g_pcand = NULL;
static float* g_pconn = NULL;
static long g_npcand = 0, g_npconn = 0, g_cap_pcand = 0, g_cap_pconn = 0;
static void push_quad(float** buf, long* n, long* cap, int limb, int a, int b, float score) {
    if (*n == *cap) {
        *cap = *cap ? 2 * *cap : 1024;
        *buf = (float*)realloc(*buf, sizeof(float) * 4 * (size_t)*cap);
    }
    float* q = *buf + 4 * *n;
    q[0] = (float)limb; q[1] = (float)a; q[2] = (float)b; q[3] = score;
    ++*n;
}
long port_params_num_cands(void) { return g_npcand; }
const float* port_params_cands(void) { return g_pcand; }
long port_params_num_conns(void) { return g_npconn; }
const float* port_params_conns(void) { return g_pconn; }

int port_process_paf_params(int p1, int p2, int p3, const float* peaks, int h1, int h2, int h3, const float* heatmap,
                            int f1, int f2, int f3, const float* pafmap, const PortParams* prm) {
    (void)h2; (void)h3; (void)heatmap; (void)f1;
    const int steps = prm->paf_samples;
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
    g_npcand = g_npconn = 0;
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
                const float step_x = (B[b].x - A[a].x) / (float)steps;   /* :224-225 */
                const float step_y = (B[b].y - A[a].y) / (float)steps;
                float scores = 0.0f;
                int crit1 = 0;
                for (int i = 0; i < steps; ++i) {
                    int lx = (int)((double)(A[a].x + i * step_x) + 0.5);    /* roundpaf, :240-242 */
                    int ly = (int)((double)(A[a].y + i * step_y) + 0.5);
                    float px = pafmap[LIMB_PAF_CH[l][0] + (size_t)f3 * (lx + (size_t)f2 * ly)];
                    float py = pafmap[LIMB_PAF_CH[l][1] + (size_t)f3 * (lx + (size_t)f2 * ly)];
                    float s = vx * px + vy * py;
                    scores += s;
                    if (s > prm->paf_thresh) crit1 += 1;
                }
                double pen = 0.5 * h1 / norm - 1.0;                /* :83 (double arithmetic) */
                float crit2 = (float)((double)(scores / (float)steps) + (pen < 0.0 ? pen : 0.0));
                if (crit1 > prm->paf_min_above && crit2 > 0) {
                    cands[nc].idx1 = a;
                    cands[nc].idx2 = b;
                    cands[nc].score = crit2;
                    ++nc;
                }
            }
        std_sort_desc(cands, nc);                                  /* :97 */
        for (int c = 0; c < nc; ++c) push_quad(&g_pcand, &g_npcand, &g_cap_pcand, l, cands[c].idx1, cands[c].idx2, cands[c].score);
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
            push_quad(&g_pconn, &g_npconn, &g_cap_pconn, l, cn.pid1, cn.pid2, cn.score);
        }
        free(used_a); free(used_b); free(cands);
    }

    /* person assembly, pafprocess.cpp:127-185 (no constant involved) */
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
                    if (rows[s1 * 20 + k] > 0 && rows[s2 * 20 + k] > 0) membership = 2;
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
        if (rows[r * 20 + 19] < (float)prm->min_parts || rows[r * 20 + 18] / rows[r * 20 + 19] < prm->min_person_score)
            continue;
        memcpy(g_rows + 20 * g_nrows++, rows + 20 * r, sizeof(float) * 20);
    }
    free(rows); free(alive);
    for (int l = 0; l < NUM_LIMB; ++l) free(conns[l]);
    for (int p = 0; p < NUM_PART; ++p) free(by_part[p]);
    return 0;
}
