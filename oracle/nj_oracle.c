/* oracle/nj_oracle.c -- a plain C restatement of NeighborJoining<>::computeTree (src/tree/NeighborJoining.cpp:33-118 of
 * FAMSA v2.5.0).  TEST INFRASTRUCTURE ONLY: built by oracle/Makefile into oracle/libnj_oracle.so.
 *
 * ISO C float arithmetic (FLT_EVAL_METHOD 0, compiled with -ffp-contract=off), so every operation is rounded on its own
 * as in the reference's build, which has no FMA to contract into.  Where the reference would go on with a step that has
 * no candidate (min_i = min_j = 0, a cluster merged with itself), this returns a status instead. */
#include <float.h>
#include <stdint.h>
#include <stdlib.h>

/* TriangleMatrix::access (src/tree/TreeDefs.h:115-120) */
static size_t tri_access(int64_t i, int64_t j) { return i >= j ? (size_t)(j + i * (i - 1) / 2) : (size_t)(i + j * (j - 1) / 2); }

typedef struct {
    float sum_of_dists;
    int row_id;
    int node_id;
} nj_cluster;

/* D: the float distance triangle (row i against j < i at i(i-1)/2 + j), updated in place as the reference does.
 * out: the merges, (left, right) per merge, n - 1 of them; *done = merges written.  Returns 0, 1 when a step has no
 * candidate (every q NaN or >= FLT_MAX), or 2 when out of memory.  n >= 2. */
int nj_oracle_tree(float* D, uint32_t n, int32_t* out, uint32_t* done)
{
    const int n_seq = (int)n;
    *done = 0;
    nj_cluster* clusters = malloc(sizeof(nj_cluster) * (n ? n : 1));
    if (!clusters) return 2;
    /* :45-55 initial sums, one float add at a time in ascending j */
    for (int i = 0; i < n_seq; ++i) {
        nj_cluster* ci = &clusters[i];
        ci->row_id = ci->node_id = i;
        ci->sum_of_dists = 0;
        for (int j = 0; j < n_seq; ++j)
            if (i != j) ci->sum_of_dists += D[tri_access(i, j)];
    }
    /* :58 merge clusters as long as more than two are left */
    int n_clusters = n_seq;
    for (int iter = 0; n_clusters > 2; ++iter) {
        /* :61-76 the first (i, j) in loop order with q < min_q, min_q from FLT_MAX */
        float min_q = FLT_MAX;
        int min_i = 0, min_j = 0;
        for (int i = 0; i < n_clusters; ++i)
            for (int j = i + 1; j < n_clusters; ++j) {
                const nj_cluster* ci = &clusters[i];
                const nj_cluster* cj = &clusters[j];
                /* :69 int (n_clusters - 2) converted to float, then product, minus the earlier sum, minus the later one */
                float q = (float)(n_clusters - 2) * D[tri_access(ci->row_id, cj->row_id)];
                q = q - ci->sum_of_dists;
                q = q - cj->sum_of_dists;
                if (q < min_q) { min_q = q; min_i = i; min_j = j; }
            }
        if (min_i == min_j) { free(clusters); return 1; }    /* no candidate: the reference merges cluster 0 with itself */
        /* :79-113 merge */
        nj_cluster* ci = &clusters[min_i];
        nj_cluster* cj = &clusters[min_j];
        const float Dij = D[tri_access(ci->row_id, cj->row_id)];
        out[2 * iter] = ci->node_id;
        out[2 * iter + 1] = cj->node_id;
        *done = (uint32_t)iter + 1;
        ci->sum_of_dists = 0;
        ci->node_id = n_seq + iter;
        for (int k = 0; k < n_clusters; ++k) {
            if (k == min_i || k == min_j) continue;
            nj_cluster* ck = &clusters[k];
            float Dik = D[tri_access(ci->row_id, ck->row_id)];
            const float Djk = D[tri_access(cj->row_id, ck->row_id)];
            const float t = Dik + Djk;
            ck->sum_of_dists -= t;                                 /* :101 */
            Dik = (t - Dij) / 2;                                   /* :104 */
            ck->sum_of_dists += Dik;
            ci->sum_of_dists += Dik;
            D[tri_access(ci->row_id, ck->row_id)] = Dik;
        }
        /* :112 erase cj, order kept */
        for (int k = min_j; k + 1 < n_clusters; ++k) clusters[k] = clusters[k + 1];
        --n_clusters;
    }
    /* :117 the two remaining clusters */
    out[2 * (n_seq - 2)] = clusters[0].node_id;
    out[2 * (n_seq - 2) + 1] = clusters[1].node_id;
    *done = n - 1;
    free(clusters);
    return 0;
}
