/*
 * oracle/upgma_oracle.c -- CPU restatement of the reference's UPGMA agglomeration.
 *
 * TEST INFRASTRUCTURE ONLY, like lcs_oracle.c: nothing in famsa_b200/ or include/ calls into it.
 *
 * upgma_oracle_tree restates UPGMA<>::computeTree<MODIFIED> (src/tree/UPGMA.cpp:114-295) as its plain sequential loops:
 *   - the init double loop over the packed triangle, each row's cache replaced only by a strictly smaller distance
 *     than the one it holds (starting from BIG_DIST = 1e29f, UPGMA.h:82), partners met in ascending index order;
 *   - the scan for the live row with the smallest cached distance (the first such row);
 *   - the new-row loop: the averaged distance to the new node overwrites row L, a row whose cached neighbour was R is
 *     relabelled to L and keeps its old distance (no re-evaluation, :256-257), the first minimum of the new row
 *     becomes L's cache;
 *   - row L reused for the new node, row R deleted.
 * Float32 throughout.  This file is ISO C (-std=c11), so the compiler contracts no a*b+c into an FMA: the MAFFT
 * average 0.05f*(x+y) + 0.9f*min(x,y) (:33) is rounded after each product and after the sum, as in the reference's
 * build (-mavx2, no -mfma).
 *
 * Where the reference would index out of range (no live row with a finite cache: a pair without a common residue has
 * distance FLT_MAX, and every average with it stays >= BIG_DIST), the restatement stops and returns 1.
 *
 * Switches that change the algorithm, used only to generate witnesses (tests/golden/make_upgma.py) that tell the
 * reference's behaviour from a plausible alternative:
 *   fresh_cache   recompute every live row's true nearest neighbour after each merge (the cache is never stale);
 *   avg_mode 1    the modified average evaluated in double from the float inputs and rounded once;
 *   avg_mode 2    the modified average as fmaf(0.05f, x+y, 0.9f*min(x,y)).
 */
#include <stdint.h>
#include <stdlib.h>
#include <math.h>

#define UPGMA_BIG 1e29f
#define UPGMA_NONE 0x7FFFFFFFu

static size_t tri_at(uint32_t a, uint32_t b)
{
    uint32_t hi = a > b ? a : b, lo = a > b ? b : a;
    return (size_t)hi * (hi - 1) / 2 + lo;
}

static float average(float x, float y, int modified, int avg_mode)
{
    if (!modified) return (x + y) * 0.5f;
    float m = y < x ? y : x;                                    /* std::min(x, y) */
    if (avg_mode == 1) return (float)((double)0.05f * ((double)x + (double)y) + (double)0.9f * (double)m);
    if (avg_mode == 2) return fmaf(0.05f, x + y, 0.9f * m);
    float a = 0.05f * (x + y);
    float b = 0.9f * m;
    return a + b;
}

/* Row r's nearest live neighbour by the init loop's rule: strictly smaller than BIG_DIST, lowest partner on ties. */
static void nearest(const float *dist, const uint32_t *node, uint32_t n, uint32_t r, float *mind, uint32_t *nn)
{
    float best = UPGMA_BIG;
    uint32_t who = UPGMA_NONE;
    for (uint32_t p = 0; p < n; ++p) {
        if (p == r || node[p] == UPGMA_NONE) continue;
        float d = dist[tri_at(r, p)];
        if (d < best) { best = d; who = p; }
    }
    mind[r] = best;
    nn[r] = who;
}

/* dist: packed lower triangle of n rows (row i at i(i-1)/2), overwritten as the reference overwrites it.
 * out[2k], out[2k+1] = children of internal node n + k.  *n_done = merges written.  Returns 0, or 1 when no live row
 * has a finite cached distance before the last merge. */
int upgma_oracle_tree(float *dist, uint32_t n, int modified, int avg_mode, int fresh_cache, int32_t *out,
                      uint32_t *n_done)
{
    *n_done = 0;
    if (n < 2) return 0;
    float *mind = (float *)malloc(sizeof(float) * n);
    uint32_t *nn = (uint32_t *)malloc(sizeof(uint32_t) * n);
    uint32_t *node = (uint32_t *)malloc(sizeof(uint32_t) * n);
    int status = 0;
    for (uint32_t i = 0; i < n; ++i) { mind[i] = UPGMA_BIG; nn[i] = UPGMA_NONE; node[i] = i; }

    for (uint32_t i = 1; i < n; ++i) {
        const float *row = dist + (size_t)i * (i - 1) / 2;
        for (uint32_t j = 0; j < i; ++j) {
            float d = row[j];
            if (d < mind[i]) { mind[i] = d; nn[i] = j; }
            if (d < mind[j]) { mind[j] = d; nn[j] = i; }
        }
    }

    for (uint32_t k = 0; k + 1 < n; ++k) {
        uint32_t L = UPGMA_NONE, R = UPGMA_NONE;
        float best = UPGMA_BIG;
        for (uint32_t j = 0; j < n; ++j) {
            if (node[j] == UPGMA_NONE) continue;
            if (mind[j] < best) { best = mind[j]; L = j; R = nn[j]; }
        }
        if (L == UPGMA_NONE) { status = 1; break; }

        float new_min = UPGMA_BIG;
        uint32_t new_nn = UPGMA_NONE;
        for (uint32_t j = 0; j < n; ++j) {
            if (j == L || j == R || node[j] == UPGMA_NONE) continue;
            size_t vL = tri_at(L, j), vR = tri_at(R, j);
            float d = average(dist[vL], dist[vR], modified, avg_mode);
            if (nn[j] == R) nn[j] = L;
            dist[vL] = d;
            if (d < new_min) { new_min = d; new_nn = j; }
        }

        out[2 * k] = (int32_t)node[L];
        out[2 * k + 1] = (int32_t)node[R];
        node[L] = n + k;
        nn[L] = new_nn;
        mind[L] = new_min;
        node[R] = UPGMA_NONE;
        *n_done = k + 1;

        if (fresh_cache)
            for (uint32_t j = 0; j < n; ++j)
                if (node[j] != UPGMA_NONE) nearest(dist, node, n, j, mind, nn);
    }
    free(mind);
    free(nn);
    free(node);
    return status;
}
