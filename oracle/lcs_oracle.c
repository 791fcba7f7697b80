/*
 * oracle/lcs_oracle.c -- CPU restatement of the reference's bit-parallel LCS path (HP-1).
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing in the product path (famsa_b200/, include/) may call
 * into this file; only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline leg do,
 * and only as the checker.
 *
 * Parity: PINNED.  tests/test_oracle_lcs.py checks this restatement against
 *   - every entry of the reference's golden test/adeno_fiber/pid_sq.csv (242 x 242 exact LCS
 *     lengths, stored as tests/golden/adeno_fiber_lcs.npz),
 *   - the 4-sequence carry-quirk vector from SURVEY.md section 7,
 *   - the reference itself compiled into oracle/_ref (scalar and AVX2 back-ends).
 *
 * What each function follows (paths relative to /root/reference):
 *   lcs_oracle_masks      src/core/sequence.cpp:190-201      (CSequence::ComputeBitMasks)
 *   lcs_oracle_pair       src/lcs/lcsbp_classic.h:67-98      (LoopCalculate; the unrolled
 *                         variants :101-221 are the same recurrence)
 *   lcs_oracle_rows       src/tree/AbstractTreeGenerator.hpp:131-182 (calculateDistanceVector,
 *                         minus the Transform)
 *   lcs_oracle_triangle   src/tree/AbstractTreeGenerator.hpp:379-398 (calculateDistanceMatrix)
 *   lcs_oracle_transform_*  src/tree/AbstractTreeGenerator.hpp:28-82 (Transform<T, Distance>)
 *   lcs_oracle_transform_tri_f32  the same Transform<float> over a packed triangle (UPGMA.cpp:75-109, computeDistances)
 *
 * Residue codes: 0..23 ("ARNDCQEGHILKMFPSTWYVBZX*", sequence.cpp:17), 22 = unknown / padding.
 * Only codes < 20 ever set a mask bit (sequence.cpp:199).
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>
#include <float.h>

#define ORACLE_N_MASK_ROWS 32u   /* NO_SYMBOLS, defs.h:69 */
#define ORACLE_N_VALID 20        /* NO_VALID_AMINOACIDS, defs.h:72 */
#define ORACLE_UNKNOWN 22        /* UNKNOWN_SYMBOL, defs.h:67 */

/* Words needed for a row sequence of `len` residues. */
uint32_t lcs_oracle_words(uint32_t len) { return (len + 63u) / 64u; }

/* masks[c * n_words + w] bit p is set iff codes[64 w + p] == c and c < 20.
 * `masks` must hold 32 * n_words words. */
void lcs_oracle_masks(const int8_t *codes, uint32_t len, uint64_t *masks, uint32_t n_words)
{
    memset(masks, 0, sizeof(uint64_t) * ORACLE_N_MASK_ROWS * n_words);
    for (uint32_t p = 0; p < len; ++p) {
        int c = codes[p];
        if (c >= 0 && c < ORACLE_N_VALID)
            masks[(uint32_t)c * n_words + p / 64u] |= 1ull << (p % 64u);
    }
}

/* LCS length as the reference computes it: row sequence supplies `masks` (n_words words per
 * symbol, stride `stride`), `codes1` is streamed.  The carry is detected as (sum < V), which
 * drops the carry when tB is all ones and a carry arrives -- reproduced on purpose
 * (lcsbp_classic.h:55-56, SURVEY.md section 7). */
uint32_t lcs_oracle_pair(const uint64_t *masks, uint32_t stride, uint32_t n_words,
                         const int8_t *codes1, uint32_t len1)
{
    uint64_t stack_x[64];
    uint64_t *x = n_words <= 64 ? stack_x : (uint64_t *)malloc(sizeof(uint64_t) * n_words);
    for (uint32_t w = 0; w < n_words; ++w) x[w] = ~0ull;

    for (uint32_t t = 0; t < len1; ++t) {
        int c = codes1[t];
        if (c == ORACLE_UNKNOWN) continue;
        const uint64_t *m = masks + (uint32_t)c * stride;
        uint64_t carry = 0;
        for (uint32_t w = 0; w < n_words; ++w) {
            uint64_t v = x[w];
            uint64_t tb = v & m[w];
            uint64_t sum = v + tb + carry;
            carry = sum < v;
            x[w] = sum | (v - tb);
        }
    }
    uint32_t lcs = 0;
    for (uint32_t w = 0; w < n_words; ++w) lcs += (uint32_t)__builtin_popcountll(~x[w]);
    if (x != stack_x) free(x);
    return lcs;
}

/* Sequence set layout shared with the C-ABI: codes[offsets[i] .. offsets[i]+lens[i]) */
void lcs_oracle_rows(const int8_t *codes, const uint64_t *offsets, const uint32_t *lens,
                     const uint32_t *ref_ids, uint32_t n_ref,
                     const uint32_t *col_ids, uint32_t n_col, uint32_t *out)
{
    for (uint32_t r = 0; r < n_ref; ++r) {
        uint32_t ri = ref_ids[r];
        uint32_t nw = lcs_oracle_words(lens[ri]);
        uint32_t nw_alloc = nw ? nw : 1;
        uint64_t *masks = (uint64_t *)malloc(sizeof(uint64_t) * ORACLE_N_MASK_ROWS * nw_alloc);
        lcs_oracle_masks(codes + offsets[ri], lens[ri], masks, nw_alloc);
        for (uint32_t k = 0; k < n_col; ++k) {
            uint32_t ci = col_ids ? col_ids[k] : k;
            out[(size_t)r * n_col + k] =
                lcs_oracle_pair(masks, nw_alloc, nw, codes + offsets[ci], lens[ci]);
        }
        free(masks);
    }
}

/* Packed lower triangle, rows [row_begin,row_end): out[i(i-1)/2 - row_begin(row_begin-1)/2 + j]
 * for j < i (TriangleMatrix::access, src/tree/TreeDefs.h:114-119).  Row i supplies the masks. */
void lcs_oracle_triangle(const int8_t *codes, const uint64_t *offsets, const uint32_t *lens,
                         uint32_t row_begin, uint32_t row_end, uint32_t *out)
{
    size_t base = (size_t)row_begin * (row_begin ? row_begin - 1 : 0) / 2;
    for (uint32_t i = row_begin; i < row_end; ++i) {
        uint32_t nw = lcs_oracle_words(lens[i]);
        uint32_t nw_alloc = nw ? nw : 1;
        uint64_t *masks = (uint64_t *)malloc(sizeof(uint64_t) * ORACLE_N_MASK_ROWS * nw_alloc);
        lcs_oracle_masks(codes + offsets[i], lens[i], masks, nw_alloc);
        size_t row_off = (size_t)i * (i ? i - 1 : 0) / 2 - base;
        for (uint32_t j = 0; j < i; ++j)
            out[row_off + j] = lcs_oracle_pair(masks, nw_alloc, nw, codes + offsets[j], lens[j]);
        free(masks);
    }
}

/* ---- Transform<T, Distance> (AbstractTreeGenerator.hpp:28-82) ----
 * kind: 0 = indel075_div_lcs, 1 = indel_div_lcs, 2 = pairwise_identity. */
double lcs_oracle_transform_f64(int kind, uint32_t lcs, uint32_t len1, uint32_t len2)
{
    if (kind == 2) {
        uint32_t m = len1 < len2 ? len1 : len2;
        return (double)lcs / m;
    }
    double indel = (double)(len1 + len2 - 2 * lcs);
    if (!lcs) return nextafter(DBL_MAX, 0.0);
    if (kind == 0) return (double)pow((double)(uint32_t)indel, 0.75) / (double)lcs;
    return indel / lcs;
}

float lcs_oracle_transform_f32(int kind, uint32_t lcs, uint32_t len1, uint32_t len2)
{
    if (kind == 2) {
        uint32_t m = len1 < len2 ? len1 : len2;
        return (float)lcs / m;
    }
    float indel = (float)(len1 + len2 - 2 * lcs);
    /* nextafter(numeric_limits<float>::max(), 0) promotes to double, then narrows (hpp:60) */
    if (!lcs) return (float)nextafter((double)FLT_MAX, 0.0);
    /* table entry is (float) pow((double) i, 0.75), hpp:46 */
    if (kind == 0) return (float)pow((double)(uint32_t)indel, 0.75) / (float)lcs;
    return indel / lcs;
}

/* lcs_oracle_transform_f32 of every pair of a packed LCS triangle (rows 0..n, elem_bytes 2 or 4, row i at i(i-1)/2):
 * out[i(i-1)/2 + j] = Transform(lcs, lens[i], lens[j]) -- the float triangle computeDistances fills
 * (src/tree/UPGMA.cpp:75-109) -- with the pow table built once instead of per pair. */
void lcs_oracle_transform_tri_f32(int kind, const void *lcs, int elem_bytes, const uint32_t *lens, uint32_t n,
                                  float *out)
{
    uint32_t max_len = 0;
    for (uint32_t i = 0; i < n; ++i) max_len = lens[i] > max_len ? lens[i] : max_len;
    float *pow075 = NULL;
    if (kind == 0) {
        pow075 = (float *)malloc(sizeof(float) * (2 * (size_t)max_len + 1));
        for (size_t k = 0; k <= 2 * (size_t)max_len; ++k) pow075[k] = (float)pow((double)k, 0.75);
    }
    const float never = (float)nextafter((double)FLT_MAX, 0.0);
    for (uint32_t i = 1; i < n; ++i) {
        const size_t base = (size_t)i * (i - 1) / 2;
        for (uint32_t j = 0; j < i; ++j) {
            const uint32_t l = elem_bytes == 2 ? ((const uint16_t *)lcs)[base + j] : ((const uint32_t *)lcs)[base + j];
            float d;
            if (kind == 2) {
                const uint32_t m = lens[i] < lens[j] ? lens[i] : lens[j];
                d = (float)l / m;
            } else if (!l) {
                d = never;
            } else {
                const uint32_t indel = lens[i] + lens[j] - 2 * l;       /* wraps as in the scalar form */
                const float p = kind != 0 ? 0.0f
                              : indel <= 2 * max_len ? pow075[indel] : (float)pow((double)(uint32_t)(float)indel, 0.75);
                d = kind == 0 ? p / (float)l : (float)indel / l;
            }
            out[base + j] = d;
        }
    }
    free(pow075);
}
