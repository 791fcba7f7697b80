// famsa_prof_refine: CFAMSA::RefineAlignment (src/msa_refinement.cpp:73-217) on the resident final profile.
//
// The alignment being refined stays on the device, column-major (column c = n_rows bytes, rows in id order, residue codes
// of defs.h and GAP = 30).  The host keeps only the loop's control -- the generator rnd_rfn, the split vectors already
// tried and prev_total_score -- and per try receives O(width + n_rows) bytes: the split, the two side widths, the gap
// counts of the candidate and the terms of its total score.  One try:
//   k_ref_split + k_ref_scan          split vector (RefineMostEmptyAndFullColumn's column, or RefineRandom's vector from
//                                     the host), the columns each side keeps (Condense), side widths     -> host, sync 1
//   k_ref_condense, k_ref_row_ends,   the two sides' rows without their all-gap columns, and their counters / scores
//   k_ref_tables                      (CalculateCountersScores for a gapped multi-row profile, profile.cpp:101-235)
//   k_ref_optimize                    OptimizeGaps (profile.cpp:436-689), one block per side, on the rows only
//   famsa_prof_merge_batch's path     Align + ConstructProfile of the two sides (unbanded, as with no_threads > 1)  sync 2
//   k_ref_path_index, k_ref_rebuild   the candidate's rows: each side's optimised rows with the path's gap columns, and
//                                     whether they equal the current alignment (CProfile::operator==)
//   k_ref_run_ends, k_ref_score_cols, CalculateTotalScore (profile.cpp:1368-1542) from the candidate's merged counters
//   k_ref_score_runs, k_ref_gapstats  and rows, and the candidate's gap counts (GetGapStats)                -> host, sync 3
// DESIGN.md §4d has the reasoning, the launch list and the formulation of the gap-open count.
//
// famsa_prof_put_rows (a resident profile from a finished alignment, CFAMSA::alignProfiles' inputs) builds its tables with
// the same k_ref_row_ends + k_ref_tables pass (gapped_tables) as a try's two sides.
#include <algorithm>
#include <chrono>
#include <cstring>
#include <random>
#include <vector>

#include "ctx.h"
#include "prof_dev.cuh"

namespace fb {

namespace {

constexpr int kRT = 256;          // threads of the per-column kernels
constexpr int kScanT = 1024;      // threads of the single-block scans
constexpr int kOptT = 512;        // threads of OptimizeGaps' block
constexpr size_t kMaxHistBytes = 200u << 10;   // k_ref_score_runs' histogram of run ends: widths up to ~51 000 columns

__device__ __forceinline__ bool is_gap(uint8_t v) { return v == kGAP; }

// sum over the block (every thread gets it); sh: >= 32 words, not in use by the caller
template <class T>
__device__ T block_sum(T v, T* sh)
{
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    T t = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += sh[w];
    return t;
}

// exclusive prefix sum over the block in thread order; *total = the block's sum.  sh: >= 32 words.
__device__ int block_excl_scan(int v, int* sh, int* total)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    int x = v;
    for (int o = 1; o < 32; o <<= 1) {
        const int y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    __syncthreads();
    if (lane == 31) sh[warp] = x;
    __syncthreads();
    if (warp == 0) {
        int w = lane < nwarps ? sh[lane] : 0;
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += y;
        }
        sh[lane] = w;
    }
    __syncthreads();
    *total = sh[nwarps - 1];
    return (warp ? sh[warp - 1] : 0) + x - v;
}

// gap count of every column (GetGapStats, profile.cpp:360-376: stats[c] = card - residues in column c); one block per column
__global__ void __launch_bounds__(kRT) k_ref_gapstats(const uint8_t* __restrict__ A, uint32_t n, uint32_t* __restrict__ stats)
{
    __shared__ int sh[32];
    const uint8_t* col = A + (size_t)blockIdx.x * n;
    int g = 0;
    for (uint32_t r = threadIdx.x; r < n; r += blockDim.x) g += is_gap(col[r]);
    g = block_sum(g, sh);
    if (threadIdx.x == 0) stats[blockIdx.x + 1] = (uint32_t)g;
}

// The split and the columns each side keeps.  col >= 1: RefineMostEmptyAndFullColumn's labels (msa_refinement.cpp:55-65):
// a row goes to profile1 (dest 1) when its gap state in column col equals row 0's, so row 0 is always in profile1;
// col == 0: dest[] was uploaded by the host (RefineRandom).  keep[s * W + c] = side s has a residue in column c.
__global__ void __launch_bounds__(kRT) k_ref_split(const uint8_t* __restrict__ A, uint32_t n, uint32_t W, uint32_t col,
                                                   uint8_t* __restrict__ dest, uint8_t* __restrict__ keep)
{
    const uint8_t* c = A + (size_t)blockIdx.x * n;
    const uint8_t* pick = col ? A + (size_t)(col - 1) * n : nullptr;
    const bool g0 = col ? is_gap(pick[0]) : false;
    bool has[2] = {false, false};
    for (uint32_t r = threadIdx.x; r < n; r += blockDim.x) {
        const int d = col ? (is_gap(pick[r]) == g0) : dest[r];
        if (!is_gap(c[r])) has[d] = true;
    }
    const int k0 = __syncthreads_or(has[0]), k1 = __syncthreads_or(has[1]);
    if (threadIdx.x == 0) { keep[blockIdx.x] = (uint8_t)k0; keep[W + blockIdx.x] = (uint8_t)k1; }
    if (col && blockIdx.x == 0)
        for (uint32_t r = threadIdx.x; r < n; r += blockDim.x) dest[r] = is_gap(pick[r]) == g0;
}

// One block: map[s * W + c] = column of side s that column c becomes (-1: removed by Condense), ridx[r] = row r's index
// within its side; info = {W0, W1, n0, n1}.
__global__ void __launch_bounds__(kScanT) k_ref_scan(const uint8_t* __restrict__ keep, uint32_t W, const uint8_t* __restrict__ dest,
                                                     uint32_t n, int* __restrict__ map, uint32_t* __restrict__ ridx,
                                                     uint32_t* __restrict__ info)
{
    __shared__ int sh[32];
    for (int s = 0; s < 2; ++s) {
        int carry = 0;
        for (uint32_t base = 0; base < W; base += blockDim.x) {
            const uint32_t c = base + threadIdx.x;
            const int v = c < W ? keep[s * W + c] : 0;
            int tot;
            const int ex = block_excl_scan(v, sh, &tot);
            if (c < W) map[s * W + c] = v ? carry + ex : -1;
            carry += tot;
        }
        if (threadIdx.x == 0) info[s] = (uint32_t)carry;
    }
    int ones = 0;
    for (uint32_t base = 0; base < n; base += blockDim.x) {
        const uint32_t r = base + threadIdx.x;
        const int v = r < n ? dest[r] : 0;
        int tot;
        const int ex = block_excl_scan(v, sh, &tot);
        if (r < n) ridx[r] = v ? ones + ex : r - (ones + ex);
        ones += tot;
    }
    if (threadIdx.x == 0) { info[2] = n - ones; info[3] = ones; }
}

struct Sides {
    uint8_t* rows[2];     // column-major rows of side 0 (profile2) and side 1 (profile1)
    uint32_t n[2], w[2];
};

// Condense (profile.cpp:380-432) of both sides at once: element (c, r) of the alignment goes to its side's column map[c]
__global__ void k_ref_condense(const uint8_t* __restrict__ A, uint32_t n, uint32_t W, const uint8_t* __restrict__ dest,
                               const int* __restrict__ map, const uint32_t* __restrict__ ridx, Sides S)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)n * W) return;
    const uint32_t c = (uint32_t)(i / n), r = (uint32_t)(i % n);
    const int d = dest[r];
    const int m = map[d * W + c];
    if (m >= 0) S.rows[d][(size_t)m * S.n[d] + ridx[r]] = A[i];
}

// first / last residue column (1-based) of every row of a side; blockIdx.y = side
__global__ void k_ref_row_ends(Sides S, uint32_t* __restrict__ first, uint32_t* __restrict__ last)
{
    const int s = blockIdx.y;
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= S.n[s]) return;
    uint32_t f = 0, l = 0;
    for (uint32_t c = 0; c < S.w[s]; ++c)
        if (!is_gap(S.rows[s][(size_t)c * S.n[s] + r])) { if (!f) f = c + 1; l = c + 1; }
    const uint32_t o = s ? 0 : S.n[1];
    first[o + r] = f; last[o + r] = l;
}

struct SideTables { long long* scores[2]; int* counters[2]; };

// CalculateCountersScores (profile.cpp:101-235) of both sides: block (column c, side).  Counters of a gapped row: its
// residue, or for a gap GAP_TERM_OPEN / GAP_TERM_EXT before its first and after its last residue (the first such column
// opens) and GAP_OPEN / GAP_EXT between (a gap right of a residue opens).
__global__ void __launch_bounds__(kRT) k_ref_tables(Sides S, const uint32_t* __restrict__ first, const uint32_t* __restrict__ last,
                                                    SideTables T, const long long* __restrict__ sm,
                                                    long long go, long long ge, long long to, long long te)
{
    __shared__ int cnt[kRows];
    const int s = blockIdx.y;
    const uint32_t c = blockIdx.x, ns = S.n[s];
    if (c > S.w[s]) return;
    if (threadIdx.x < kRows) cnt[threadIdx.x] = 0;
    __syncthreads();
    if (c) {
        const uint8_t* col = S.rows[s] + (size_t)(c - 1) * ns;
        const uint32_t o = s ? 0 : S.n[1];
        for (uint32_t r = threadIdx.x; r < ns; r += blockDim.x) {
            const uint8_t v = col[r];
            int k;
            if (!is_gap(v)) k = v < kNAA ? v : 22;
            else if (c < first[o + r]) k = c == 1 ? kTO : kTE;
            else if (c > last[o + r]) k = c == last[o + r] + 1 ? kTO : kTE;
            else k = is_gap((col - ns)[r]) ? kGE : kGO;
            atomicAdd(&cnt[k], 1);
        }
    }
    __syncthreads();
    if (threadIdx.x >= 32) return;
    const int lane = threadIdx.x;
    const int cn = cnt[lane];
    long long sc;
    if (!c) sc = gap_lanes(lane, ns, go, ge, to, te);
    else {
        int tot = 0;
        long long sym = 0;
        for (int k = 0; k < kNAA; ++k) {
            const int nk = cnt[k];
            tot += nk;
            if (lane < kNAA && nk) sym += sm[k * kNAA + lane] * nk;
        }
        const long long gap_cost = cnt[kGO] * go + cnt[kTO] * to + cnt[kGE] * ge + cnt[kTE] * te;
        sc = lane < kNAA ? gap_cost + sym : gap_lanes(lane, tot, go, ge, to, te);
    }
    T.scores[s][(size_t)c * kRows + lane] = sc;
    T.counters[s][(size_t)c * kRows + lane] = cn;
}

enum : uint8_t { kNone, kLeft, kRight, kBoth, kBothNE, kBothToLeft, kBothToRight };

// OptimizeGaps (profile.cpp:436-689), one block per side.  The candidates are the columns i < W where no row has residues
// in both i and i+1 (gap_sym_broundaries), visited right to left; max_possible_col_id carries over, so the scan is
// sequential, and every loop over the rows inside a step is a block-wide one.  The reference decodes the gap pattern
// once; an exchange moves gaps only inside (left_col, right_col] and every later step reads columns < left_col, so reading
// the rows as they are is the same.  Every row has a gap at a candidate column or the next, so its exch_type vector
// (filled only for such rows, indexed by row) is indexed consistently.
__global__ void __launch_bounds__(kOptT) k_ref_optimize(Sides S, uint8_t* __restrict__ type_all, int* __restrict__ rf_all, int* __restrict__ rs_all)
{
    __shared__ int sh[32];
    const int s = blockIdx.x;
    uint8_t* A = S.rows[s];
    const uint32_t n = S.n[s];
    const int W = (int)S.w[s];
    const uint32_t o = s ? 0 : S.n[1];
    uint8_t* type = type_all + o;
    int* rf = rf_all + o;
    int* rs = rs_all + o;
    auto g = [&](int c, uint32_t r) { return is_gap(A[(size_t)(c - 1) * n + r]); };   // 1-based column
    int maxp = W;
    for (int curr = W - 1; curr >= 1; --curr) {
        if (curr + 2 > maxp) continue;
        bool ok = true;
        for (uint32_t r = threadIdx.x; r < n; r += blockDim.x) ok &= g(curr, r) || g(curr + 1, r);
        if (!__syncthreads_and(ok)) continue;
        for (uint32_t r = threadIdx.x; r < n; r += blockDim.x) {
            const bool a = g(curr, r), b = g(curr + 1, r);
            type[r] = a && b ? kBoth : a ? kLeft : kRight;
            rf[r] = a; rs[r] = b;
        }
        int L;
        for (L = 2; curr + 1 - L > 0; ++L) {
            const int col = curr + 1 - L;
            bool stop = false;
            for (uint32_t r = threadIdx.x; r < n; r += blockDim.x) {
                if (type[r] == kLeft) { if (g(col, r)) rf[r] = L; else stop = true; }
                else if (type[r] == kBoth) { if (g(col, r)) rf[r] = L; else type[r] = kBothNE; }
            }
            if (__syncthreads_or(stop)) break;
        }
        for (uint32_t r = threadIdx.x; r < n; r += blockDim.x) if (type[r] == kBothNE) type[r] = kBoth;
        int R;
        for (R = 2; curr + R < maxp; ++R) {
            const int col = curr + R;
            bool stop = false;
            for (uint32_t r = threadIdx.x; r < n; r += blockDim.x) {
                if (type[r] == kRight) { if (g(col, r)) rs[r] = R; else stop = true; }
                else if (type[r] == kBoth) { if (g(col, r)) rs[r] = R; else type[r] = kBothNE; }
            }
            if (__syncthreads_or(stop)) break;
        }
        bool unprofitable = false;
        for (uint32_t r = threadIdx.x; r < n; r += blockDim.x) {
            if (type[r] == kBothNE) type[r] = kBoth;
            if (type[r] != kBoth) continue;
            const bool l = rf[r] >= L - 1, rr = rs[r] >= R - 1;
            if (!l && !rr) unprofitable = true;
            else if (l && rr) ;
            else type[r] = l ? kBothToLeft : kBothToRight;
        }
        if (__syncthreads_or(unprofitable)) continue;
        if (curr - L <= 0 || curr + R >= W) continue;
        const int left_col = curr - (L - 1), right_col = curr + R;
        int bal = 0;
        for (uint32_t r = threadIdx.x; r < n; r += blockDim.x) {
            const uint8_t t = type[r];
            const bool gl = g(left_col, r), gr = g(right_col, r);
            if (t == kLeft) bal += (gr ? 0 : 1) - (gl ? 0 : 1);
            else if (t == kRight) bal += (gl ? 0 : 1) - (gr ? 0 : 1);
            else if (t == kBothToLeft) bal += !gr;
            else if (t == kBothToRight) bal += !gl;
        }
        if (block_sum(bal, sh) >= 0) continue;
        // the exchange: InsertGap / RemoveGap of profile.cpp:661-676 as moves inside the window (left_col, right_col)
        for (uint32_t r = threadIdx.x; r < n; r += blockDim.x) {
            const uint8_t t = type[r];
            uint8_t* row = A + r;
            auto at = [&](int c) -> uint8_t& { return row[(size_t)(c - 1) * n]; };
            if (t == kLeft || t == kBothToLeft) {            // the L-1 gaps left of curr+1 move to just before right_col
                for (int c = left_col + 1; c <= right_col - L; ++c) at(c) = at(c + L - 1);
                for (int c = right_col - L + 1; c < right_col; ++c) at(c) = kGAP;
            } else if (t == kRight || t == kBothToRight) {   // the R-1 gaps right of curr move to just after left_col
                for (int c = right_col - 1; c >= left_col + R; --c) at(c) = at(c - (R - 1));
                for (int c = left_col + 1; c < left_col + R; ++c) at(c) = kGAP;
            }
        }
        maxp = left_col;
    }
}

// merged column k -> column of the DP's row profile (iR) / column profile (iC) it holds, -1 for a gap column (H: gap in
// the row profile's members, V: in the column profile's); one block
__global__ void __launch_bounds__(kScanT) k_ref_path_index(const uint8_t* __restrict__ path, uint32_t len, int* __restrict__ iR, int* __restrict__ iC)
{
    __shared__ int sh[32];
    int cr = 0, cc = 0;
    for (uint32_t base = 0; base < len; base += blockDim.x) {
        const uint32_t k = base + threadIdx.x;
        const uint8_t d = k < len ? path[k] : 1;
        const int vr = k < len && d != 1, vc = k < len && d != 2;
        int tr, tc;
        const int er = block_excl_scan(vr, sh, &tr);
        const int ec = block_excl_scan(vc, sh, &tc);
        if (k < len) { iR[k] = vr ? cr + er : -1; iC[k] = vc ? cc + ec : -1; }
        cr += tr; cc += tc;
    }
}

// the candidate's rows in id order: row r of side dest[r] (after OptimizeGaps) with the path's gap columns; when the
// widths agree, info[4] is set if any byte differs from the current alignment
__global__ void k_ref_rebuild(const uint8_t* __restrict__ A, uint8_t* __restrict__ C, uint32_t n, uint32_t Wm, int row_side, Sides S,
                              const uint8_t* __restrict__ dest, const uint32_t* __restrict__ ridx, const int* __restrict__ iR,
                              const int* __restrict__ iC, int compare, uint32_t* __restrict__ info)
{
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    bool diff = false;
    if (i < (size_t)n * Wm) {
        const uint32_t k = (uint32_t)(i / n), r = (uint32_t)(i % n);
        const int d = dest[r];
        const int src = d == row_side ? iR[k] : iC[k];
        const uint8_t v = src < 0 ? (uint8_t)kGAP : S.rows[d][(size_t)src * S.n[d] + ridx[r]];
        C[i] = v;
        diff = compare && A[i] != v;
    }
    if (__any_sync(0xffffffffu, diff) && (threadIdx.x & 31) == 0) atomicOr(&info[4], 1u);
}

// E[c][r] = last column (1-based) of the gap run through column c+1 of row r, 0 where row r has a residue
__global__ void k_ref_run_ends(const uint8_t* __restrict__ A, uint32_t n, uint32_t W, uint32_t* __restrict__ E)
{
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= n) return;
    uint32_t e = 0;
    for (uint32_t c = W; c-- > 0;) {
        e = is_gap(A[(size_t)c * n + r]) ? (e ? e : c + 1) : 0;
        E[(size_t)c * n + r] = e;
    }
}

// acc[0..2] += CalculateTotalScore's per-column terms (profile.cpp:1389-1411) from the merged counters: symbol pairs,
// residue x internal-gap and residue x terminal-gap pairs.  One warp per column.
__global__ void __launch_bounds__(kRT) k_ref_score_cols(const int* __restrict__ counters, uint32_t W, uint32_t card,
                                                        const long long* __restrict__ sm, unsigned long long* __restrict__ acc)
{
    __shared__ long long sh[32];
    const int lane = threadIdx.x & 31;
    const uint32_t c = 1 + blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    long long pair = 0, ext = 0, text = 0;
    if (c <= W) {
        const int cn = counters[(size_t)c * kRows + lane];
        const long long n1 = lane < kNAA ? cn : 0;
        for (int k = 0; k < kNAA; ++k) {
            const long long n2 = __shfl_sync(0xffffffffu, cn, k);
            if (k > lane && n1 && n2) pair += sm[lane * kNAA + k] * n1 * n2;
        }
        if (n1) pair += sm[lane * kNAA + lane] * n1 * (n1 - 1) / 2;
        const long long ng = __shfl_sync(0xffffffffu, cn, kGO) + __shfl_sync(0xffffffffu, cn, kGE);
        const long long nt = __shfl_sync(0xffffffffu, cn, kTO) + __shfl_sync(0xffffffffu, cn, kTE);
        if (lane == 0) { const long long ns = (long long)card - ng - nt; ext = ns * ng; text = ns * nt; }
    }
    pair = block_sum(pair, sh);
    ext = block_sum(ext, sh);
    text = block_sum(text, sh);
    if (threadIdx.x == 0) {
        atomicAdd(&acc[0], (unsigned long long)pair);
        atomicAdd(&acc[1], (unsigned long long)ext);
        atomicAdd(&acc[2], (unsigned long long)text);
    }
}

// acc[3] / acc[4] += the gap opens / terminal gap opens of the runs that start in column s = blockIdx.x + 1
// (profile.cpp:1503-1525).  For a run [s, e] of one row the reference adds, once per row holding that exact run,
// n - (number of runs [s', e'] of all rows with s' <= s and e' >= e); a run containing column s is the one run through s
// of its row, so that number is how many rows have a gap at s whose run ends at e or later: a histogram of the run ends
// through s in shared memory, summed from the right.  Terminal: s == 1 or e == W.
__global__ void __launch_bounds__(kRT) k_ref_score_runs(const uint32_t* __restrict__ E, uint32_t n, uint32_t W, unsigned long long* __restrict__ acc)
{
    extern __shared__ int hist[];
    __shared__ int sh[32];
    __shared__ long long shl[32];
    const uint32_t s = blockIdx.x + 1;
    const uint32_t* es = E + (size_t)(s - 1) * n;
    const uint32_t* ep = s > 1 ? E + (size_t)(s - 2) * n : nullptr;
    uint32_t maxe = 0;
    bool starts = false;
    for (uint32_t r = threadIdx.x; r < n; r += blockDim.x) {
        const uint32_t e = es[r];
        maxe = max(maxe, e);
        starts |= e && (!ep || !ep[r]);
    }
    if (!__syncthreads_or(starts)) return;
    for (int o = 16; o; o >>= 1) maxe = max(maxe, __shfl_xor_sync(0xffffffffu, maxe, o));
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = (int)maxe;
    __syncthreads();
    maxe = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) maxe = max(maxe, (uint32_t)sh[w]);
    const uint32_t len = maxe - s + 1;
    for (uint32_t k = threadIdx.x; k < len; k += blockDim.x) hist[k] = 0;
    __syncthreads();
    for (uint32_t r = threadIdx.x; r < n; r += blockDim.x)
        if (es[r]) atomicAdd(&hist[es[r] - s], 1);
    __syncthreads();                                                // every bin complete before the scan reads it
    int carry = 0;                                                  // suffix sums: hist[k] = rows whose run ends at >= s + k
    for (uint32_t base = 0; base < len; base += blockDim.x) {
        const uint32_t j = base + threadIdx.x;
        const int v = j < len ? hist[len - 1 - j] : 0;
        int tot;
        const int ex = block_excl_scan(v, sh, &tot);
        if (j < len) hist[len - 1 - j] = carry + ex + v;
        carry += tot;
        __syncthreads();
    }
    long long open = 0, topen = 0;
    for (uint32_t r = threadIdx.x; r < n; r += blockDim.x) {
        const uint32_t e = es[r];
        if (!e || (ep && ep[r])) continue;
        const long long v = (long long)n - hist[e - s];
        if (s == 1 || e == W) topen += v; else open += v;
    }
    open = block_sum(open, shl);
    topen = block_sum(topen, shl);
    if (threadIdx.x == 0) {
        atomicAdd(&acc[3], (unsigned long long)open);
        atomicAdd(&acc[4], (unsigned long long)topen);
    }
}

// row-major <-> column-major
__global__ void k_ref_transpose(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, uint32_t rows, uint32_t cols)
{
    __shared__ uint8_t t[32][33];
    const uint32_t c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
    for (uint32_t y = threadIdx.y; y < 32; y += blockDim.y) {
        const uint32_t r = r0 + y, c = c0 + threadIdx.x;
        if (r < rows && c < cols) t[y][threadIdx.x] = in[(size_t)r * cols + c];
    }
    __syncthreads();
    for (uint32_t y = threadIdx.y; y < 32; y += blockDim.y) {
        const uint32_t c = c0 + y, r = r0 + threadIdx.x;
        if (r < rows && c < cols) out[(size_t)c * rows + r] = t[threadIdx.x][y];
    }
}

unsigned blocks(size_t n, unsigned t) { return (unsigned)((n + t - 1) / t); }

// CalculateCountersScores (profile.cpp:101-235) of the column-major gapped rows of S's sides 0..n_sides-1 into T: the one
// builder of tables from gapped rows, for a refinement try's two sides and for famsa_prof_put_rows' one alignment (side 0,
// with S.n[1] = 0).  first / last: scratch of S.n[0] + S.n[1] words each.
int gapped_tables(famsa_ctx* ctx, cudaStream_t st, const Sides& S, int n_sides, uint32_t* first, uint32_t* last,
                  const SideTables& T, const int64_t g[4])
{
    const uint32_t nmax = n_sides > 1 ? std::max(S.n[0], S.n[1]) : S.n[0], wmax = n_sides > 1 ? std::max(S.w[0], S.w[1]) : S.w[0];
    k_ref_row_ends<<<dim3(blocks(nmax, 128), n_sides), 128, 0, st>>>(S, first, last);
    FB_CUDA(cudaGetLastError());
    k_ref_tables<<<dim3(wmax + 1, n_sides), kRT, 0, st>>>(S, first, last, T, ctx->prof.d_sm.as<long long>(), (long long)g[0],
                                                         (long long)g[1], (long long)g[2], (long long)g[3]);
    FB_CUDA(cudaGetLastError());
    ctx->launches += 2;
    return FAMSA_OK;
}

// The device state of one famsa_prof_refine call.
struct Run {
    famsa_ctx* ctx;
    RefineState& R;
    cudaStream_t st;
    uint32_t n, W;                 // rows, width of the current alignment (R.d_cur)
    int64_t g[4];
    // per-row scratch (R.d_rows): dest, ridx, first, last, OptimizeGaps' state
    uint8_t* dest; uint32_t* ridx; uint32_t* first; uint32_t* last; uint8_t* otype; int* orf; int* ors;
    // host side of the per-try results (pinned)
    uint8_t* h_dest; uint32_t* h_info; uint32_t* h_stats; long long* h_acc;

    template <class K, class... A>
    int launch(K k, dim3 grid, dim3 block, size_t smem, A... a)
    {
        k<<<grid, block, smem, st>>>(a...);
        FB_CUDA(cudaGetLastError());
        ++ctx->launches;
        return FAMSA_OK;
    }

    // column-wide scratch for a current width W and a candidate width up to Wm
    struct Cols { uint8_t* keep; int* map; uint32_t* stats; uint32_t* info; int* iR; int* iC; };
    Cols cols(uint32_t Wm) const
    {
        Layout L;
        const size_t o_keep = L.add(2 * (size_t)W), o_map = L.add(8 * (size_t)W), o_stats = L.add(4 * ((size_t)Wm + 1));
        const size_t o_info = L.add(64), o_ir = L.add(4 * (size_t)Wm), o_ic = L.add(4 * (size_t)Wm);
        char* b = R.d_cols.as<char>();
        return Cols{reinterpret_cast<uint8_t*>(b + o_keep), reinterpret_cast<int*>(b + o_map), reinterpret_cast<uint32_t*>(b + o_stats),
                    reinterpret_cast<uint32_t*>(b + o_info), reinterpret_cast<int*>(b + o_ir), reinterpret_cast<int*>(b + o_ic)};
    }
    static size_t cols_bytes(uint32_t W, uint32_t Wm) { return 2 * (size_t)W + 8 * (size_t)W + 4 * ((size_t)Wm + 1) + 64 + 8 * (size_t)Wm + 6 * 256; }

    // total score (CalculateTotalScore) of the alignment A (width w) with merged counters `counters` into acc; gap counts
    // of A into stats.  Queued only; the caller copies and waits.
    int score(const uint8_t* A, uint32_t w, const int* counters, bool with_score, uint32_t* d_stats)
    {
        unsigned long long* acc = R.d_acc.as<unsigned long long>();
        FB_CUDA(cudaMemsetAsync(acc, 0, 5 * sizeof(unsigned long long), st));
        if (with_score) {
            FB_TRY(R.d_ends.reserve((size_t)n * w * sizeof(uint32_t)));
            uint32_t* E = R.d_ends.as<uint32_t>();
            FB_TRY(launch(k_ref_run_ends, blocks(n, 128), 128, 0, A, n, w, E));
            FB_TRY(launch(k_ref_score_cols, blocks(w, kRT / 32), kRT, 0, counters, w, n, ctx->prof.d_sm.as<long long>(), acc));
            const size_t hist = ((size_t)w + 1) * sizeof(int);
            FB_TRY(launch(k_ref_score_runs, w, kRT, hist, (const uint32_t*)E, n, w, acc));
        }
        FB_TRY(launch(k_ref_gapstats, w, kRT, 0, A, n, d_stats));
        FB_CUDA(cudaMemcpyAsync(h_acc, acc, 5 * sizeof(long long), cudaMemcpyDeviceToHost, st));
        FB_CUDA(cudaMemcpyAsync(h_stats, d_stats, ((size_t)w + 1) * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        return FAMSA_OK;
    }
    // profile.cpp:1527-1531 from the accumulated terms
    int64_t total() const
    {
        const long long open = h_acc[3], topen = h_acc[4];
        return h_acc[0] + ((h_acc[1] - open) * g[1] + open * g[0] + (h_acc[2] - topen) * g[3] + topen * g[2]);
    }
};

int pinned(RefineState& R, size_t bytes)
{
    if (bytes <= R.h_pinned_cap) return FAMSA_OK;
    if (R.h_pinned) cudaFreeHost(R.h_pinned);
    R.h_pinned = nullptr; R.h_pinned_cap = 0;
    FB_CUDA(cudaMallocHost(&R.h_pinned, bytes + bytes / 2));
    R.h_pinned_cap = bytes + bytes / 2;
    return FAMSA_OK;
}

} // namespace

// The call's body.  `held`: the resident profiles the call owns at any moment (the root once the arguments are checked,
// the two sides of a try until the merge consumes them, the candidate until it is accepted or dropped); on success only
// the refined profile is left in it and it passes to the caller.
static int refine_run(famsa_ctx* ctx, uint32_t root_id, const uint8_t* rows, uint32_t n, uint32_t width, const int64_t gaps[4],
                      uint32_t n_refinements, int flags, uint32_t* refined_id, uint32_t* width_out, int64_t* total_score,
                      famsa_refine_stats* stats, std::vector<uint32_t>& held)
{
    auto let_go = [&](uint32_t id) {
        const auto it = std::find(held.begin(), held.end(), id);
        if (it != held.end()) held.erase(it);
    };
    const auto t0 = std::chrono::steady_clock::now();
    ProfState& P = ctx->prof;
    RefineState& R = ctx->refine;
    if (!P.has_scoring) { set_error("famsa_prof_refine: famsa_prof_set_scoring has not been called"); return FAMSA_E_STATE; }
    if (root_id >= P.entries.size() || !P.entries[root_id].live) {
        set_error("famsa_prof_refine: " + std::to_string(root_id) + " is not a resident profile");
        return FAMSA_E_INVALID;
    }
    if (n < 2) { set_error("famsa_prof_refine: an alignment of fewer than 2 rows cannot be split"); return FAMSA_E_INVALID; }
    const ProfEntry& root = P.entries[root_id];
    if (root.width != width || root.card != n) {
        set_error("famsa_prof_refine: the rows (" + std::to_string(n) + " x " + std::to_string(width) + ") are not those of profile " +
                  std::to_string(root_id) + " (" + std::to_string(root.card) + " x " + std::to_string(root.width) + ")");
        return FAMSA_E_INVALID;
    }
    const bool tree_rows = flags & FAMSA_REFINE_TREE_ROWS;           // the rows famsa_prof_tree_rows kept on the device
    if (tree_rows && (!P.tree_rows_valid || root_id != P.tree_rows_root || root.gen != P.tree_rows_root_gen || n != P.tree_rows_n ||
                      width != P.tree_rows_w)) {
        set_error(P.tree_rows_valid ? "famsa_prof_refine: FAMSA_REFINE_TREE_ROWS: the kept rows (" + std::to_string(P.tree_rows_n) + " x " +
                                          std::to_string(P.tree_rows_w) + ") belong to root " + std::to_string(P.tree_rows_root) +
                                          ", not to this root_id / n_rows / width"
                                    : std::string("famsa_prof_refine: FAMSA_REFINE_TREE_ROWS without rows kept by famsa_prof_tree_rows"));
        return FAMSA_E_INVALID;
    }
    // The kept rows need no check: k_tree_rows writes codes 0..23 and GAP only, and every row holds its sequence's residues,
    // which is at least one, since famsa_prof_align_tree rejects an empty leaf (prof_resolve) before it keeps a tree.
    for (uint32_t r = 0; r < n && !tree_rows; ++r) {
        bool residue = false;
        for (uint32_t c = 0; c < width; ++c) {
            const uint8_t v = rows[(size_t)r * width + c];
            if (v != kGAP && v >= kNAA) { set_error("famsa_prof_refine: row " + std::to_string(r) + " holds code " + std::to_string(v)); return FAMSA_E_INVALID; }
            residue |= v != kGAP;
        }
        if (!residue) { set_error("famsa_prof_refine: row " + std::to_string(r) + " has no residue"); return FAMSA_E_INVALID; }
    }
    if ((size_t)(width + 1) * sizeof(int) > kMaxHistBytes) { set_error("famsa_prof_refine: alignments wider than 51 199 columns are not supported"); return FAMSA_E_INVALID; }
    held.push_back(root_id);                                        // consumed from here on, also when the call fails
    const bool opt_gaps = !(flags & FAMSA_REFINE_NO_GAP_OPT), with_score = !(flags & FAMSA_REFINE_NO_TOTAL_SCORE);

    cudaStream_t st = ctx->stream;
    R.have_rows = false;
    // k_ref_score_runs' limit once per context, before its first launch: without it the default budget is 48 KiB less
    // the kernel's 384 bytes of static shared memory, which fails widths of 12 192 .. 12 287 columns (and hid the
    // failure whenever a wider call had raised the limit before)
    if (!R.configured) {
        FB_CUDA(cudaFuncSetAttribute(k_ref_score_runs, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxHistBytes));
        R.configured = true;
    }
    FB_TRY(R.d_cur.reserve((size_t)n * width));
    FB_TRY(R.d_rows.reserve((size_t)n * 24 + 1024));
    FB_TRY(R.d_acc.reserve(64));
    famsa_refine_stats S{};
    for (auto& e : R.ev)
        if (!e) FB_CUDA(cudaEventCreate(&e));
    cudaEvent_t ev0 = R.ev[0], ev1 = R.ev[1];
    FB_CUDA(cudaEventRecord(ev0, st));
    // the caller's rows (or the kept tree rows), column-major
    {
        const uint8_t* src = P.d_tree_rows.as<uint8_t>();
        if (!tree_rows) {
            FB_TRY(R.d_cand.reserve((size_t)n * width));
            FB_CUDA(cudaMemcpyAsync(R.d_cand.p, rows, (size_t)n * width, cudaMemcpyHostToDevice, st));
            src = R.d_cand.as<uint8_t>();
        }
        k_ref_transpose<<<dim3(blocks(width, 32), blocks(n, 32)), dim3(32, 8), 0, st>>>(src, R.d_cur.as<uint8_t>(), n, width);
        FB_CUDA(cudaGetLastError());
        ++ctx->launches;
    }
    Run X{ctx, R, st, n, width, {gaps[0], gaps[1], gaps[2], gaps[3]}};
    {
        Layout L;
        const size_t o_dest = L.add(n), o_ridx = L.add(4 * (size_t)n), o_first = L.add(4 * (size_t)n), o_last = L.add(4 * (size_t)n);
        const size_t o_t = L.add(n), o_rf = L.add(4 * (size_t)n), o_rs = L.add(4 * (size_t)n);
        FB_TRY(R.d_rows.reserve(L.end));
        char* b = R.d_rows.as<char>();
        X.dest = reinterpret_cast<uint8_t*>(b + o_dest); X.ridx = reinterpret_cast<uint32_t*>(b + o_ridx);
        X.first = reinterpret_cast<uint32_t*>(b + o_first); X.last = reinterpret_cast<uint32_t*>(b + o_last);
        X.otype = reinterpret_cast<uint8_t*>(b + o_t); X.orf = reinterpret_cast<int*>(b + o_rf); X.ors = reinterpret_cast<int*>(b + o_rs);
    }
    auto host_layout = [&](uint32_t wmax) -> int {
        // [acc 64][info 64][stats (wmax+1) u32][dest n]
        FB_TRY(pinned(R, 128 + 4 * ((size_t)wmax + 1) + n + 64));
        char* h = static_cast<char*>(R.h_pinned);
        X.h_acc = reinterpret_cast<long long*>(h); X.h_info = reinterpret_cast<uint32_t*>(h + 64);
        X.h_stats = reinterpret_cast<uint32_t*>(h + 128); X.h_dest = reinterpret_cast<uint8_t*>(h + 128 + 4 * ((size_t)wmax + 1));
        return FAMSA_OK;
    };

    // n_ref clamps (msa_refinement.cpp:84-92)
    size_t n_ref = n_refinements;
    if (n_ref > 2 * (size_t)n) n_ref = 2 * (size_t)n;
    if (n_ref > 0 && n_ref < 100 && n < 100) n_ref = 100;

    uint32_t cur_id = root_id;
    // prev_total_score from the root's merged counters (:114), and the gap counts of the first try
    FB_TRY(R.d_cols.reserve(Run::cols_bytes(width, width)));
    FB_TRY(host_layout(width));
    FB_TRY(X.score(R.d_cur.as<uint8_t>(), width, root.counters, with_score, X.cols(width).stats));
    FB_CUDA(cudaStreamSynchronize(st));
    int64_t prev = with_score ? X.total() : 0;
    std::vector<uint32_t> gap_stats(X.h_stats, X.h_stats + width + 1);

    std::mt19937 rnd_rfn;
    rnd_rfn.seed(5489u);
    std::vector<std::vector<uint8_t>> tried;
    std::vector<uint8_t> dest_h(n);
    std::vector<std::pair<uint32_t, uint32_t>> tmp;
    size_t i_ref, i_succ;
    for (i_ref = i_succ = 0; i_succ < n_ref && i_ref < 20 * n_ref; ++i_ref) {
        const uint32_t W = X.W;
        // RefineMostEmptyAndFullColumn (msa_refinement.cpp:21-66) on the gap counts; RefineRandom (:7-18) without a candidate
        tmp.clear();
        for (uint32_t i = 1; i <= W; ++i) {
            const uint32_t x = std::min(gap_stats[i], n - gap_stats[i]);
            if (x > 0) tmp.emplace_back(x, i);
        }
        std::sort(tmp.begin(), tmp.end());                          // stable_sort by (x, column): the pairs are distinct
        uint32_t col = 0;
        if (tmp.empty()) {
            for (uint32_t i = 0; i < n; ++i) dest_h[i] = (uint8_t)(rnd_rfn() % 2);
            const size_t ones = std::count(dest_h.begin(), dest_h.end(), 1);
            if (ones == 0 || ones == n) { const size_t id = rnd_rfn() % n; dest_h[id] = !dest_h[id]; }
        } else
            col = tmp[rnd_rfn() % tmp.size()].second;
        FB_TRY(R.d_cols.reserve(Run::cols_bytes(W, W)));
        Run::Cols C0 = X.cols(W);
        if (!col) FB_CUDA(cudaMemcpyAsync(X.dest, dest_h.data(), n, cudaMemcpyHostToDevice, st));
        FB_TRY(X.launch(k_ref_split, W, kRT, 0, (const uint8_t*)R.d_cur.as<uint8_t>(), n, W, col, X.dest, C0.keep));
        FB_TRY(X.launch(k_ref_scan, 1, kScanT, 0, (const uint8_t*)C0.keep, W, (const uint8_t*)X.dest, n, C0.map, X.ridx, C0.info));
        FB_CUDA(cudaMemcpyAsync(X.h_info, C0.info, 4 * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        if (col) FB_CUDA(cudaMemcpyAsync(X.h_dest, X.dest, n, cudaMemcpyDeviceToHost, st));
        FB_CUDA(cudaStreamSynchronize(st));                         // sync 1: the split
        if (col) std::copy(X.h_dest, X.h_dest + n, dest_h.begin());
        if (std::find(tried.begin(), tried.end(), dest_h) != tried.end()) continue;
        const uint32_t w0 = X.h_info[0], w1 = X.h_info[1], n0 = X.h_info[2], n1 = X.h_info[3];

        // the two sides: profile1 = dest 1 (child1 of the merge), profile2 = dest 0
        uint32_t ids[2], widths[2] = {w1, w0}, cards[2] = {n1, n0};
        FB_TRY(prof_new(ctx, 2, widths, cards, ids));
        held.push_back(ids[0]); held.push_back(ids[1]);
        FB_TRY(R.d_side.reserve((size_t)n1 * w1 + (size_t)n0 * w0 + 256));
        Sides SD;
        SD.rows[1] = R.d_side.as<uint8_t>(); SD.rows[0] = SD.rows[1] + (size_t)n1 * w1;
        SD.n[0] = n0; SD.n[1] = n1; SD.w[0] = w0; SD.w[1] = w1;
        SideTables T{{P.entries[ids[1]].scores, P.entries[ids[0]].scores}, {P.entries[ids[1]].counters, P.entries[ids[0]].counters}};
        FB_TRY(X.launch(k_ref_condense, blocks((size_t)n * W, kRT), kRT, 0, (const uint8_t*)R.d_cur.as<uint8_t>(), n, W,
                        (const uint8_t*)X.dest, (const int*)C0.map, (const uint32_t*)X.ridx, SD));
        FB_TRY(gapped_tables(ctx, st, SD, 2, X.first, X.last, T, gaps));
        if (opt_gaps) FB_TRY(X.launch(k_ref_optimize, 2, kOptT, 0, SD, X.otype, X.orf, X.ors));

        // Align + ConstructProfile through the merge path of famsa_prof_merge_batch; the sides are consumed
        const famsa_prof_merge m{ids[0], ids[1]};                  // ids[0]: profile1 (dest 1), ids[1]: profile2
        famsa_dp_result res{};
        std::vector<uint8_t> path((size_t)w0 + w1);
        uint32_t merged = 0;
        FB_TRY(prof_merge_batch(ctx, &m, 1, gaps, &merged, &res, path.data(), path.size()));          // sync 2
        let_go(ids[0]); let_go(ids[1]);                             // consumed by the merge
        held.push_back(merged);
        S.cells += (uint64_t)w0 * w1;
        const uint32_t Wm = res.path_len;
        if ((size_t)(Wm + 1) * sizeof(int) > kMaxHistBytes) {
            set_error("famsa_prof_refine: a realignment is " + std::to_string(Wm) + " columns wide; more than 51 199 are not supported");
            return FAMSA_E_INVALID;
        }
        const int row_side = res.swapped ? 0 : 1;

        // the candidate's rows, equality, total score and gap counts
        FB_TRY(R.d_cand.reserve((size_t)n * Wm));
        FB_TRY(R.d_path.reserve(Wm));
        FB_TRY(R.d_cols.reserve(Run::cols_bytes(W, std::max(W, Wm))));
        FB_TRY(host_layout(std::max(W, Wm)));
        Run::Cols C1 = X.cols(std::max(W, Wm));
        FB_CUDA(cudaMemcpyAsync(R.d_path.p, path.data() + res.path_offset, Wm, cudaMemcpyHostToDevice, st));
        FB_CUDA(cudaMemsetAsync(C1.info + 4, 0, sizeof(uint32_t), st));
        FB_TRY(X.launch(k_ref_path_index, 1, kScanT, 0, (const uint8_t*)R.d_path.as<uint8_t>(), Wm, C1.iR, C1.iC));
        FB_TRY(X.launch(k_ref_rebuild, blocks((size_t)n * Wm, kRT), kRT, 0, (const uint8_t*)R.d_cur.as<uint8_t>(), R.d_cand.as<uint8_t>(),
                        n, Wm, row_side, SD, (const uint8_t*)X.dest, (const uint32_t*)X.ridx, (const int*)C1.iR, (const int*)C1.iC,
                        (int)(Wm == W), C1.info));
        FB_CUDA(cudaMemcpyAsync(X.h_info + 4, C1.info + 4, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        FB_TRY(X.score(R.d_cand.as<uint8_t>(), Wm, P.entries[merged].counters, with_score, C1.stats));
        FB_CUDA(cudaStreamSynchronize(st));                         // sync 3: equality, score, gap counts
        const bool identical = Wm == W && !X.h_info[4];
        bool accept = false;
        if (!identical) {
            const int64_t tot = with_score ? X.total() : 0;
            if (tot >= prev) { prev = tot; accept = true; }
        } else
            ++S.n_identical;
        if (accept) {
            std::swap(R.d_cur, R.d_cand);
            X.W = Wm;
            FB_TRY(prof_drop(ctx, &cur_id, 1));
            let_go(cur_id);
            cur_id = merged;
            gap_stats.assign(X.h_stats, X.h_stats + Wm + 1);
            ++S.n_accepted;
            tried.clear();
        } else {
            FB_TRY(prof_drop(ctx, &merged, 1));
            let_go(merged);
        }
        tried.push_back(dest_h);
        ++i_succ;
    }
    FB_CUDA(cudaEventRecord(ev1, st));
    FB_CUDA(cudaEventSynchronize(ev1));
    float dev_ms = 0.f;
    FB_CUDA(cudaEventElapsedTime(&dev_ms, ev0, ev1));
    R.n = n; R.width = X.W; R.have_rows = true;
    *refined_id = cur_id;
    *width_out = X.W;
    *total_score = prev;
    S.n_tries = (uint32_t)i_ref;
    S.n_realigned = (uint32_t)i_succ;
    S.device_ms = dev_ms;
    S.wall_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
    if (stats) *stats = S;
    held.clear();                                                   // the refined profile is the caller's
    return FAMSA_OK;
}

int prof_refine(famsa_ctx* ctx, uint32_t root_id, const uint8_t* rows, uint32_t n, uint32_t width, const int64_t gaps[4],
                uint32_t n_refinements, int flags, uint32_t* refined_id, uint32_t* width_out, int64_t* total_score,
                famsa_refine_stats* stats)
{
    std::vector<uint32_t> held;
    const int rc = refine_run(ctx, root_id, rows, n, width, gaps, n_refinements, flags, refined_id, width_out, total_score, stats, held);
    if (rc != FAMSA_OK) {
        // nothing the call owned stays resident; the error message of the failure is kept
        cudaStreamSynchronize(ctx->stream);
        ProfState& P = ctx->prof;
        for (uint32_t id : held)
            if (id < P.entries.size() && P.entries[id].live) {
                const std::string msg = get_error();
                prof_drop(ctx, &id, 1);
                set_error(msg);
            }
        ctx->refine.have_rows = false;
    }
    return rc;
}

int prof_refined_rows(famsa_ctx* ctx, uint8_t* rows, uint64_t cap)
{
    RefineState& R = ctx->refine;
    if (!R.have_rows) { set_error("famsa_prof_refined_rows: no famsa_prof_refine has completed"); return FAMSA_E_STATE; }
    const size_t bytes = (size_t)R.n * R.width;
    if (cap < bytes) { set_error("famsa_prof_refined_rows: " + std::to_string(bytes) + " bytes needed, " + std::to_string(cap) + " given"); return FAMSA_E_INVALID; }
    FB_TRY(R.d_cand.reserve(bytes));
    k_ref_transpose<<<dim3(blocks(R.n, 32), blocks(R.width, 32)), dim3(32, 8), 0, ctx->stream>>>(R.d_cur.as<uint8_t>(), R.d_cand.as<uint8_t>(), R.width, R.n);
    FB_CUDA(cudaGetLastError());
    ++ctx->launches;
    FB_CUDA(cudaMemcpyAsync(rows, R.d_cand.p, bytes, cudaMemcpyDeviceToHost, ctx->stream));
    FB_CUDA(cudaStreamSynchronize(ctx->stream));
    return FAMSA_OK;
}

// famsa_prof_put_rows: the rows go up into stream-ordered scratch of the call's own (refine's state stays as it is), are
// turned column-major and gapped_tables builds the new entry's tables.
static int put_rows_run(famsa_ctx* ctx, const uint8_t* rows, uint32_t n, uint32_t width, const int64_t gaps[4], uint32_t id)
{
    cudaStream_t st = ctx->stream;
    Layout L;
    const size_t cells = (size_t)n * width;
    const size_t o_raw = L.add(cells), o_cm = L.add(cells), o_first = L.add(4 * (size_t)n), o_last = L.add(4 * (size_t)n);
    char* blob = nullptr;
    const cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&blob), L.end, st);
    if (e != cudaSuccess) {
        cudaGetLastError();
        set_error("famsa_prof_put_rows: cudaMallocAsync(" + std::to_string(L.end) + ") failed: " + cudaGetErrorString(e));
        return FAMSA_E_NOMEM;
    }
    uint8_t* raw = reinterpret_cast<uint8_t*>(blob + o_raw);
    uint8_t* cm = reinterpret_cast<uint8_t*>(blob + o_cm);
    auto body = [&]() -> int {
        FB_CUDA(cudaMemcpyAsync(raw, rows, cells, cudaMemcpyHostToDevice, st));
        k_ref_transpose<<<dim3(blocks(width, 32), blocks(n, 32)), dim3(32, 8), 0, st>>>(raw, cm, n, width);
        FB_CUDA(cudaGetLastError());
        ++ctx->launches;
        Sides S{};
        S.rows[0] = cm; S.n[0] = n; S.w[0] = width;
        const ProfEntry& E = ctx->prof.entries[id];
        const SideTables T{{E.scores, nullptr}, {E.counters, nullptr}};
        return gapped_tables(ctx, st, S, 1, reinterpret_cast<uint32_t*>(blob + o_first), reinterpret_cast<uint32_t*>(blob + o_last), T, gaps);
    };
    int rc = body();
    const cudaError_t f = cudaFreeAsync(blob, st);
    if (rc == FAMSA_OK && f != cudaSuccess) { set_error(std::string("famsa_prof_put_rows: cudaFreeAsync failed: ") + cudaGetErrorString(f)); rc = FAMSA_E_CUDA; }
    return rc;
}

int prof_put_rows(famsa_ctx* ctx, const uint8_t* rows, uint32_t n, uint32_t width, const int64_t gaps[4], int flags, uint32_t* id_out)
{
    if (!ctx->prof.has_scoring) { set_error("famsa_prof_put_rows: famsa_prof_set_scoring has not been called"); return FAMSA_E_STATE; }
    const bool from_text = flags & FAMSA_PUT_ROWS_FROM_TEXT;
    if (!n || width < (from_text ? 2u : 1u)) {
        set_error("famsa_prof_put_rows: an alignment of " + std::to_string(n) + " x " + std::to_string(width) + " is empty");
        return FAMSA_E_INVALID;
    }
    const uint32_t kept = from_text ? width - 1 : width;          // the columns of the profile
    for (uint32_t r = 0; r < n; ++r) {
        bool residue = false, gap = false;
        for (uint32_t c = 0; c < width; ++c) {
            const uint8_t v = rows[(size_t)r * width + c];
            if (v != kGAP && v >= kNAA) { set_error("famsa_prof_put_rows: row " + std::to_string(r) + " holds code " + std::to_string(v)); return FAMSA_E_INVALID; }
            residue |= v != kGAP;
            gap |= v == kGAP && c < kept;
        }
        if (!residue) { set_error("famsa_prof_put_rows: row " + std::to_string(r) + " has no residue"); return FAMSA_E_INVALID; }
        // a one-row profile is aligned as a sequence whose residues are its columns (AlignSeqSeq / AlignSeqProf)
        if (n == 1 && gap) { set_error("famsa_prof_put_rows: a one-row alignment cannot hold a gap"); return FAMSA_E_INVALID; }
    }
    uint32_t id;
    FB_TRY(prof_new(ctx, 1, &width, &n, &id));
    const int rc = put_rows_run(ctx, rows, n, width, gaps, id);
    if (rc != FAMSA_OK) {
        // the new entry does not stay resident; the error message of the failure is kept
        const std::string msg = get_error();
        cudaStreamSynchronize(ctx->stream);
        prof_drop(ctx, &id, 1);
        set_error(msg);
        return rc;
    }
    // FAMSA_PUT_ROWS_FROM_TEXT: the reference's profile is these tables without their last column (see the header).  Its
    // counters still hold that column, with the residues alone (no terminal gap reaches past the width), and ProfProf's
    // orientation counts it (DpJobExt::x1 / x2).
    if (from_text) {
        ProfEntry& E = ctx->prof.entries[id];
        const cudaError_t z = cudaMemsetAsync(E.counters + (size_t)width * kRows + kNAA, 0, (kRows - kNAA) * sizeof(int), ctx->stream);
        if (z != cudaSuccess) {
            set_error(std::string("famsa_prof_put_rows: cudaMemsetAsync failed: ") + cudaGetErrorString(z));
            cudaStreamSynchronize(ctx->stream);
            prof_drop(ctx, &id, 1);
            return FAMSA_E_CUDA;
        }
        --E.width;
        E.text_col = true;
    }
    *id_out = id;
    return FAMSA_OK;
}

void refine_release(famsa_ctx* ctx)
{
    RefineState& R = ctx->refine;
    if (R.h_pinned) cudaFreeHost(R.h_pinned);
    R.h_pinned = nullptr; R.h_pinned_cap = 0;
    for (auto& e : R.ev)
        if (e) { cudaEventDestroy(e); e = nullptr; }
}

} // namespace fb
