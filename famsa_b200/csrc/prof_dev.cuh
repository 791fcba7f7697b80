// Device code of the resident-profile kernels (leaf materialisation, ConstructProfile's table building), shared by
// prof.cu's batch kernels and the fused one-block-per-merge kernel in dp.cu.  See prof.cu for the reasoning.
#pragma once
#include <cstdint>

#include "../../include/famsa_b200.h"
#include "dp_dev.h"

namespace fb {

constexpr int kRows = 32;                 // NO_SYMBOLS, defs.h:69
constexpr int kGO = 25, kGE = 26, kTE = 27, kTO = 28, kGAP = 30, kNAA = 24;   // defs.h:62-74
constexpr int kConThreads = 256, kConTile = 64;
constexpr size_t kColBytes = kRows * (sizeof(long long) + sizeof(int));        // 384 B per profile column

// The four gap lanes of a profile column's scores: `tot` members times each gap cost (CalculateScores, profile.cpp:171-174
// for column 0 with tot = card, :212-215 for a column with tot residues); the other lanes get 0.
__device__ __forceinline__ long long gap_lanes(int lane, long long tot, long long go, long long ge, long long to, long long te)
{
    return lane == kGO ? go * tot : lane == kGE ? ge * tot : lane == kTO ? to * tot : lane == kTE ? te * tot : 0;
}

struct LeafDesc {
    uint32_t seq;
    long long* scores;
    int* counters;
};

// One block per leaf: CalculateCounters + CalculateScores for a profile of one ungapped sequence
// (profile.cpp:101-217): column c >= 1 holds counter 1 at its residue, the residue's substitution row in
// scores[0..23] and the four gap costs; column 0 holds card(=1) x gap costs.
__device__ __forceinline__ void leaf_body(const LeafDesc L, const int8_t* __restrict__ codes,
                                          const uint64_t* __restrict__ off, const uint32_t* __restrict__ len,
                                          const long long* __restrict__ sm, long long go, long long ge,
                                          long long to, long long te, int warp_first = 0)
{
    // the block's warps warp_first .. take part (all of them by default)
    const uint32_t n = len[L.seq];
    const int8_t* s = codes + off[L.seq];
    const int lane = threadIdx.x & 31, warp = (int)(threadIdx.x >> 5) - warp_first, nwarps = (int)(blockDim.x >> 5) - warp_first;
    if (warp < 0) return;
    const long long gapv = gap_lanes(lane, 1, go, ge, to, te);
    for (uint32_t c = warp; c <= n; c += nwarps) {
        long long sc = gapv;
        int cn = 0;
        if (c) {
            int sym = s[c - 1];
            if (sym < 0 || sym >= kNAA) sym = 22;                      // anything outside the alphabet counts as UNKNOWN
            cn = lane == sym;
            if (lane < kNAA) sc = sm[sym * kNAA + lane];
        }
        L.scores[(size_t)c * kRows + lane] = sc;
        L.counters[(size_t)c * kRows + lane] = cn;
    }
}

// One merge of a batch for k_prof_construct.  Everything that depends on the outcome of the DP -- which child is the row
// profile, the real widths, the merged width -- is read on the device from the DP's own records, so the kernel can be
// queued right behind the fill without the host looking at the results first.
struct ConJobDev {
    long long* os; int* oc;                // merged profile, sized for the upper bound w1 + w2
    uint32_t job;                          // index into meta / results
    uint32_t tile0;                        // first block of this merge (tiles counted with the upper bound)
};

// One merge of a batch for the fused one-block-per-merge kernel (dp.cu): leaf children to materialise (seq = 0xffffffff:
// not a leaf) and where the merged tables go.
struct FusedJob {
    LeafDesc leaf[2];
    ConJobDev con;
};
struct FusedParams {
    const FusedJob* jobs;
    const uint32_t* level_start;                                    // n_levels + 1 job indices: the launch runs these dependency levels
    uint32_t n_levels;                                              // one after the other, a grid barrier in between
    const int8_t* codes; const uint64_t* off; const uint32_t* len;   // the uploaded sequences (caller order)
    const long long* sm;                                            // 24 x 24 score matrix
    int timing;                                                     // development aid: accumulate per-phase times
    // completion without a CUDA event (an event record between two short kernels costs more than the kernels' launch gap):
    // the last block to finish publishes `done_seq` in mapped host memory, after everybody's results have been fenced
    unsigned* block_counter;                                        // device, two words, zero between launches: [0] finished blocks, [1] barrier arrivals
    volatile unsigned long long* h_done;                            // mapped host memory, or NULL
    unsigned long long done_seq;
};

struct GapSplit { int o, e, to, te; };

// Column of gaps inserted into a child (counters `c`, width `w`, `card` members) after its column `src`.
// col / nxt: this lane's counters of columns src and src+1 (nxt = 0 past the end).
__device__ __forceinline__ GapSplit gap_split(int col, int nxt, uint32_t src, uint32_t w, int card, bool starts)
{
    const int go_s = __shfl_sync(0xffffffffu, col, kGO), ge_s = __shfl_sync(0xffffffffu, col, kGE);
    const int to_s = __shfl_sync(0xffffffffu, col, kTO), te_s = __shfl_sync(0xffffffffu, col, kTE);
    const int to_n = __shfl_sync(0xffffffffu, nxt, kTO);
    GapSplit g{0, 0, 0, 0};
    if (starts) {
        if (src == 0) g.to = card;
        else if (src >= w) { g.te = to_s + te_s; g.to = card - g.te; }
        else { g.to = to_n; g.te = to_s + te_s; g.e = go_s + ge_s; g.o = card - g.e - g.to - g.te; }
    } else {
        if (src == 0 || src == w) g.te = card;
        else { g.te = to_n + to_s + te_s; g.e = card - g.te; }
    }
    return g;
}

struct ConJob {                            // resolved on the device at the top of k_prof_construct
    const long long* sr; const int* cr;    // row child (ConstructProfile's profile1)
    const long long* sc; const int* cc;    // column child (profile2)
    long long* os; int* oc;                // merged profile
    const uint8_t* path;
    uint32_t wr, wc, cardr, cardc, W, tile0;
};

// the merge as k_prof_construct needs it, from the DP's own records
__device__ __forceinline__ bool con_resolve(const ConJobDev D, const DpMeta& M, const famsa_dp_result& r, const uint8_t* path_base, ConJob& J)
{
    if (M.bad || r.variant == 0xFF) return false;
    J.sr = M.SR; J.cr = M.CR; J.sc = M.SC; J.cc = M.CC; J.os = D.os; J.oc = D.oc;
    J.path = path_base + r.path_offset;
    J.wr = M.WR; J.wc = M.WC; J.cardr = (uint32_t)M.nR; J.cardc = (uint32_t)M.nC; J.W = r.path_len; J.tile0 = D.tile0;
    return true;
}

struct ConShared {
    uint32_t s_cnt[2][kConThreads / 32];
    uint8_t s_dir[kConTile + 4];                                    // s_dir[t] = path[k0 + t - 2]  (dir of column k0+t-1)
    uint32_t s_nh[kConTile], s_nv[kConTile];
};

// One tile of kConTile merged columns (k0 = its first column), by all threads of the block (a multiple of 32, <= kConThreads).
__device__ __forceinline__ void construct_tile(const ConJob& J, uint32_t k0, ConShared& S, long long go, long long ge, long long to, long long te)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nthr = blockDim.x, nwarps = blockDim.x >> 5;
    uint32_t (&s_cnt)[2][kConThreads / 32] = S.s_cnt;
    uint8_t (&s_dir)[kConTile + 4] = S.s_dir;
    uint32_t (&s_nh)[kConTile] = S.s_nh;
    uint32_t (&s_nv)[kConTile] = S.s_nv;

    // H / V counts over the path entries of the columns before the tile: path[0 .. k0-2]
    const uint32_t before = k0 ? k0 - 1 : 0;
    uint32_t nh = 0, nv = 0;
    for (uint32_t p = threadIdx.x; p < before; p += nthr) {
        const uint8_t d = J.path[p];
        nh += d == 1; nv += d == 2;
    }
    for (int o = 16; o; o >>= 1) { nh += __shfl_xor_sync(0xffffffffu, nh, o); nv += __shfl_xor_sync(0xffffffffu, nv, o); }
    if (lane == 0) { s_cnt[0][warp] = nh; s_cnt[1][warp] = nv; }
    for (uint32_t x = threadIdx.x; x <= (uint32_t)kConTile; x += nthr) {
        const long long p = (long long)k0 + x - 2;
        s_dir[x] = (p >= 0 && p < (long long)J.W) ? J.path[p] : 0;                // "previous" of the first column is D
    }
    __syncthreads();
    nh = nv = 0;
    for (int w = 0; w < nwarps; ++w) { nh += s_cnt[0][w]; nv += s_cnt[1][w]; }
    for (uint32_t x = threadIdx.x; x < (uint32_t)kConTile; x += nthr) {
        // inclusive counts up to and including the direction of column k0 + x
        uint32_t a = nh, b = nv;
        for (uint32_t u = (k0 ? 0 : 1); u <= x; ++u) { a += s_dir[u + 1] == 1; b += s_dir[u + 1] == 2; }
        s_nh[x] = a; s_nv[x] = b;
    }
    __syncthreads();

    const long long tr_open = ge - go, tr_term = te - to;
    // Every warp builds the columns t = warp, warp + nwarps, ... of the tile, kBatch of them at a time: first ALL the child
    // values those columns need are requested (independent loads, nothing waits), then the columns are finished -- the
    // block is small, so a column at a time would pay the memory latency once per column.
    constexpr int kBatch = 4;
    struct ColIn { int cr, cc, gcol, gnxt; long long sr, sc; };
    for (int t0 = warp; t0 < kConTile; t0 += nwarps * kBatch) {
        ColIn in[kBatch];
#pragma unroll
        for (int u = 0; u < kBatch; ++u) {
            const int t = t0 + u * nwarps;
            const uint32_t k = k0 + t;
            in[u] = ColIn{0, 0, 0, 0, 0, 0};
            if (t >= kConTile || k > J.W || k == 0) continue;
            const int d = s_dir[t + 1];
            const uint32_t i = k - s_nh[t], j = k - s_nv[t];        // child columns consumed after this step
            if (d != 1) { in[u].cr = J.cr[(size_t)i * kRows + lane]; in[u].sr = J.sr[(size_t)i * kRows + lane]; }
            if (d != 2) { in[u].cc = J.cc[(size_t)j * kRows + lane]; in[u].sc = J.sc[(size_t)j * kRows + lane]; }
            if (d != 0) {
                const bool isH = d == 1;
                const int* cg = isH ? J.cr : J.cc;
                const uint32_t src = isH ? i : j, w = isH ? J.wr : J.wc;
                in[u].gcol = cg[(size_t)src * kRows + lane];
                in[u].gnxt = src < w ? cg[(size_t)(src + 1) * kRows + lane] : 0;
            }
        }
#pragma unroll
        for (int u = 0; u < kBatch; ++u) {
            const int t = t0 + u * nwarps;
            const uint32_t k = k0 + t;
            if (t >= kConTile || k > J.W) continue;
            long long os = 0;
            int oc = 0;
            if (k == 0) {                                               // profile.cpp:998-1001
                os = gap_lanes(lane, (long long)J.cardr + J.cardc, go, ge, to, te);
            } else {
                const int d = s_dir[t + 1], prev = s_dir[t];
                const uint32_t i = k - s_nh[t], j = k - s_nv[t];
                if (d != 1) {                                           // D or V: the row child's column i
                    const int c = in[u].cr;
                    long long sv = in[u].sr;
                    int tt = __shfl_sync(0xffffffffu, c, kTO), tg = __shfl_sync(0xffffffffu, c, kGO);
                    if (prev != 1) tt = tg = 0;
                    if (i == 1) tg = 0;                                 // the run sat before the first column: terminal only
                    oc += c + (lane == kGE ? tg : lane == kGO ? -tg : lane == kTE ? tt : lane == kTO ? -tt : 0);
                    if (lane < kNAA) sv += tg * tr_open + tt * tr_term;
                    os += sv;
                }
                if (d != 2) {                                           // D or H: the column child's column j
                    const int c = in[u].cc;
                    long long sv = in[u].sc;
                    int tt = __shfl_sync(0xffffffffu, c, kTO), tg = __shfl_sync(0xffffffffu, c, kGO);
                    if (prev != 2) tt = tg = 0;
                    if (j == 1) tg = 0;
                    oc += c + (lane == kGE ? tg : lane == kGO ? -tg : lane == kTE ? tt : lane == kTO ? -tt : 0);
                    if (lane < kNAA) sv += tg * tr_open + tt * tr_term;
                    os += sv;
                }
                if (d != 0) {                                           // a column of gaps in the row (H) / column (V) child
                    const bool isH = d == 1;
                    const uint32_t src = isH ? i : j, w = isH ? J.wr : J.wc;
                    const int card = (int)(isH ? J.cardr : J.cardc);
                    const GapSplit g = gap_split(in[u].gcol, in[u].gnxt, src, w, card, prev != d);
                    oc += lane == kGO ? g.o : lane == kGE ? g.e : lane == kTO ? g.to : lane == kTE ? g.te : lane == kGAP ? card : 0;
                    if (lane < kNAA) os += g.o * go + g.e * ge + g.to * to + g.te * te;
                }
            }
            J.os[(size_t)k * kRows + lane] = os;
            J.oc[(size_t)k * kRows + lane] = oc;
        }
    }
    __syncthreads();                                                // the shared arrays are reused by the next tile
}

} // namespace fb
