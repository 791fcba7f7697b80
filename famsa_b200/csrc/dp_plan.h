// Launch policy of the profile DP (dp.cu): how a batch of merges is cut into sub-batches, which fill kernel runs each
// merge, in which order and on which stream.  Plain C++ without CUDA headers: the policy compiles and can be checked on
// its own (tests/cpp/dp_plan_check.cpp).
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <numeric>
#include <string>
#include <vector>

namespace fb {

constexpr uint32_t kDpTeamMinWidth = 96;  // min(w1, w2) above which a merge gets a team
constexpr uint32_t kDpClusterMinWidth = 1024;   // min(w1, w2) above which a merge gets a whole cluster
constexpr int kTThreads = 256, kTCellsPerThread = 4;

// rows of the DP matrix as far as the host can tell (the orientation of ProfProf merges is decided on the device)
inline uint32_t host_rows(uint32_t w1, uint32_t card1, uint32_t w2, uint32_t card2)
{
    return card1 == 1 ? w1 : (card2 == 1 ? w2 : std::min(w1, w2));
}

// bytes of a merge's path slot; align16: 16-byte slots, because the traceback then stores paths to the host in uint4 units
inline unsigned long long path_slot(uint32_t w1, uint32_t w2, bool align16)
{
    const unsigned long long w = (unsigned long long)w1 + w2;
    return align16 ? (w + 15) / 16 * 16 : w;
}

// Development knobs, read from the environment once per call.
struct DpKnobs {
    unsigned long long max_cells = 1ull << 32;  // FAMSA_DP_MAX_CELLS: matrix cells per sub-batch
    uint32_t team_min = kDpTeamMinWidth;        // FAMSA_DP_TEAM_MIN
    int team_warps = 0;                         // FAMSA_DP_TEAM_WARPS: forced team width (0: by the number of merges)
    uint32_t cluster_min = kDpClusterMinWidth;  // FAMSA_DP_CLUSTER_MIN
    uint32_t max_cluster = 0xffffffffu;         // FAMSA_DP_MAX_CLUSTER: cap on the latency-mode cluster size
    int latency_mode = -1;                      // FAMSA_DP_LATENCY_MODE: 0 / 1 forces the regime (-1: by the batch's demand)
    bool duo = true;                            // FAMSA_DP_DUO: 0 runs clustered ProfProf merges one warp per stripe
    int compact = 1;                            // FAMSA_DP_COMPACT: 0 never, 1 from two merges per SM on, 2 always
    bool debug = false;                         // FAMSA_DP_DEBUG: one `[dp] batch of ...` line per launch class on stderr
};

inline DpKnobs dp_knobs()
{
    DpKnobs K;
    if (const char* e = getenv("FAMSA_DP_MAX_CELLS")) K.max_cells = strtoull(e, nullptr, 10);
    if (const char* e = getenv("FAMSA_DP_TEAM_MIN")) K.team_min = (uint32_t)atoi(e);
    if (const char* e = getenv("FAMSA_DP_TEAM_WARPS")) K.team_warps = atoi(e);
    if (const char* e = getenv("FAMSA_DP_CLUSTER_MIN")) K.cluster_min = (uint32_t)atoi(e);
    if (const char* e = getenv("FAMSA_DP_MAX_CLUSTER")) K.max_cluster = (uint32_t)atoi(e);
    if (const char* e = getenv("FAMSA_DP_LATENCY_MODE")) K.latency_mode = atoi(e) != 0;
    if (const char* e = getenv("FAMSA_DP_DUO")) K.duo = atoi(e) != 0;
    if (const char* e = getenv("FAMSA_DP_COMPACT")) K.compact = atoi(e);
    K.debug = getenv("FAMSA_DP_DEBUG") != nullptr;
    return K;
}

// What the device allows (probed once per context) and the shapes the fill kernels are compiled for (dp.cu).
struct DpCaps {
    uint32_t sm_count;
    uint32_t cl_cap;       // largest cluster of 4-warp k_dp_fill blocks (8 or 16)
    uint32_t duo_cap;      // largest cluster of k_dp_fill_duo blocks (1 .. 16)
    int team_warps;        // kDpTeamWarps: warps of the largest team, and of a throughput-cluster block
    uint32_t cluster;      // kDpCluster: blocks of a throughput cluster
};

// One merge as the host sees it: layout widths (upper bounds when a child is still queued), members, and the bytes of
// its scratch and skewed direction matrix.  dp_cut() fills in the offsets inside the merge's sub-batch.
struct DpGeom {
    uint32_t w1, card1, w2, card2;
    unsigned long long scratch, skew;
    unsigned long long scratch_off = 0, t_off = 0;
};

inline uint32_t host_stripes(const DpGeom& g) { return (host_rows(g.w1, g.card1, g.w2, g.card2) + 31) / 32; }

struct DpSub {
    uint32_t j0 = 0, j1 = 0;                     // jobs j0 .. j1-1
    unsigned long long scratch = 0, skew = 0;    // bytes of scratch and skewed directions of the sub-batch
    std::vector<unsigned long long> tblock{0};   // k_dp_unskew: first block of each job (j1 - j0 + 1 entries)
};

// Sub-batches of consecutive jobs bound the device scratch (direction bytes are 1 byte per cell): at most
// max_cells matrix cells each, unless a single job has more.  Returns false when a sub-batch needs more unskew
// blocks than one launch has.
inline bool dp_cut(unsigned long long max_cells, std::vector<DpGeom>& jobs, std::vector<DpSub>& subs)
{
    const uint32_t n = (uint32_t)jobs.size();
    for (uint32_t j0 = 0; j0 < n;) {
        DpSub sb;
        sb.j0 = j0;
        uint32_t j1 = j0;
        unsigned long long mat_sum = 0;
        while (j1 < n) {
            DpGeom& g = jobs[j1];
            const unsigned long long mat = ((unsigned long long)g.w1 + 1) * (g.w2 + 1);
            if (j1 > j0 && mat_sum + mat > max_cells) break;
            g.scratch_off = sb.scratch;
            g.t_off = sb.skew;                                  // skewed directions are per sub-batch
            sb.scratch += g.scratch;
            sb.skew += g.skew;
            mat_sum += mat;
            sb.tblock.push_back(sb.tblock.back() + (mat + kTThreads * kTCellsPerThread - 1) / (kTThreads * kTCellsPerThread));
            ++j1;
        }
        sb.j1 = j1;
        if (sb.tblock.back() > 0x7fffffffull) return false;
        subs.push_back(std::move(sb));
        j0 = j1;
    }
    return true;
}

enum class DpKernel { Fill, Compact, Duo };   // k_dp_fill<NW, cluster > 1>, k_dp_fill_compact<NW>, k_dp_fill_duo

// One fill launch: the merges order[q0 .. q1) of a sub-batch.
struct DpLaunch {
    int cls;            // launch class (the sort key): 0 one warp per merge, 1 a team, 2 a throughput cluster,
                        // 10 + CL a latency cluster of CL blocks, 100 + CL producer / consumer pairs in CL blocks
    DpKernel kernel;
    int nw;             // warps per block (Fill with NW = 1: one warp per merge, several merges per block)
    uint32_t cluster;   // blocks per merge
    bool wide_only;     // only the merges whose T needs 8 bytes (the k_dp_fill_compact launch before it did the others)
    uint32_t q0, q1;
    uint32_t slot;      // 0: the caller's stream, 1 + a: auxiliary stream a
};

struct DpSubPlan {
    std::vector<uint32_t> order;     // launch slot -> job index
    std::vector<DpLaunch> launches;
    uint32_t n_classes = 0;
    unsigned long long demand = 0;   // stripes the merges can use (latency mode while they fit one per SM sub-partition)
    uint32_t cl_cap = 0;
    bool small_batch = false;        // latency mode
};

// Two regimes.  A batch large enough to fill the device with one warp per stripe-pipeline is THROUGHPUT-bound: wide
// merges get a block (2, 4 or 8 warps by how many there are), the very widest a cluster of 8 x 8 warps, the rest run
// one warp per merge.  A small batch (the chain-like parts and the top of a guide tree, where a level is one or a few
// merges) is LATENCY-bound: every merge with more than one stripe gets a cluster of 4-warp blocks, one stripe per SM
// sub-partition, as many blocks as its stripes can use (up to 16).
inline DpSubPlan dp_plan(const DpKnobs& K, const DpCaps& C, const std::vector<DpGeom>& jobs, const DpSub& sb)
{
    DpSubPlan S;
    const uint32_t j0 = sb.j0, m = sb.j1 - sb.j0, sms = C.sm_count;
    S.cl_cap = std::max(1u, std::min(C.cl_cap, K.max_cluster));
    uint32_t n_teamable = 0;
    for (uint32_t a = j0; a < sb.j1; ++a) {
        S.demand += std::min(host_stripes(jobs[a]), 4u * S.cl_cap);
        n_teamable += std::min(jobs[a].w1, jobs[a].w2) > K.team_min;
    }
    S.small_batch = K.latency_mode >= 0 ? K.latency_mode != 0 : S.demand <= 4ull * sms;
    // throughput mode with only a handful of block-sized merges: give every merge with more than 8 stripes a cluster
    uint32_t cl_min = K.cluster_min;
    if (n_teamable * C.cluster <= 2u * sms) cl_min = std::min(K.cluster_min, std::max(K.team_min, 256u));
    const uint32_t duo_cap = K.duo ? C.duo_cap : 1;
    std::vector<int> cls(m);
    for (uint32_t a = 0; a < m; ++a) {
        const DpGeom& g = jobs[j0 + a];
        const uint32_t w = std::min(g.w1, g.w2);
        if (S.small_batch) {
            const uint32_t stripes = host_stripes(g);
            if (stripes < 2) { cls[a] = 0; continue; }
            const uint32_t want = (stripes + 3) / 4;              // blocks of 4 warps
            uint32_t cl = 1;
            while (cl < want && cl < S.cl_cap) cl *= 2;
            // ProfProf merges wide enough for a cluster: producer / consumer pairs (k_dp_fill_duo)
            cls[a] = K.duo && cl >= 2 && g.card1 > 1 && g.card2 > 1 ? 100 + (int)std::min(cl, duo_cap) : 10 + (int)cl;
        } else
            cls[a] = w > cl_min ? 2 : (w > K.team_min ? 1 : 0);
    }
    auto cls_of = [&](uint32_t job) { return cls[job - j0]; };
    S.order.resize(m);
    std::iota(S.order.begin(), S.order.end(), j0);
    std::stable_sort(S.order.begin(), S.order.end(), [&](uint32_t a, uint32_t b) {   // larger class first, then larger merge
        if (cls_of(a) != cls_of(b)) return cls_of(a) > cls_of(b);
        return (unsigned long long)jobs[a].w1 * jobs[a].w2 > (unsigned long long)jobs[b].w1 * jobs[b].w2;
    });

    // one launch per run of equal class in `order` (two for the compact kernel); different classes run side by side
    // (fork after prep, join before the traceback) so that a level pays for its slowest merge once, not once per shape
    for (uint32_t q0 = 0; q0 < m; ++S.n_classes) {
        const int c = cls_of(S.order[q0]);
        uint32_t q1 = q0;
        while (q1 < m && cls_of(S.order[q1]) == c) ++q1;
        const uint32_t n = q1 - q0;
        // class 0 (first in launch order is the heaviest) stays on the main stream, the others go to the aux streams
        const uint32_t slot = S.n_classes == 0 ? 0 : 1 + (S.n_classes - 1) % 4;
        if (c == 0) S.launches.push_back({c, DpKernel::Fill, 1, 1, false, q0, q1, slot});
        else if (c >= 100) S.launches.push_back({c, DpKernel::Duo, 8, (uint32_t)c - 100, false, q0, q1, slot});
        else if (c >= 10) S.launches.push_back({c, DpKernel::Fill, 4, (uint32_t)c - 10, false, q0, q1, slot});
        else if (c == 2) S.launches.push_back({c, DpKernel::Fill, C.team_warps, C.cluster, false, q0, q1, slot});
        else {
            // Throughput mode: the first wave of blocks lands on the SMs in launch order, so deal the merges (sorted by
            // size) in snake rows of one block per SM -- the SM that got the largest merge of a row gets the smallest of
            // the next one.
            for (uint32_t r = q0 + sms, row = 1; r < q1; r += sms, ++row)
                if (row & 1) std::reverse(S.order.begin() + r, S.order.begin() + std::min(q1, r + sms));
            // Team size by how many merges there are: every SM holds 8 fill warps (shared memory), so a level with many
            // block-class merges runs them with smaller teams -- 4 warps from 2 merges per SM on, 2 from 4 -- which lose
            // less to the ramp-up / ramp-down of the stripe pipeline.
            // From two merges per SM on, the compact kernel (12 warps per SM): 6, 4 or 2 warps per merge.
            int nw = C.team_warps;
            bool compact = K.compact == 2 || (K.compact == 1 && n >= 2u * sms);
            if (compact) nw = n >= 6u * sms ? 2 : (n >= 3u * sms ? 4 : 6);
            else if (n >= 4u * sms) nw = 2;
            else if (n >= 2u * sms) nw = 4;
            if (K.team_warps) { nw = K.team_warps; compact = compact && (nw == 2 || nw == 4 || nw == 6); }
            const int team = nw == 2 || nw == 4 ? nw : (compact ? 6 : C.team_warps);
            if (compact) S.launches.push_back({c, DpKernel::Compact, team, 1, false, q0, q1, slot});
            // behind the compact kernel: the merges whose T needs 8 bytes, in a k_dp_fill team (4 warps behind NW = 6)
            S.launches.push_back({c, DpKernel::Fill, compact && team == 6 ? 4 : team, 1, compact, q0, q1, slot});
        }
        q0 = q1;
    }
    return S;
}

// The `[dp] batch of ...` line of a launch (FAMSA_DP_DEBUG); a class-1 line also names the team width and whether the
// compact kernel ran.
inline std::string dp_debug_line(const DpSubPlan& S, const DpLaunch& L, const std::vector<DpGeom>& jobs)
{
    const DpGeom& g = jobs[S.order[L.q0]];
    char buf[256];
    int k = snprintf(buf, sizeof(buf), "[dp] batch of %u: class %d x %u (first %u x %u, %u stripes), demand %llu, cl_cap %u, latency_mode %d",
                     (uint32_t)S.order.size(), L.cls, L.q1 - L.q0, g.w1, g.w2, host_stripes(g), S.demand, S.cl_cap, (int)S.small_batch);
    if (L.cls == 1) k += snprintf(buf + k, sizeof(buf) - k, ", team %d, compact %d", L.nw, (int)(L.kernel == DpKernel::Compact));
    return std::string(buf, k) + "\n";
}

} // namespace fb
