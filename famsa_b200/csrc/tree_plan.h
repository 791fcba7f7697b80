// Scheduling policy of famsa_prof_align_tree (prof.cu): dependency levels, which levels run fused, when the host waits for
// the device.  Plain C++ without CUDA headers, checked on its own by tests/cpp/tree_plan_check.cpp.
#pragma once
#include "../../include/famsa_b200.h"
#include "dp_plan.h"

namespace fb {

constexpr size_t kTreeMaxInFlight = 8;             // batches queued on the stream and not yet collected
constexpr size_t kTreeMaxFusedUncollected = 2;     // of them right after a fused launch is queued, itself included
constexpr uint32_t kTreeMaxFusedLevels = 32;       // dependency levels in one fused launch
constexpr size_t kTreeMaxFusedJobs = 8192;         // merges in one fused launch
constexpr uint32_t kTreeDriftSlack = 1024;         // a bound has drifted above kTreeDriftSlack + 2 x the widest exact width
constexpr uint64_t kTreeHeavyCells = 64ull << 20;  // bound cells above which a level is heavy
constexpr size_t kFusedMaxJobs = 4096;             // a batch of more merges never runs in the fused kernel,
constexpr uint32_t kFusedMaxHostRows = 512;        // nor one with a merge of more rows (host_rows)
constexpr uint32_t kFusedMaxWidth = 8192;          // or a wider child

// FAMSA_PROF_FUSED=0 runs every batch launch by launch (development knob, read from the environment once per call).
inline bool fused_allowed() { const char* e = getenv("FAMSA_PROF_FUSED"); return !e || atoi(e) != 0; }

// Dependency levels (appended to `levels`) of a tree_structure tree: merge k joins tree[2k] and tree[2k + 1] into node
// n_leaves + k, level d holds the merges whose deeper child is on level d - 1 in ascending order.  Children must precede
// their parent and be used once: returns -1, or the first node whose children break that.
inline int64_t tree_levels(const int32_t* tree, uint32_t n_leaves, std::vector<std::vector<uint32_t>>& levels)
{
    const uint32_t n_merges = n_leaves ? n_leaves - 1 : 0;
    std::vector<uint32_t> depth(n_leaves + n_merges, 0);
    std::vector<uint8_t> used(n_leaves + n_merges, 0);
    for (uint32_t k = 0; k < n_merges; ++k) {
        const int32_t a = tree[2 * k], b = tree[2 * k + 1];
        if (a < 0 || b < 0 || (uint32_t)a >= n_leaves + k || (uint32_t)b >= n_leaves + k || a == b || used[a] || used[b])
            return (int64_t)n_leaves + k;
        used[a] = used[b] = 1;
        const uint32_t d = std::max(depth[a], depth[b]) + 1;
        depth[n_leaves + k] = d;
        if (levels.size() < d) levels.resize(d);
        levels[d - 1].push_back(k);
    }
    return -1;
}

// May a batch run whole in k_merge_fused, every merge in one block?  allowed: fused_allowed()
inline bool fused_eligible(bool allowed, const std::vector<famsa_dp_job>& jobs)
{
    if (!allowed || jobs.size() > kFusedMaxJobs) return false;
    for (const famsa_dp_job& j : jobs)
        if (host_rows(j.p1.width, j.p1.card, j.p2.width, j.p2.card) > kFusedMaxHostRows || std::max(j.p1.width, j.p2.width) > kFusedMaxWidth) return false;
    return true;
}

// May a level of level_jobs merges join a fused launch of acc_levels levels and acc_jobs merges?  (The rings decide too.)
inline bool fused_joins(uint32_t acc_levels, size_t acc_jobs, size_t level_jobs) { return acc_levels < kTreeMaxFusedLevels && acc_jobs + level_jobs <= kTreeMaxFusedJobs; }

// A queued child is known by an upper bound (its children's summed), and along a chain bounds add up level after level.
// Has one drifted so far from the widest width the host knows that the host should wait for exact widths?
inline bool bound_drifted(uint32_t bound, uint32_t max_exact) { return bound > kTreeDriftSlack + 2 * max_exact; }

// How many of in_flight batches may stay queued before a level goes launch by launch ((size_t)-1: no need to wait)?  None
// when a child still pends and the level is heavy (the bounds would inflate its direction matrices) or when its paths
// end beyond the arena (which moves only while nothing is in flight); kTreeMaxInFlight - 1 when the queue is full.
inline size_t level_keep(bool pending_child, uint64_t bound_cells, uint64_t path_end, uint64_t path_cap, size_t in_flight)
{
    if ((pending_child && bound_cells > kTreeHeavyCells) || path_end > path_cap) return 0;
    return in_flight >= kTreeMaxInFlight ? kTreeMaxInFlight - 1 : (size_t)-1;
}

} // namespace fb
