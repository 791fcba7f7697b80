// Runs the progressive-alignment scheduling policy (famsa_b200/csrc/tree_plan.h) without a GPU.
//   tree_plan_check levels < tree         tree: "n_leaves" then one merge per line, "a b" (tree_structure order);
//                                          prints "bad NODE" or one line per dependency level, its merge indices
//   tree_plan_check limits                 one "name value" line per named limit
//   tree_plan_check eligible < batch       batch: one merge per line, "w1 card1 w2 card2"; prints 0 / 1
//                                          (FAMSA_PROF_FUSED comes from the environment, as in the library)
//   tree_plan_check joins ACC_LEVELS ACC_JOBS LEVEL_JOBS
//   tree_plan_check drifted BOUND MAX_EXACT
//   tree_plan_check keep PENDING_CHILD BOUND_CELLS PATH_END PATH_CAP IN_FLIGHT   prints the batches that may stay, or -1
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../famsa_b200/csrc/tree_plan.h"

static unsigned long long arg(char** argv, int i) { return strtoull(argv[i], nullptr, 10); }

int main(int argc, char** argv)
{
    const char* cmd = argc > 1 ? argv[1] : "";
    if (!strcmp(cmd, "levels") && argc == 2) {
        unsigned n_leaves;
        if (scanf("%u", &n_leaves) != 1) return 2;
        std::vector<int32_t> tree;
        int a, b;
        while (scanf("%d %d", &a, &b) == 2) { tree.push_back(a); tree.push_back(b); }
        if (tree.size() != 2 * (size_t)(n_leaves - 1)) { fprintf(stderr, "%u leaves need %u merges\n", n_leaves, n_leaves - 1); return 2; }
        std::vector<std::vector<uint32_t>> levels;
        const int64_t bad = fb::tree_levels(tree.data(), n_leaves, levels);
        if (bad >= 0) { printf("bad %lld\n", (long long)bad); return 0; }
        for (const auto& level : levels) {
            for (size_t i = 0; i < level.size(); ++i) printf(i ? " %u" : "%u", level[i]);
            printf("\n");
        }
    } else if (!strcmp(cmd, "limits") && argc == 2) {
        printf("max_in_flight %zu\nmax_fused_uncollected %zu\nmax_fused_levels %u\nmax_fused_jobs %zu\ndrift_slack %u\n"
               "heavy_cells %llu\nfused_max_jobs %zu\nfused_max_host_rows %u\nfused_max_width %u\n",
               fb::kTreeMaxInFlight, fb::kTreeMaxFusedUncollected, fb::kTreeMaxFusedLevels, fb::kTreeMaxFusedJobs, fb::kTreeDriftSlack,
               (unsigned long long)fb::kTreeHeavyCells, fb::kFusedMaxJobs, fb::kFusedMaxHostRows, fb::kFusedMaxWidth);
    } else if (!strcmp(cmd, "eligible") && argc == 2) {
        std::vector<famsa_dp_job> jobs;
        unsigned w1, c1, w2, c2;
        while (scanf("%u %u %u %u", &w1, &c1, &w2, &c2) == 4) {
            famsa_dp_job j{};
            j.p1.width = w1; j.p1.card = c1; j.p2.width = w2; j.p2.card = c2;
            jobs.push_back(j);
        }
        printf("%d\n", (int)fb::fused_eligible(fb::fused_allowed(), jobs));
    } else if (!strcmp(cmd, "joins") && argc == 5) {
        printf("%d\n", (int)fb::fused_joins((uint32_t)arg(argv, 2), arg(argv, 3), arg(argv, 4)));
    } else if (!strcmp(cmd, "drifted") && argc == 4) {
        printf("%d\n", (int)fb::bound_drifted((uint32_t)arg(argv, 2), (uint32_t)arg(argv, 3)));
    } else if (!strcmp(cmd, "keep") && argc == 7) {
        printf("%lld\n", (long long)fb::level_keep(arg(argv, 2) != 0, arg(argv, 3), arg(argv, 4), arg(argv, 5), arg(argv, 6)));
    } else {
        fprintf(stderr, "usage: %s levels | limits | eligible | joins L J N | drifted B M | keep P C E CAP N\n", argv[0]);
        return 2;
    }
    return 0;
}
