// Runs the DP launch planner (famsa_b200/csrc/dp_plan.h) on a batch without a GPU.
//   dp_plan_check SM_COUNT CL_CAP DUO_CAP TEAM_WARPS CLUSTER < batch
// (TEAM_WARPS and CLUSTER: dp.cu's kDpTeamWarps and kDpCluster)
// batch: one merge per line, "w1 card1 w2 card2".  The knobs come from the environment, as in the library.
// Output per sub-batch: "sub j0 j1", "order <job>...", one "launch cls kernel nw cluster wide_only q0 q1 slot" line per
// launch (kernel 0 k_dp_fill, 1 k_dp_fill_compact, 2 k_dp_fill_duo) and, with FAMSA_DP_DEBUG, the library's [dp] lines.
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../../famsa_b200/csrc/dp_plan.h"

int main(int argc, char** argv)
{
    if (argc != 6) { fprintf(stderr, "usage: %s SM_COUNT CL_CAP DUO_CAP TEAM_WARPS CLUSTER < batch\n", argv[0]); return 2; }
    const fb::DpCaps caps{(uint32_t)atoi(argv[1]), (uint32_t)atoi(argv[2]), (uint32_t)atoi(argv[3]), atoi(argv[4]), (uint32_t)atoi(argv[5])};
    std::vector<fb::DpGeom> jobs;
    unsigned w1, c1, w2, c2;
    while (scanf("%u %u %u %u", &w1, &c1, &w2, &c2) == 4) jobs.push_back(fb::DpGeom{w1, c1, w2, c2, 0, 0});
    const fb::DpKnobs K = fb::dp_knobs();
    std::vector<fb::DpSub> subs;
    if (!fb::dp_cut(K.max_cells, jobs, subs)) { printf("too large\n"); return 1; }
    for (const fb::DpSub& sb : subs) {
        printf("sub %u %u\n", sb.j0, sb.j1);
        const fb::DpSubPlan plan = fb::dp_plan(K, caps, jobs, sb);
        printf("order");
        for (uint32_t j : plan.order) printf(" %u", j);
        printf("\n");
        for (const fb::DpLaunch& L : plan.launches) {
            printf("launch %d %d %d %u %d %u %u %u\n", L.cls, (int)L.kernel, L.nw, L.cluster, (int)L.wide_only, L.q0, L.q1, L.slot);
            if (K.debug && !L.wide_only) fputs(fb::dp_debug_line(plan, L, jobs).c_str(), stdout);
        }
    }
    return 0;
}
