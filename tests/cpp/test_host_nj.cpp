// The C++ mirror's NeighborJoiningTree (famsa_b200/host/famsa_b200_host.hpp) on a random set in FAMSA's order: argv[1]
// names a file that receives the merges, one "left right" line each, for the Python test to compare with Engine.nj.
#include <cstdio>
#include <random>

#include "../../famsa_b200/host/famsa_b200_host.hpp"

#define REQUIRE(c) do { if (!(c)) { std::printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #c); return 1; } } while (0)

int main(int argc, char** argv)
{
    using namespace famsa_b200;
    if (argc != 2) return 2;
    std::mt19937 rng(11);
    const uint32_t n = 200;
    std::vector<std::vector<int8_t>> seqs(n);
    for (auto& s : seqs) { s.resize(20 + rng() % 120); for (auto& c : s) c = (int8_t)(rng() % 6); }
    std::sort(seqs.begin(), seqs.end(), [](auto& a, auto& b) { return a.size() > b.size(); });
    std::vector<SequenceView> views(n);
    for (uint32_t i = 0; i < n; ++i) views[i] = {seqs[i].data(), (uint32_t)seqs[i].size()};
    Context ctx(0);
    CLCSBP lcsbp(ctx, views.data(), n);
    const auto tree = NeighborJoiningTree(ctx, Distance::indel075_div_lcs);
    REQUIRE(tree.size() == n - 1);
    std::vector<int> used(2 * n - 1, 0);
    for (uint32_t k = 0; k + 1 < n; ++k) {
        REQUIRE(tree[k].first >= 0 && tree[k].second >= 0 && (uint32_t)tree[k].first < n + k && (uint32_t)tree[k].second < n + k);
        ++used[tree[k].first]; ++used[tree[k].second];
    }
    for (uint32_t v = 0; v + 1 < 2 * n - 1; ++v) REQUIRE(used[v] == 1);              // every node but the root merged once
    bool threw = false;
    try { NeighborJoiningTree(ctx, Distance::pairwise_identity); } catch (const std::runtime_error&) { threw = true; }
    REQUIRE(threw);
    FILE* f = std::fopen(argv[1], "w");
    REQUIRE(f);
    for (uint32_t i = 0; i < n; ++i) {                                                  // the set, then the merges
        for (int8_t c : seqs[i]) std::fputc('0' + c, f);
        std::fputc('\n', f);
    }
    for (auto& m : tree) std::fprintf(f, "%d %d\n", m.first, m.second);
    std::fclose(f);
    std::printf("host mirror nj ok\n");
    return 0;
}
