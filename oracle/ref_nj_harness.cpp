// oracle/ref_nj_harness.cpp -- C entry points over the UNMODIFIED reference's neighbour-joining guide tree (-gt nj).
//
// TEST INFRASTRUCTURE ONLY.  Compiled by oracle/Makefile into oracle/_ref/libfamsa_ref_nj.so, linked against
// oracle/_ref/libfamsa_ref.so, which already holds the reference's own src/tree/NeighborJoining.cpp.  Nothing under
// famsa_b200/ may load it.
//
// Reference seams exercised (paths relative to the FAMSA source tree):
//   NeighborJoining<distance>::run                         src/tree/NeighborJoining.cpp:10-21
//   NeighborJoining<distance>::computeTree                 src/tree/NeighborJoining.cpp:33-118 (protected: reached
//                                                          through a derived class)
//   AbstractTreeGenerator::operator()                      src/tree/AbstractTreeGenerator.cpp:25-32
#include <chrono>
#include <cstdint>
#include <string>
#include <vector>

#include "core/sequence.h"
#include "tree/NeighborJoining.h"

namespace {
template <Distance d>
struct NjOnTriangle : NeighborJoining<d> {
    NjOnTriangle() : NeighborJoining<d>(1, instruction_set_t::avx2) {}
    void tree_of(float* distances, int n, tree_structure& tree) { this->computeTree(distances, n, tree); }
};
} // namespace

extern "C" {

// The reference's NJ tree of sequences letters[0..n) in the given order, padded to the longest with UNKNOWN_SYMBOL as
// msa.cpp does before a tree is built.  kind 0 indel075_div_lcs, 1 indel_div_lcs.  out_pairs receives (left, right) for
// all 2n-1 nodes of tree_structure (leaves are -1, -1).  *seconds (if not NULL) = wall time of the generator call.
// Returns 0 on success.
int ref_nj_tree(const char* const* letters, uint32_t n, int kind, int* out_pairs, double* seconds)
{
    std::vector<CSequence> seqs;
    seqs.reserve(n);
    uint32_t max_len = 0;
    for (uint32_t i = 0; i < n; ++i) {
        seqs.emplace_back("s" + std::to_string(i), std::string(letters[i]), (int)i, nullptr);
        if (seqs.back().length > max_len) max_len = seqs.back().length;
    }
    for (auto& q : seqs)
        if (q.length) q.DataResize(max_len, UNKNOWN_SYMBOL);
    std::vector<CSequence*> ptrs;
    for (auto& q : seqs) ptrs.push_back(&q);
    tree_structure tree;
    const auto t0 = std::chrono::steady_clock::now();
    if (kind == 0) {
        NeighborJoining<Distance::indel075_div_lcs> gen(1, instruction_set_t::avx2);
        gen(ptrs, tree);
    } else if (kind == 1) {
        NeighborJoining<Distance::indel_div_lcs> gen(1, instruction_set_t::avx2);
        gen(ptrs, tree);
    } else {
        return 1;
    }
    if (seconds) *seconds = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    for (size_t i = 0; i < tree.size(); ++i) { out_pairs[2 * i] = tree[i].first; out_pairs[2 * i + 1] = tree[i].second; }
    return 0;
}

// The reference's computeTree on an external float triangle (row i against j < i at i(i-1)/2 + j), updated in place.
// out_pairs receives the n-1 merges.  Returns 0 on success.
int ref_nj_tree_from_distances(float* tri, int n, int kind, int* out_pairs)
{
    tree_structure tree;
    if (kind == 0) NjOnTriangle<Distance::indel075_div_lcs>().tree_of(tri, n, tree);
    else if (kind == 1) NjOnTriangle<Distance::indel_div_lcs>().tree_of(tri, n, tree);
    else return 1;
    for (size_t i = 0; i < tree.size(); ++i) { out_pairs[2 * i] = tree[i].first; out_pairs[2 * i + 1] = tree[i].second; }
    return 0;
}

} // extern "C"
