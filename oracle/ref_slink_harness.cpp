// oracle/ref_slink_harness.cpp -- a C entry point over the UNMODIFIED reference's single-linkage guide tree (-gt slink).
//
// TEST INFRASTRUCTURE ONLY.  Compiled by oracle/Makefile into oracle/_ref/libfamsa_ref_slink.so, linked against
// oracle/_ref/libfamsa_ref.so, which already holds the reference's own src/tree/SingleLinkage.cpp.  Nothing under
// famsa_b200/ may load it.
//
// Reference seams exercised (paths relative to the FAMSA source tree):
//   SingleLinkage<distance>::run                           src/tree/SingleLinkage.cpp:30-189
//   AbstractTreeGenerator::operator()                      src/tree/AbstractTreeGenerator.cpp:25-32
#include <cstdint>
#include <string>
#include <vector>

#include "core/sequence.h"
#include "tree/SingleLinkage.h"

extern "C" {

// The reference's SLINK tree of sequences letters[0..n) in the given order, padded to the longest with UNKNOWN_SYMBOL
// as msa.cpp does before a tree is built.  kind 0 indel075_div_lcs, 1 indel_div_lcs.  out_pairs receives (left, right)
// for all 2n-1 nodes of tree_structure (leaves are -1, -1).  Returns 0 on success.
int ref_slink_tree(const char* const* letters, uint32_t n, int kind, int n_threads, int* out_pairs)
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
    if (kind == 0) {
        SingleLinkage<Distance::indel075_div_lcs> gen(n_threads, instruction_set_t::avx2);
        gen(ptrs, tree);
    } else if (kind == 1) {
        SingleLinkage<Distance::indel_div_lcs> gen(n_threads, instruction_set_t::avx2);
        gen(ptrs, tree);
    } else {
        return 1;
    }
    for (size_t i = 0; i < tree.size(); ++i) { out_pairs[2 * i] = tree[i].first; out_pairs[2 * i + 1] = tree[i].second; }
    return 0;
}

} // extern "C"
