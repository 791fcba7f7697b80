// oracle/ref_dist_harness.cpp -- C entry points over the UNMODIFIED reference's -dist_export path.
//
// TEST INFRASTRUCTURE ONLY.  Compiled by oracle/Makefile together with the reference's own
// src/tree/DistanceCalculator.cpp into oracle/_ref/libfamsa_ref_dist.so, linked against
// oracle/_ref/libfamsa_ref.so (the rest of the reference).  Nothing under famsa_b200/ may load it.
//
// Reference seams exercised (paths relative to the FAMSA source tree):
//   DistanceCalculator<distance>::run                      src/tree/DistanceCalculator.cpp:10-122
//   num2str(float) -> NumericConversions::Double2PChar     src/utils/conversion.h:52-133
//   CFAMSA::ComputeMSA, -dist_export branch                src/msa.cpp:518-526
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

#include "core/sequence.h"
#include "tree/DistanceCalculator.h"
#include "utils/conversion.h"

extern "C" {

// The file `famsa -dist_export [-square_matrix] [-pid]` writes for sequences letters[0..n) with ids[0..n) (FASTA
// headers without '>'), in input order: the sequences are padded to the longest with UNKNOWN_SYMBOL as msa.cpp does
// before the calculator runs (extendSequences).  kind 0 indel075_div_lcs, 1 indel_div_lcs.  Returns 0 on success.
int ref_dist_export(const char* const* letters, const char* const* ids, uint32_t n, int kind, int square, int pid,
                    const char* path, int n_threads)
{
    std::vector<CSequence> seqs;
    seqs.reserve(n);
    uint32_t max_len = 0;
    for (uint32_t i = 0; i < n; ++i) {
        seqs.emplace_back(std::string(">") + ids[i], std::string(letters[i]), (int)i, nullptr);
        if (seqs.back().length > max_len) max_len = seqs.back().length;
    }
    for (auto& q : seqs)
        if (q.length) q.DataResize(max_len, UNKNOWN_SYMBOL);
    std::vector<CSequence*> ptrs;
    for (auto& q : seqs) ptrs.push_back(&q);
    tree_structure tree;
    if (kind == 0) {
        DistanceCalculator<Distance::indel075_div_lcs> calc(n_threads, instruction_set_t::avx2, path, square != 0, pid != 0);
        calc(ptrs, tree);
    } else if (kind == 1) {
        DistanceCalculator<Distance::indel_div_lcs> calc(n_threads, instruction_set_t::avx2, path, square != 0, pid != 0);
        calc(ptrs, tree);
    } else {
        return 1;
    }
    return 0;
}

// num2str of every value, each followed by ',' (num2str(const T*, size, delim, out)); returns the bytes written
// (out must hold 40 * n bytes)
uint64_t ref_num2str_f32(const float* values, uint64_t n, char* out)
{
    return (uint64_t)num2str(values, (size_t)n, ',', out);
}

} // extern "C"
