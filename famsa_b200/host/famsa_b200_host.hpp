// famsa_b200_host.hpp -- C++ host side above the C ABI, shaped like the reference's own interfaces so
// that FAMSA's guide-tree builders and CProfile can be pointed at the GPU with one-line changes
// (INTEGRATION.md shows the exact seams).  Header-only; link with -lfamsa_b200.
//
//   reference                                                     here
//   ------------------------------------------------------------  -----------------------------------------
//   CLCSBP lcsbp(instruction_set)            src/lcs/lcsbp.h:15   famsa_b200::CLCSBP lcsbp(ctx, sequences)
//   lcsbp.GetLCSBP(seq0, s1..s8, dist)       lcsbp.h:38-46        lcsbp.GetLCSBP(seq0, ids, n, dist)
//   calculateDistanceVector/Range/Matrix     AbstractTreeGenerator.hpp:131,191,379   same names, same transforms
//   Transform<T, Distance::*>                AbstractTreeGenerator.hpp:28-82         famsa_b200::Transform<T, D>
//   CProfile::Align(p1, p2, ...)             src/core/profile.cpp:244                famsa_b200::AlignBatch(...)
//   MSTPrim<>::run_view's vertex loop        src/tree/MSTPrim.cpp:280-549            CLCSBP::PrimEdges(...)
//   CProfile(p1, p2) merge ctor, tables kept  profile.cpp:69-75, 784-1002            famsa_b200::ResidentProfiles
//   DistanceCalculator<distance>::run        src/tree/DistanceCalculator.cpp:10-122   famsa_b200::ExportDistances(...)
//   SingleLinkage<distance>::run             src/tree/SingleLinkage.cpp:30-189        famsa_b200::SingleLinkageTree(...)
//     on the device between tree levels
// Errors: the reference throws std::runtime_error and catches it in main() (src/famsa.cpp:160-165);
// every non-zero C-ABI status is rethrown here the same way.  There is no CPU fallback.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <limits>
#include <ostream>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/famsa_b200.h"

namespace famsa_b200 {

inline void check(int rc)
{
    if (rc != FAMSA_OK) throw std::runtime_error(std::string("famsa_b200: ") + famsa_last_error());
}

class Context {
    famsa_ctx* h_ = nullptr;
public:
    explicit Context(int device = -1) { check(famsa_create(device, &h_)); }
    ~Context() { famsa_destroy(h_); }
    Context(const Context&) = delete;
    Context& operator=(const Context&) = delete;
    famsa_ctx* get() const { return h_; }
};

// ---- LCS -> distance, on the host, bit-identical to the reference (AbstractTreeGenerator.hpp:28-82)
enum class Distance { indel_div_lcs, indel075_div_lcs, pairwise_identity };

template <class T, Distance measure> struct Transform;

template <class T> struct Transform<T, Distance::indel075_div_lcs> {
    std::vector<T> pp_pow075_rec;           // lazily grown table of (T) pow(i, 0.75), like the reference's
    T operator()(uint32_t lcs, uint32_t len1, uint32_t len2)
    {
        const T indel = (T)(len1 + len2 - 2 * lcs);
        const T l = (T)lcs;
        if (indel >= (T)pp_pow075_rec.size()) {
            const uint32_t upto = (uint32_t)indel;
            for (uint32_t v = (uint32_t)pp_pow075_rec.size(); v <= upto; ++v) pp_pow075_rec.push_back((T)std::pow(v, 0.75));
        }
        if (l) return pp_pow075_rec[(size_t)indel] / l;
        return (T)std::nextafter(std::numeric_limits<T>::max(), 0);
    }
};
template <class T> struct Transform<T, Distance::indel_div_lcs> {
    T operator()(uint32_t lcs, uint32_t len1, uint32_t len2)
    {
        const T indel = (T)(len1 + len2 - 2 * lcs);
        if (lcs) return (T)indel / lcs;
        return (T)std::nextafter(std::numeric_limits<T>::max(), 0);
    }
};
template <class T> struct Transform<T, Distance::pairwise_identity> {
    T operator()(uint32_t lcs, uint32_t len1, uint32_t len2) { return (T)lcs / std::min(len1, len2); }
};

// what the batch drivers need to know about a sequence (CSequence::data / CSequence::length)
struct SequenceView {
    const int8_t* data;
    uint32_t length;
};

// One instance serves every worker thread (the C ABI serialises calls on a context); in the reference each
// worker owns a CLCSBP because the CPU implementation keeps per-thread scratch (lcsbp_avx2_intr.h:27-36).
class CLCSBP {
    Context& ctx_;
    std::vector<uint32_t> lens_;
public:
    // uploads the set = ComputeBitMasks for every sequence (sequence.cpp:190-201), once
    CLCSBP(Context& ctx, const SequenceView* seqs, uint32_t n) : ctx_(ctx), lens_(n)
    {
        std::vector<uint64_t> off(n);
        uint64_t total = 0;
        for (uint32_t i = 0; i < n; ++i) { off[i] = total; lens_[i] = seqs[i].length; total += seqs[i].length; }
        std::vector<int8_t> codes(std::max<uint64_t>(total, 1));
        for (uint32_t i = 0; i < n; ++i) std::copy(seqs[i].data, seqs[i].data + seqs[i].length, codes.begin() + off[i]);
        check(famsa_lcs_upload(ctx_.get(), codes.data(), off.data(), lens_.data(), n));
    }
    uint32_t length(uint32_t i) const { return lens_[i]; }

    // the raw seam: LCS lengths of row `seq0` against n others (GetLCSBP's 4- and 8-way calls, any n)
    void GetLCSBP(uint32_t seq0, const uint32_t* ids, uint32_t n, uint32_t* dist)
    {
        check(famsa_lcs_rows(ctx_.get(), &seq0, 1, ids, n, dist, 4));
    }

    // AbstractTreeGenerator::calculateDistanceVector: ref against sequences[0 .. n_seqs)
    template <class distance_type, class Tr>
    void calculateDistanceVector(Tr& transform, uint32_t ref, uint32_t n_seqs, distance_type* out_vector)
    {
        std::vector<uint32_t> lcs(std::max(1u, n_seqs));
        check(famsa_lcs_rows(ctx_.get(), &ref, 1, nullptr, n_seqs, lcs.data(), 4));
        for (uint32_t k = 0; k < n_seqs; ++k) out_vector[k] = transform(lcs[k], lens_[ref], lens_[k]);
    }

    // AbstractTreeGenerator::calculateDistanceRange / RangeSV: ref against an id range
    template <class distance_type, class Iter, class Tr>
    void calculateDistanceRange(Tr& transform, uint32_t ref, Iter first, Iter last, distance_type* out_vector)
    {
        std::vector<uint32_t> ids(first, last), lcs(std::max<size_t>(1, ids.size()));
        check(famsa_lcs_rows(ctx_.get(), &ref, 1, ids.data(), (uint32_t)ids.size(), lcs.data(), 4));
        for (size_t k = 0; k < ids.size(); ++k) out_vector[k] = transform(lcs[k], lens_[ref], lens_[ids[k]]);
    }

    // AbstractTreeGenerator::calculateDistanceMatrix: packed lower triangle (TriangleMatrix::access)
    template <class distance_type, class Tr>
    void calculateDistanceMatrix(Tr& transform, uint32_t n_seq, distance_type* out_matrix)
    {
        const size_t pairs = (size_t)n_seq * (n_seq ? n_seq - 1 : 0) / 2;
        std::vector<uint32_t> lcs(std::max<size_t>(1, pairs));
        check(famsa_lcs_triangle(ctx_.get(), 0, n_seq, lcs.data(), 4));
        size_t at = 0;
        for (uint32_t i = 1; i < n_seq; ++i)
            for (uint32_t j = 0; j < i; ++j, ++at) out_matrix[at] = transform(lcs[at], lens_[i], lens_[j]);
    }
};

// MST edges in Prim order, ready for the reference's mst_to_dendogram (MSTPrim.cpp:784-833): edge k joins
// from[k] < to[k] at distance dist[k] (store -dist[k] in mst_edge_t as MSTPrim.cpp:384 does), order[i] = visiting
// position of sequence i.
struct PrimEdges {
    std::vector<int32_t> from, to, order;
    std::vector<double> dist;
};

// The default -gt sl guide tree: MSTPrim<distance>::run_view's relax/elect loop on the device.
inline PrimEdges PrimMST(Context& ctx, Distance measure)
{
    const uint32_t n = famsa_lcs_n_seqs(ctx.get());
    PrimEdges e;
    e.from.resize(n ? n - 1 : 0); e.to.resize(n ? n - 1 : 0); e.dist.resize(n ? n - 1 : 0); e.order.resize(n);
    if (measure == Distance::pairwise_identity) throw std::runtime_error("famsa_b200: MSTPrim is instantiated for the two indel distances only");
    check(famsa_lcs_prim(ctx.get(), measure == Distance::indel075_div_lcs ? 0 : 1, e.from.data(), e.to.data(), e.dist.data(), e.order.data()));
    return e;
}

// ---- profile alignment: what CProfile::Align hands to ConstructProfile
struct AlignResult {
    std::vector<uint8_t> path;     // direction_t per merged column, forward order (ConstructProfile's path[1..width])
    int64_t total_score;
    int64_t last[3];               // dp_row_elem_t {D,H,V} at the corner
    bool swapped;                  // true: the DP's row profile is the second argument (Align called the loop as (p2,p1))
    int variant;                   // 0 AlignSeqSeq, 1 AlignSeqProf, 2 AlignProfProf
};

// All ready merges of the guide tree in one call (the level-synchronous replacement for CProfileQueue's
// one-at-a-time hand-out, queues.cpp:127-187).
inline std::vector<AlignResult> AlignBatch(Context& ctx, const std::vector<famsa_dp_job>& jobs, const int64_t gaps[4])
{
    std::vector<famsa_dp_result> res(std::max<size_t>(1, jobs.size()));
    size_t path_total = 0;
    for (auto& j : jobs) path_total += (size_t)j.p1.width + j.p2.width;
    std::vector<uint8_t> path(std::max<size_t>(1, path_total));
    check(famsa_dp_align_batch(ctx.get(), jobs.data(), (uint32_t)jobs.size(), gaps, res.data(), path.data(), nullptr));
    std::vector<AlignResult> out(jobs.size());
    for (size_t k = 0; k < jobs.size(); ++k) {
        const famsa_dp_result& r = res[k];
        out[k].path.assign(path.begin() + r.path_offset, path.begin() + r.path_offset + r.path_len);
        out[k].total_score = r.total_score;
        std::copy(r.last, r.last + 3, out[k].last);
        out[k].swapped = r.swapped != 0;
        out[k].variant = r.variant;
    }
    return out;
}

// (first merged column, run length) of the gap columns a path inserts into the members of the DP's row profile
// (direction H = 1) or column profile (direction V = 2) -- ConstructProfile's v_gaps_prof1 / v_gaps_prof2
// (profile.cpp:1020-1029), the input of FinalizeGaps (profile.cpp:1053-1104).
inline std::vector<std::pair<uint32_t, uint32_t>> GapRuns(const std::vector<uint8_t>& path, uint8_t dir)
{
    std::vector<std::pair<uint32_t, uint32_t>> runs;
    for (uint32_t k = 0; k < path.size();) {
        if (path[k] != dir) { ++k; continue; }
        uint32_t e = k;
        while (e < path.size() && path[e] == dir) ++e;
        runs.emplace_back(k + 1, e - k);
        k = e;
    }
    return runs;
}

// Profiles whose scores/counters stay in HBM between the levels of the guide tree (famsa_prof_*).  A node is either
// a leaf (sequence id of CLCSBP's upload) or the id a previous MergeLevel returned.  Per merge only the path comes
// back; the host applies GapRuns(path, 1 / 2) to the member sequences of the row / column profile with the
// reference's FinalizeGaps and concatenates `data` as ConstructProfile does (profile.cpp:990-996).
class ResidentProfiles {
    Context& ctx_;
    std::vector<uint32_t> width_;           // by resident id
    std::vector<uint32_t> leaf_len_;
public:
    static uint32_t Leaf(uint32_t seq_id) { return FAMSA_PROF_LEAF | seq_id; }
    // score_matrix: CParams::score_matrix, 24 x 24; leaf_lengths: CSequence::length of the uploaded sequences
    ResidentProfiles(Context& ctx, const int64_t* score_matrix, std::vector<uint32_t> leaf_lengths)
        : ctx_(ctx), leaf_len_(std::move(leaf_lengths)) { check(famsa_prof_set_scoring(ctx.get(), score_matrix)); }
    uint32_t Width(uint32_t node) const { return (node & FAMSA_PROF_LEAF) ? leaf_len_.at(node & ~FAMSA_PROF_LEAF) : width_.at(node); }
    // all ready merges of one level; children are consumed; out_ids[k] = resident id of merge k
    std::vector<AlignResult> MergeLevel(const std::vector<famsa_prof_merge>& merges, const int64_t gaps[4], std::vector<uint32_t>& out_ids)
    {
        const size_t n = merges.size();
        size_t cap = 0;
        for (auto& m : merges) cap += (size_t)Width(m.child1) + Width(m.child2);
        std::vector<famsa_dp_result> res(std::max<size_t>(1, n));
        std::vector<uint8_t> path(std::max<size_t>(1, cap));
        out_ids.assign(n, 0);
        check(famsa_prof_merge_batch(ctx_.get(), merges.data(), (uint32_t)n, gaps, out_ids.data(), res.data(), path.data(), cap));
        std::vector<AlignResult> out(n);
        for (size_t k = 0; k < n; ++k) {
            const famsa_dp_result& r = res[k];
            out[k].path.assign(path.begin() + r.path_offset, path.begin() + r.path_offset + r.path_len);
            out[k].total_score = r.total_score;
            std::copy(r.last, r.last + 3, out[k].last);
            out[k].swapped = r.swapped != 0;
            out[k].variant = r.variant;
            if (width_.size() <= out_ids[k]) width_.resize(out_ids[k] + 1);
            width_[out_ids[k]] = r.path_len;
        }
        return out;
    }
    // scores ((width+1) x 32) and counters of a resident profile, e.g. the root for refinement
    void Download(uint32_t id, std::vector<int64_t>& scores, std::vector<int32_t>& counters, uint32_t& card)
    {
        uint32_t w = 0;
        check(famsa_prof_get(ctx_.get(), id, &w, &card, nullptr, nullptr));
        scores.resize(((size_t)w + 1) * 32); counters.resize(((size_t)w + 1) * 32);
        check(famsa_prof_get(ctx_.get(), id, nullptr, nullptr, scores.data(), counters.data()));
    }
    void Drop(const std::vector<uint32_t>& ids) { check(famsa_prof_drop(ctx_.get(), ids.data(), (uint32_t)ids.size())); }
};

// The whole merge loop of CFAMSA::ComputeAlignment (msa.cpp:360-438, with CProfileQueue, queues.cpp:17-187) as one call:
// guide_tree = the reference's tree_structure (n_leaves leaf entries, then one (left, right) pair per internal node,
// children before parents); leaves are the sequences of CLCSBP's upload.  merges[k] describes internal node n_leaves + k.
struct TreeAlignment {
    std::vector<AlignResult> merges;
    uint32_t root_id = 0;              // resident id of the final profile (ResidentProfiles::Download / Drop)
    famsa_tree_stats stats{};
};
inline TreeAlignment AlignTree(Context& ctx, const std::vector<std::pair<int, int>>& guide_tree, uint32_t n_leaves, const int64_t gaps[4])
{
    static_assert(sizeof(std::pair<int, int>) == 2 * sizeof(int32_t), "tree_structure is a vector of int pairs");
    TreeAlignment out;
    const size_t n_merges = guide_tree.size() > n_leaves ? guide_tree.size() - n_leaves : 0;
    std::vector<famsa_dp_result> res(std::max<size_t>(1, n_merges));
    uint64_t path_bytes = 0;
    check(famsa_prof_align_tree(ctx.get(), reinterpret_cast<const int32_t*>(guide_tree.data() + n_leaves), n_leaves, gaps, res.data(),
                                &out.root_id, &path_bytes, &out.stats));
    std::vector<uint8_t> paths(std::max<uint64_t>(1, path_bytes));
    check(famsa_prof_tree_paths(ctx.get(), paths.data(), paths.size()));
    out.merges.resize(n_merges);
    for (size_t k = 0; k < n_merges; ++k) {
        const famsa_dp_result& r = res[k];
        out.merges[k].path.assign(paths.begin() + r.path_offset, paths.begin() + r.path_offset + r.path_len);
        out.merges[k].total_score = r.total_score;
        std::copy(r.last, r.last + 3, out.merges[k].last);
        out.merges[k].swapped = r.swapped != 0;
        out.merges[k].variant = r.variant;
    }
    return out;
}

// The finished alignment of `tree` (the most recent AlignTree on ctx), built on the device by famsa_prof_tree_rows: what
// FinalizeGaps does at every merge (profile.cpp:1053-1104), with no host work per merge.  Row k is leaf order[k] (empty
// order: leaf k), width codes each, GAP = 30; a drop-in rebuilds its CGappedSequences from them (INTEGRATION.md).  The rows
// also stay on the device for famsa_prof_refine with FAMSA_REFINE_TREE_ROWS (order = the id order there).
struct TreeRowsOut {
    std::vector<uint8_t> rows;         // n_rows x width, row-major
    uint32_t n_rows = 0, width = 0;
};
inline TreeRowsOut TreeRows(Context& ctx, const TreeAlignment& tree, const std::vector<uint32_t>& order = {})
{
    TreeRowsOut out;
    out.n_rows = (uint32_t)tree.merges.size() + 1;
    const uint32_t width = tree.merges.empty() ? 0 : (uint32_t)tree.merges.back().path.size();
    out.rows.resize((size_t)out.n_rows * width);
    check(famsa_prof_tree_rows(ctx.get(), order.empty() ? nullptr : order.data(), out.n_rows, out.rows.data(), out.rows.size(), &out.width));
    return out;
}

// CFAMSA::alignProfiles (msa.cpp:675-718) without its RefineAlignment: the two alignments' profiles as the reference builds
// them from rows read as text (famsa_prof_put_rows with FAMSA_PUT_ROWS_FROM_TEXT: each profile leaves out its last column)
// and one unbanded merge.  rows: codes 0..23 or GAP = 30, every row of an alignment as long as its first.  Needs
// famsa_prof_set_scoring.  gaps1 / gaps2: the GapRuns FinalizeGaps applies to rows1's / rows2's members (the row profile's
// H runs, the column profile's V runs); the last column of every input row stays apart and ends its merged row.
// order[k]: input row (k < n1: rows1[k], else rows2[k - n1]) of merged row k -- the column profile's rows, then the row
// profile's (ConstructProfile, profile.cpp:992-993).  merged_id: the merged resident profile, the caller's to drop.
struct ProfileAlignment {
    AlignResult merge;
    uint32_t merged_id = 0;
    std::vector<std::pair<uint32_t, uint32_t>> gaps1, gaps2;
    std::vector<uint32_t> order;
};
inline ProfileAlignment AlignProfiles(Context& ctx, const std::vector<std::vector<uint8_t>>& rows1,
                                      const std::vector<std::vector<uint8_t>>& rows2, const int64_t gaps[4])
{
    const std::vector<std::vector<uint8_t>>* in[2] = {&rows1, &rows2};
    uint32_t ids[2], widths[2];
    int n_put = 0;
    try {
        for (int s = 0; s < 2; ++s) {
            const auto& rows = *in[s];
            if (rows.empty()) throw std::runtime_error("Incorrect profile");      // famsa.cpp:83-89
            std::vector<uint8_t> flat;
            for (const auto& r : rows) {
                if (r.size() != rows.front().size()) throw std::runtime_error("Incorrect profile");
                flat.insert(flat.end(), r.begin(), r.end());
            }
            check(famsa_prof_put_rows(ctx.get(), flat.data(), (uint32_t)rows.size(), (uint32_t)rows.front().size(), gaps,
                                      FAMSA_PUT_ROWS_FROM_TEXT, &ids[s]));
            widths[s] = (uint32_t)rows.front().size() - 1;
            ++n_put;
        }
    } catch (...) {
        if (n_put) famsa_prof_drop(ctx.get(), ids, (uint32_t)n_put);
        throw;
    }
    const famsa_prof_merge m{ids[0], ids[1]};
    famsa_dp_result r{};
    std::vector<uint8_t> path((size_t)widths[0] + widths[1]);
    ProfileAlignment out;
    check(famsa_prof_merge_batch(ctx.get(), &m, 1, gaps, &out.merged_id, &r, path.data(), path.size()));
    out.merge.path.assign(path.begin() + r.path_offset, path.begin() + r.path_offset + r.path_len);
    out.merge.total_score = r.total_score;
    std::copy(r.last, r.last + 3, out.merge.last);
    out.merge.swapped = r.swapped != 0;
    out.merge.variant = r.variant;
    const uint32_t n1 = (uint32_t)rows1.size(), n2 = (uint32_t)rows2.size();
    auto row_runs = GapRuns(out.merge.path, 1), col_runs = GapRuns(out.merge.path, 2);
    out.gaps1 = out.merge.swapped ? col_runs : row_runs;
    out.gaps2 = out.merge.swapped ? row_runs : col_runs;
    const uint32_t col_first = out.merge.swapped ? 0 : n1, col_n = out.merge.swapped ? n1 : n2;
    const uint32_t row_first = out.merge.swapped ? n1 : 0, row_n = out.merge.swapped ? n2 : n1;
    for (uint32_t i = 0; i < col_n; ++i) out.order.push_back(col_first + i);
    for (uint32_t i = 0; i < row_n; ++i) out.order.push_back(row_first + i);
    return out;
}

// UPGMA<distance>::run (UPGMA.cpp:39-51) on the device: the n - 1 merges, tree_structure's internal-node part
inline std::vector<std::pair<int, int>> UPGMATree(Context& ctx, Distance measure, bool modified)
{
    const uint32_t n = famsa_lcs_n_seqs(ctx.get());
    if (measure == Distance::pairwise_identity) throw std::runtime_error("famsa_b200: UPGMA is instantiated for the two indel distances only");
    std::vector<int32_t> t(2 * (size_t)std::max<uint32_t>(n, 1));
    check(famsa_lcs_upgma(ctx.get(), measure == Distance::indel075_div_lcs ? 0 : 1, modified ? 1 : 0, t.data()));
    std::vector<std::pair<int, int>> out;
    for (uint32_t k = 0; k + 1 < n; ++k) out.emplace_back(t[2 * k], t[2 * k + 1]);
    return out;
}

// SingleLinkage<distance>::run (SingleLinkage.cpp:30-189) on the device: the n - 1 merges, tree_structure's internal-node part
inline std::vector<std::pair<int, int>> SingleLinkageTree(Context& ctx, Distance measure)
{
    const uint32_t n = famsa_lcs_n_seqs(ctx.get());
    if (measure == Distance::pairwise_identity) throw std::runtime_error("famsa_b200: SingleLinkage is instantiated for the two indel distances only");
    std::vector<int32_t> t(2 * (size_t)std::max<uint32_t>(n, 1));
    check(famsa_lcs_slink(ctx.get(), measure == Distance::indel075_div_lcs ? 0 : 1, t.data()));
    std::vector<std::pair<int, int>> out;
    for (uint32_t k = 0; k + 1 < n; ++k) out.emplace_back(t[2 * k], t[2 * k + 1]);
    return out;
}

// NeighborJoining<distance>::run (NeighborJoining.cpp:10-21) on the device: the n - 1 merges, tree_structure's internal-node part
inline std::vector<std::pair<int, int>> NeighborJoiningTree(Context& ctx, Distance measure)
{
    const uint32_t n = famsa_lcs_n_seqs(ctx.get());
    if (measure == Distance::pairwise_identity) throw std::runtime_error("famsa_b200: NeighborJoining is instantiated for the two indel distances only");
    std::vector<int32_t> t(2 * (size_t)std::max<uint32_t>(n, 1));
    check(famsa_lcs_nj(ctx.get(), measure == Distance::indel075_div_lcs ? 0 : 1, t.data()));
    std::vector<std::pair<int, int>> out;
    for (uint32_t k = 0; k + 1 < n; ++k) out.emplace_back(t[2 * k], t[2 * k + 1]);
    return out;
}

// DistanceCalculator<distance>::run (DistanceCalculator.cpp:10-122) on the device: the -dist_export CSV of the set of
// the last famsa_lcs_upload (input order) into `os`, byte for byte.  ids: CSequence::id without the leading '>'.
// Returns the bytes written; a failing stream stops the export and throws.
inline uint64_t ExportDistances(Context& ctx, const std::vector<std::string>& ids, Distance measure, bool square_matrix,
                                std::ostream& os, uint64_t chunk_bytes = 0)
{
    std::string blob;
    std::vector<uint64_t> offsets{0};
    for (const std::string& id : ids) { blob += id; offsets.push_back(blob.size()); }
    const bool pid = measure == Distance::pairwise_identity;
    const int kind = measure == Distance::indel_div_lcs ? 1 : 0;
    auto sink = [](void* user, const char* bytes, uint64_t n) -> int {
        std::ostream& o = *static_cast<std::ostream*>(user);
        o.write(bytes, (std::streamsize)n);
        return o.good() ? 0 : 1;
    };
    uint64_t written = 0;
    check(famsa_dist_export(ctx.get(), kind, square_matrix ? 1 : 0, pid ? 1 : 0, blob.data(), offsets.data(), chunk_bytes,
                            sink, &os, &written));
    return written;
}

// Level-synchronous order of the guide tree's merges (replaces CProfileQueue's one-at-a-time hand-out,
// queues.cpp:17-187): tree = the reference's tree_structure, n leaves then internal nodes (left, right).
// Returns, per level, the indices (into the internal-node part) of the merges whose children are finished.
inline std::vector<std::vector<uint32_t>> ReadyLevels(const std::vector<std::pair<int, int>>& tree, uint32_t n_leaves)
{
    std::vector<uint32_t> depth(tree.size(), 0);
    std::vector<std::vector<uint32_t>> levels;
    for (uint32_t node = n_leaves; node < tree.size(); ++node) {
        const uint32_t d = std::max(depth[tree[node].first], depth[tree[node].second]) + 1;
        depth[node] = d;
        if (levels.size() < d) levels.resize(d);
        levels[d - 1].push_back(node - n_leaves);
    }
    return levels;
}

} // namespace famsa_b200
