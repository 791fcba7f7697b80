// oracle/ref_harness.cpp -- thin C entry points over the UNMODIFIED reference sources.
//
// TEST INFRASTRUCTURE ONLY (see oracle/README.md).  This translation unit is ours; it is linked
// against object files compiled straight from /root/reference/src (never copied into the repo)
// by oracle/Makefile, producing oracle/_ref/libfamsa_ref.so.  It is used
//   * by tests/ to pin oracle/lcs_oracle.c and oracle/dp_oracle.c against the real reference,
//   * by bench.py --impl reference / cpu_baseline (kind "reference") as the timed CPU arm.
// Nothing under famsa_b200/ may load it.
//
// Reference seams exercised (paths relative to /root/reference):
//   CSequence ctor / DataResize / ComputeBitMasks          src/core/sequence.cpp:22-201
//   CLCSBP::GetLCSBP (8-way CSequence* overload)           src/lcs/lcsbp.cpp:163-264
//   AbstractTreeGenerator::calculateDistanceVector         src/tree/AbstractTreeGenerator.hpp:131-182
//   Transform<T, Distance>                                 src/tree/AbstractTreeGenerator.hpp:28-82
//   CProfile(const CGappedSequence&, CParams*)             src/core/profile.cpp:45-51
//   CProfile(CProfile*, CProfile*, CParams*, ...) -> Align src/core/profile.cpp:69-75, 244-305
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <thread>
#include <type_traits>
#include <vector>

#define private public      // harness TU only: read CProfile internals, nothing is modified
#define protected public
#include "core/defs.h"
#include "core/params.h"
#include "core/profile.h"
#include "core/queues.h"
#include "core/sequence.h"
#include "lcs/lcsbp.h"
#include "tree/AbstractTreeGenerator.h"
#include "tree/AbstractTreeGenerator.hpp"
#include "tree/UPGMA.h"
#include "tree/MSTPrim.h"
#undef private
#undef protected

namespace {

// Smallest concrete generator: we only want the batch-driver templates of the base class.
struct DriverOnly : public AbstractTreeGenerator {
    DriverOnly(instruction_set_t isa) : AbstractTreeGenerator(1, isa) {}
    void run(std::vector<CSequence*>&, tree_structure&) override {}
};

// "Transform" that hands back the raw LCS length instead of a distance.
struct RawLcs {
    uint32_t operator()(uint32_t lcs, uint32_t, uint32_t) { return lcs; }
};

instruction_set_t isa_from_int(int isa)
{
    switch (isa) {
    case 0: return instruction_set_t::none;      // scalar CLCSBP_Classic
    case 1: return instruction_set_t::avx;       // 2 pairs / call
    default: return instruction_set_t::avx2;     // 4 pairs / call (the metric's CPU baseline)
    }
}

struct SeqSet {
    std::vector<CSequence> seqs;       // padded to the set-wide max length with UNKNOWN (msa.cpp:271,297)
    std::vector<CSequence*> ptrs;
};

} // namespace

// CProfile::ConstructProfile and its dp_row_elem_t parameter sit in the class's default-private section (no
// `private:` keyword for the macro above to catch).  An explicit template instantiation may name a private
// member, which hands us the member-function pointer without touching the reference source.
auto stolen_construct_profile();
template <auto M> struct StealMember {
    friend auto stolen_construct_profile() { return M; }
};
template struct StealMember<&CProfile::ConstructProfile>;
template <class T> struct ConstructTraits;
template <class C, class R, class A1, class A2, class A3, class A4, class A5>
struct ConstructTraits<R (C::*)(A1, A2, A3, A4, A5)> {
    using elem_t = std::remove_reference_t<A4>;      // CProfile::dp_row_elem_t
};

// Same trick for MSTPrim<>::mst_to_dendogram (private) and its vector<mst_edge_t> argument.
using PrimRef = MSTPrim<Distance::indel075_div_lcs>;
auto stolen_mst_to_dendogram();
template <auto M> struct StealPrimMember {
    friend auto stolen_mst_to_dendogram() { return M; }
};
template struct StealPrimMember<&PrimRef::mst_to_dendogram>;
template <class T> struct DendTraits;
template <class C, class R, class A1, class A2, class A3>
struct DendTraits<R (C::*)(A1, A2, A3)> {
    using edges_t = std::remove_reference_t<A1>;     // std::vector<MSTPrim::mst_edge_t>
};

extern "C" {

// ---------------------------------------------------------------- sequence sets
// `letters[i]` is the raw residue string; encoding is the reference's own (sequence.cpp:53-79).
void* ref_seqset_create(const char* const* letters, uint32_t n)
{
    auto* s = new SeqSet();
    s->seqs.reserve(n);
    uint32_t max_len = 0;
    for (uint32_t i = 0; i < n; ++i) {
        s->seqs.emplace_back("s" + std::to_string(i), std::string(letters[i]), (int)i, nullptr);
        if (s->seqs.back().length > max_len) max_len = s->seqs.back().length;
    }
    for (auto& q : s->seqs)
        if (q.length) q.DataResize(max_len, UNKNOWN_SYMBOL);
    for (auto& q : s->seqs) s->ptrs.push_back(&q);
    return s;
}

void ref_seqset_destroy(void* h) { delete static_cast<SeqSet*>(h); }

uint32_t ref_seqset_len(void* h, uint32_t i) { return static_cast<SeqSet*>(h)->seqs[i].length; }

// copies the reference's residue codes (without padding) into out[0..len)
void ref_seqset_codes(void* h, uint32_t i, int8_t* out)
{
    auto& q = static_cast<SeqSet*>(h)->seqs[i];
    if (q.length) memcpy(out, q.data, q.length);
}

// ---------------------------------------------------------------- HP-1: LCS
// Row `ref` (supplies the bit masks) against sequences[0..n_cols) -- exactly what SLINK/UPGMA/NJ/
// DistanceCalculator do per row.  out[k] = LCS length.
void ref_lcs_row_prefix(void* h, uint32_t ref, uint32_t n_cols, uint32_t* out, int isa)
{
    auto* s = static_cast<SeqSet*>(h);
    DriverOnly drv(isa_from_int(isa));
    CLCSBP lcsbp(isa_from_int(isa));
    RawLcs raw;
    drv.calculateDistanceVector<CSequence*, uint32_t, RawLcs>(raw, s->ptrs[ref], s->ptrs.data(),
                                                              (int)n_cols, out, lcsbp);
}

// Row `ref` against an arbitrary id list (Prim / medoid shape, calculateDistanceRange).
void ref_lcs_row_ids(void* h, uint32_t ref, const int* ids, uint32_t n_ids, uint32_t* out, int isa)
{
    auto* s = static_cast<SeqSet*>(h);
    DriverOnly drv(isa_from_int(isa));
    CLCSBP lcsbp(isa_from_int(isa));
    RawLcs raw;
    s->ptrs[ref]->ComputeBitMasks();       // calculateDistanceRange expects the caller to do this
    drv.calculateDistanceRange<CSequence*, uint32_t, const int*, RawLcs>(
        raw, s->ptrs[ref], s->ptrs.data(), std::make_pair(ids, ids + n_ids), out, lcsbp);
    s->ptrs[ref]->ReleaseBitMasks();
}

// Multi-threaded triangle rows [row_begin,row_end) with the reference's default transform
// (float indel075_div_lcs, the UPGMA shape, UPGMA.cpp:75-109).  Returns wall seconds; *n_pairs is
// the number of LCS lengths produced.  If out_lcs != nullptr, raw LCS lengths are stored packed
// (row i at i(i-1)/2 - row_begin(row_begin-1)/2) instead of being transformed.
double ref_lcs_triangle_mt(void* h, uint32_t row_begin, uint32_t row_end, int n_threads, int isa,
                           uint32_t* out_lcs, uint64_t* n_pairs)
{
    auto* s = static_cast<SeqSet*>(h);
    std::atomic<int64_t> next((int64_t)row_end - 1);      // big rows first, like CUPGMAQueue
    std::atomic<uint64_t> pairs(0);
    const size_t base = (size_t)row_begin * (row_begin ? row_begin - 1 : 0) / 2;
    // every worker needs its own copy of the row sequence state? No: ComputeBitMasks mutates the
    // row CSequence only, and each row is owned by exactly one worker at a time.
    auto t0 = std::chrono::steady_clock::now();
    std::vector<std::thread> workers;
    for (int t = 0; t < n_threads; ++t)
        workers.emplace_back([&] {
            DriverOnly drv(isa_from_int(isa));
            CLCSBP lcsbp(isa_from_int(isa));
            Transform<float, Distance::indel075_div_lcs> tr;
            RawLcs raw;
            std::vector<float> row(row_end ? row_end : 1);
            uint64_t mine = 0;
            for (;;) {
                int64_t i = next.fetch_sub(1);
                if (i < (int64_t)row_begin) break;
                if (out_lcs) {
                    size_t off = (size_t)i * (i ? i - 1 : 0) / 2 - base;
                    drv.calculateDistanceVector<CSequence*, uint32_t, RawLcs>(
                        raw, s->ptrs[i], s->ptrs.data(), (int)i, out_lcs + off, lcsbp);
                } else {
                    drv.calculateDistanceVector<CSequence*, float, decltype(tr)>(
                        tr, s->ptrs[i], s->ptrs.data(), (int)i, row.data(), lcsbp);
                }
                mine += (uint64_t)i;
            }
            pairs += mine;
        });
    for (auto& w : workers) w.join();
    double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    if (n_pairs) *n_pairs = pairs.load();
    return sec;
}

// ---------------------------------------------------------------- guide tree consumers of HP-1
// (a) the reference's UPGMA end to end on the set (its own CLCSBP distances);
// (b) the reference's UPGMA agglomeration (UPGMA<>::computeTree, UPGMA.cpp:114-295) on an EXTERNAL float
//     distance triangle -- used to show that GPU LCS lengths + the host Transform reproduce the same tree.
// out_pairs receives (left, right) for all 2n-1 nodes of tree_structure (leaves are -1, -1).
void ref_upgma_tree(void* h, int modified, int n_threads, int* out_pairs)
{
    auto* s = static_cast<SeqSet*>(h);
    UPGMA<Distance::indel075_div_lcs> gen(n_threads, instruction_set_t::avx2, modified != 0);
    tree_structure tree;
    gen(s->ptrs, tree);
    for (size_t i = 0; i < tree.size(); ++i) { out_pairs[2 * i] = tree[i].first; out_pairs[2 * i + 1] = tree[i].second; }
}

void ref_upgma_tree_from_distances(const float* tri, int n, int modified, int* out_pairs)
{
    UPGMA<Distance::indel075_div_lcs> gen(1, instruction_set_t::avx2, modified != 0);
    std::vector<float> d(tri, tri + (size_t)n * (n - 1) / 2);
    tree_structure tree;
    tree.resize(n, std::make_pair<int, int>(-1, -1));
    if (modified) gen.computeTree<true>(d.data(), n, tree);
    else gen.computeTree<false>(d.data(), n, tree);
    for (size_t i = 0; i < tree.size(); ++i) { out_pairs[2 * i] = tree[i].first; out_pairs[2 * i + 1] = tree[i].second; }
}

// (c) the reference's default guide tree: MSTPrim<indel075_div_lcs> end to end (MSTPrim.cpp:280-549 + 784-833)
void ref_mst_prim_tree(void* h, int n_threads, int* out_pairs)
{
    auto* s = static_cast<SeqSet*>(h);
    PrimRef gen(n_threads, instruction_set_t::avx2);
    tree_structure tree;
    gen(s->ptrs, tree);
    for (size_t i = 0; i < tree.size(); ++i) { out_pairs[2 * i] = tree[i].first; out_pairs[2 * i + 1] = tree[i].second; }
}

// (d) the reference's own mst_to_dendogram (MSTPrim.cpp:784-833) on EXTERNAL MST edges given in Prim order:
// edge k (k = 0..n-2) joins from[k] < to[k] at distance dist[k] and was found when the (k+1)-th vertex was added;
// prim_orders[i] = position of sequence i in the Prim visiting order.
void ref_mst_to_dendogram(int n, const int* from, const int* to, const double* dist, const int* prim_orders, int* out_pairs)
{
    PrimRef gen(1, instruction_set_t::avx2);
    auto pmf = stolen_mst_to_dendogram();
    typename DendTraits<decltype(pmf)>::edges_t edges;
    edges.reserve(n);
    for (int k = 0; k + 1 < n; ++k) edges.emplace_back(from[k], to[k], k + 1, -dist[k]);   // negated: MSTPrim.cpp:384
    std::vector<int> orders(prim_orders, prim_orders + n);
    tree_structure tree;
    tree.resize(n, std::make_pair<int, int>(-1, -1));
    (gen.*pmf)(edges, orders, tree);
    for (size_t i = 0; i < tree.size(); ++i) { out_pairs[2 * i] = tree[i].first; out_pairs[2 * i + 1] = tree[i].second; }
}

// The reference's own Transform functors.  kind: 0 indel075_div_lcs, 1 indel_div_lcs, 2 pairwise_identity.
double ref_transform_f64(int kind, uint32_t lcs, uint32_t len1, uint32_t len2)
{
    if (kind == 0) { Transform<double, Distance::indel075_div_lcs> t; return t(lcs, len1, len2); }
    if (kind == 1) { Transform<double, Distance::indel_div_lcs> t; return t(lcs, len1, len2); }
    Transform<double, Distance::pairwise_identity> t; return t(lcs, len1, len2);
}
float ref_transform_f32(int kind, uint32_t lcs, uint32_t len1, uint32_t len2)
{
    if (kind == 0) { Transform<float, Distance::indel075_div_lcs> t; return t(lcs, len1, len2); }
    if (kind == 1) { Transform<float, Distance::indel_div_lcs> t; return t(lcs, len1, len2); }
    Transform<float, Distance::pairwise_identity> t; return t(lcs, len1, len2);
}

// ---------------------------------------------------------------- HP-2: profile alignment
// A DP session owns a CParams prepared exactly as CFAMSA does before ComputeAlignment:
//   score matrix  = round(matrix * cost_cast_factor)         (msa.cpp:59-80, initScoreMatrix)
//   gap costs     = CParams defaults, rescaled by 1 + log2(n/45)/7 when n >= 45 (msa.cpp:83-106)
// (those two small routines live in msa.cpp, which drags in the I/O libraries; their arithmetic is
// restated here in the harness -- the DP itself is the reference's own object code).
struct DpSession {
    CParams params;
    std::unique_ptr<refresh::active_thread_pool_v2> atp;
};

void* ref_dp_create(int n_seqs_for_rescale, int matrix_type, int pool_threads)
{
    auto* s = new DpSession();
    CParams& P = s->params;
    P.matrix_type = (ScoringMatrices::matrix_type_t)matrix_type;   // 0 MIQS, 1 PFASUM31, 2 PFASUM43 (default), 3 PFASUM60
    auto& sm = ScoringMatrices::get_matrix(P.matrix_type);
    P.score_matrix.assign(NO_AMINOACIDS, std::vector<score_t>());
    P.score_vector.clear();
    for (int i = 0; i < NO_AMINOACIDS; ++i) {
        P.score_vector.emplace_back((score_t)round(sm[i][i] * cost_cast_factor));
        for (int j = 0; j < NO_AMINOACIDS; ++j)
            P.score_matrix[i].emplace_back((score_t)round(sm[i][j] * cost_cast_factor));
    }
    if (n_seqs_for_rescale > 0 && P.enable_gap_rescaling) {
        double gap_scaler = log2(n_seqs_for_rescale / (double)P.scaler_log);
        if (n_seqs_for_rescale < (int)P.scaler_log) gap_scaler = 1.0;
        else gap_scaler = 1.0 + (gap_scaler / P.scaler_div);
        P.gap_ext = (score_t)(P.gap_ext * gap_scaler);
        P.gap_open = (score_t)(P.gap_open * gap_scaler);
        P.gap_term_ext = (score_t)(P.gap_term_ext * gap_scaler);
        P.gap_term_open = (score_t)(P.gap_term_open * gap_scaler);
    }
    P.instruction_set = instruction_set_t::avx2;
    P.n_threads = pool_threads;
    s->atp.reset(new refresh::active_thread_pool_v2(pool_threads, pool_threads));
    return s;
}
void ref_dp_destroy(void* h) { delete static_cast<DpSession*>(h); }

// out4 = {gap_open, gap_ext, gap_term_open, gap_term_ext}
void ref_dp_gaps(void* h, int64_t* out4)
{
    CParams& P = static_cast<DpSession*>(h)->params;
    out4[0] = P.gap_open; out4[1] = P.gap_ext; out4[2] = P.gap_term_open; out4[3] = P.gap_term_ext;
}
void ref_dp_set_gaps(void* h, const int64_t* in4)
{
    CParams& P = static_cast<DpSession*>(h)->params;
    P.gap_open = in4[0]; P.gap_ext = in4[1]; P.gap_term_open = in4[2]; P.gap_term_ext = in4[3];
}
void ref_dp_score_matrix(void* h, int64_t* out24x24)
{
    CParams& P = static_cast<DpSession*>(h)->params;
    for (int i = 0; i < 24; ++i)
        for (int j = 0; j < 24; ++j) out24x24[i * 24 + j] = P.score_matrix[i][j];
}

// profile from already-aligned (gapped) strings: AppendRawSequence + CalculateCountersScores,
// the way CFAMSA::alignProfiles does (msa.cpp:680-689); one ungapped string = a leaf profile.
void* ref_profile_create(void* h, const char* const* gapped, const int* seq_nos, uint32_t n)
{
    auto* s = static_cast<DpSession*>(h);
    auto* p = new CProfile(&s->params, s->atp.get());
    for (uint32_t i = 0; i < n; ++i) {
        CGappedSequence gs("s" + std::to_string(seq_nos[i]), std::string(gapped[i]), seq_nos[i], nullptr);
        p->AppendRawSequence(gs);
    }
    p->CalculateCountersScores();
    return p;
}
// leaf profile as the main flow builds it: CSequence -> CGappedSequence(CSequence&&) (msa.cpp:595)
// -> new CProfile(*gs, &params) (msa.cpp:391).  `letters` is the ungapped residue string.
void* ref_profile_leaf(void* h, const char* letters, int seq_no)
{
    auto* s = static_cast<DpSession*>(h);
    CSequence seq("s" + std::to_string(seq_no), std::string(letters), seq_no, nullptr);
    CGappedSequence gs(std::move(seq));
    return new CProfile(gs, &s->params);
}
void ref_profile_destroy(void* p) { delete static_cast<CProfile*>(p); }
uint32_t ref_profile_width(void* p) { return (uint32_t)static_cast<CProfile*>(p)->width; }
uint32_t ref_profile_card(void* p) { return (uint32_t)static_cast<CProfile*>(p)->data.size(); }
int64_t ref_profile_total_score(void* p) { return static_cast<CProfile*>(p)->total_score; }

// scores: (width+1) x 32 int64, counters: (width+1) x 32 int32, column-major as in CProfileValues
void ref_profile_tables(void* p, int64_t* scores, int32_t* counters)
{
    auto* q = static_cast<CProfile*>(p);
    for (size_t c = 0; c <= q->width; ++c)
        for (size_t r = 0; r < NO_SYMBOLS; ++r) {
            scores[c * NO_SYMBOLS + r] = q->scores.get_value(c, r);
            counters[c * NO_SYMBOLS + r] = q->counters.get_value(c, r);
        }
}

// overwrites the profile's scores ((width+1) x 32 int64, layout as ref_profile_tables), counters untouched: CProfile::Align
// reads the stored table, so crafted scores steer its path while ConstructProfile still works on the real counters
void ref_profile_set_scores(void* p, const int64_t* scores)
{
    auto* q = static_cast<CProfile*>(p);
    for (size_t c = 0; c <= q->width; ++c)
        for (size_t r = 0; r < NO_SYMBOLS; ++r) q->scores.set_value(c, r, scores[c * NO_SYMBOLS + r]);
}

// gapped row i of the profile (width characters + NUL) and its sequence number
int ref_profile_row(void* p, uint32_t i, char* out)
{
    // CGappedSequence::Decode() rewrites symbols[] in place (sequence.cpp:430-437), so the row is
    // rendered here without touching the object: n_gaps[0] gaps, then symbol k followed by n_gaps[k].
    static const char* letters = "ARNDCQEGHILKMFPSTWYVBZX*";
    auto* q = static_cast<CProfile*>(p);
    CGappedSequence* gs = q->data[i];
    size_t at = 0;
    for (uint32_t g = 0; g < gs->n_gaps[0]; ++g) out[at++] = '-';
    for (size_t k = 1; k <= gs->size; ++k) {
        const int c = gs->symbols[k];
        out[at++] = (c >= 0 && c < 24) ? letters[c] : '?';
        for (uint32_t g = 0; g < gs->n_gaps[k]; ++g) out[at++] = '-';
    }
    out[at] = 0;
    return gs->sequence_no;
}

// new CProfile(p1, p2, params, no_threads, 4, atp): CProfile::Align + ConstructProfile.  The children
// are consumed (their rows move into the result) exactly as in ComputeAlignment (msa.cpp:404-407);
// the caller still has to ref_profile_destroy() them.
void* ref_profile_align(void* h, void* p1, void* p2, int no_threads)
{
    auto* s = static_cast<DpSession*>(h);
    return new CProfile(static_cast<CProfile*>(p1), static_cast<CProfile*>(p2), &s->params,
                        (uint32_t)no_threads, 4, s->atp.get());
}

// The host half of a merge driven from OUTSIDE: the reference's own, unmodified ConstructProfile
// (profile.cpp:694-1002) run on a CDPMatrix whose bytes were produced elsewhere (by the GPU in
// tests/test_dp_gpu.py::test_gpu_driven_progressive_alignment), with `last` = (D,H,V) at the corner.
// swapped != 0 means the DP's row profile is p2 (what CProfile::Align decides at profile.cpp:254-304).
// Children are consumed like in ref_profile_align; the caller frees them.
void* ref_profile_construct(void* h, void* p1, void* p2, const uint8_t* dirs, const int64_t* last, int swapped)
{
    auto* s = static_cast<DpSession*>(h);
    auto* a = static_cast<CProfile*>(p1);
    auto* b = static_cast<CProfile*>(p2);
    CProfile* R = swapped ? b : a;
    CProfile* C = swapped ? a : b;
    CProfile* m = new CProfile(&s->params, s->atp.get());
    CDPMatrix matrix(R->width + 1, C->width + 1);
    memcpy(matrix.get_row(0), dirs, (R->width + 1) * (C->width + 1));
    auto pmf = stolen_construct_profile();
    typename ConstructTraits<decltype(pmf)>::elem_t le(last[0], last[1], last[2]);
    (m->*pmf)(R, C, matrix, le, 1u);
    return m;
}

// Times n independent merges on n_threads host threads (one merge per task, each merge sequential:
// CProfile::Align with no_threads = 1 + ConstructProfile, as ComputeAlignment's workers run them,
// msa.cpp:375-426).  The children are consumed and freed.  Returns wall seconds; *cells = sum W1*W2.
double ref_dp_align_pairs_mt(void* h, void** p1s, void** p2s, uint32_t n, int n_threads, uint64_t* cells)
{
    auto* s = static_cast<DpSession*>(h);
    uint64_t c = 0;
    for (uint32_t k = 0; k < n; ++k)
        c += (uint64_t)static_cast<CProfile*>(p1s[k])->width * static_cast<CProfile*>(p2s[k])->width;
    if (cells) *cells = c;
    std::atomic<uint32_t> next(0);
    auto t0 = std::chrono::steady_clock::now();
    std::vector<std::thread> workers;
    for (int t = 0; t < n_threads; ++t)
        workers.emplace_back([&] {
            refresh::active_thread_pool_v2 atp(1, 1);
            for (;;) {
                uint32_t k = next.fetch_add(1);
                if (k >= n) break;
                auto* a = static_cast<CProfile*>(p1s[k]);
                auto* b = static_cast<CProfile*>(p2s[k]);
                CProfile* m = new CProfile(a, b, &s->params, 1, 4, &atp);
                delete a; delete b; delete m;
            }
        });
    for (auto& w : workers) w.join();
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

// The whole progressive alignment the way CFAMSA::ComputeAlignment runs it (msa.cpp:360-438): n_threads workers take
// tasks from the reference's own CProfileQueue (queues.cpp: deepest ready node first, leaves included) and build
// `new CProfile(gs, params)` for a leaf or `new CProfile(p1, p2, params, no_threads, no_rows_per_box, atp)` for an
// internal node (internal refinement is off: thr_internal_refinement = 0, and the sets timed here are above
// thr_refinement).  The worker loop below restates msa.cpp:375-426 because msa.cpp itself drags in the I/O libraries;
// queue, profiles and DP are the reference's object code.  tree: (2n-1) x 2 child ids, leaves (-1, -1).
// Returns wall seconds (= the reference's time.alignment); *cells = sum of W1*W2 over the merges, *total / *width = total
// score and width of the final profile, rows_out (optional, n x (width+1) bytes, row i = sequence number i).
double ref_align_tree_mt(void* h, const char* const* letters, uint32_t n, const int* tree, int n_threads, uint64_t* cells,
                         int64_t* total, uint32_t* width, char* rows_out, uint32_t rows_stride)
{
    auto* s = static_cast<DpSession*>(h);
    CParams params = s->params;
    params.n_threads = (uint32_t)n_threads;
    refresh::active_thread_pool_v2 atp(n_threads, n_threads);
    std::vector<CGappedSequence*> gapped;
    for (uint32_t i = 0; i < n; ++i) {
        CSequence seq("s" + std::to_string(i), std::string(letters[i]), (int)i, nullptr);
        gapped.push_back(new CGappedSequence(std::move(seq)));
    }
    tree_structure guide_tree;
    for (uint32_t i = 0; i < 2 * n - 1; ++i) guide_tree.emplace_back(tree[2 * i], tree[2 * i + 1]);
    std::map<size_t, CProfile*> profiles;
    std::atomic<uint64_t> c(0);
    auto t0 = std::chrono::steady_clock::now();
    {
        CProfileQueue pq(&gapped, &profiles, &guide_tree, (uint32_t)n_threads);
        std::vector<std::thread> workers;
        for (int t = 0; t < n_threads; ++t)
            workers.emplace_back([&] {
                CGappedSequence* gs;
                CProfile *prof1, *prof2, *prof_sol;
                size_t prof_id;
                uint32_t no_threads, no_rows_per_box;
                while (pq.GetTask(prof_id, gs, prof1, prof2, no_threads, no_rows_per_box)) {
                    if (gs != nullptr)
                        prof_sol = new CProfile(*gs, &params);
                    else {
                        c += (uint64_t)prof1->width * prof2->width;
                        prof_sol = new CProfile(prof1, prof2, &params, no_threads, no_rows_per_box, &atp);
                        delete prof1;
                        delete prof2;
                    }
                    pq.AddSolution(prof_id, prof_sol);
                }
            });
        for (auto& w : workers) w.join();
    }
    const double sec = std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    CProfile* root = profiles.begin()->second;
    if (cells) *cells = c.load();
    if (total) *total = root->total_score;
    if (width) *width = (uint32_t)root->width;
    if (rows_out)
        for (uint32_t i = 0; i < root->data.size(); ++i) {
            std::vector<char> buf(root->width + 2);
            const int no = ref_profile_row(root, i, buf.data());
            if ((size_t)root->width + 1 <= rows_stride) memcpy(rows_out + (size_t)no * rows_stride, buf.data(), root->width + 1);
        }
    delete root;
    for (auto* g : gapped) delete g;
    return sec;
}

} // extern "C"
