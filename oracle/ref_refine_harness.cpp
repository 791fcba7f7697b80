// oracle/ref_refine_harness.cpp -- the reference's refinement for the tests of famsa_prof_refine.  TEST INFRASTRUCTURE ONLY.
//
// Linked against _ref/libfamsa_ref.so (oracle/Makefile), which holds the UNMODIFIED reference's CProfile
// (src/core/profile.cpp: Condense, OptimizeGaps, CalculateCountersScores, CalculateTotalScore, Align) and CGappedSequence.
// CFAMSA::RefineAlignment itself lives in src/msa_refinement.cpp, whose class drags in msa.cpp and the I/O libraries
// (unbuildable here, DESIGN.md §2), so its loop (msa_refinement.cpp:7-66, 113-209) is restated below, line by line, on the
// reference's own objects.  The progressive alignment before it is the reference's CProfile(p1, p2, ...) along the given
// tree, as in ComputeAlignment (msa.cpp:375-426).
#include <algorithm>
#include <array>
#include <condition_variable>
#include <cstdint>
#include <cstring>
#include <functional>
#include <future>
#include <iostream>
#include <list>
#include <map>
#include <memory>
#include <mutex>
#include <queue>
#include <random>
#include <set>
#include <sstream>
#include <string>
#include <thread>
#include <vector>

#define private public      // harness TU only: read CProfile internals, nothing is modified
#define protected public
#include "core/defs.h"
#include "core/params.h"
#include "core/profile.h"
#include "core/sequence.h"
#undef private
#undef protected

namespace {

struct Session {
    CParams params;
    std::unique_ptr<refresh::active_thread_pool_v2> atp;
    uint32_t no_threads = 2;
};

void render(const CGappedSequence* gs, char* out)
{
    static const char* letters = "ARNDCQEGHILKMFPSTWYVBZX*";
    size_t at = 0;
    for (uint32_t g = 0; g < gs->n_gaps[0]; ++g) out[at++] = '-';
    for (size_t k = 1; k <= gs->size; ++k) {
        const int c = gs->symbols[k];
        out[at++] = (c >= 0 && c < 24) ? letters[c] : '?';
        for (uint32_t g = 0; g < gs->n_gaps[k]; ++g) out[at++] = '-';
    }
    out[at] = 0;
}

CProfile* from_rows(Session* s, const char* const* rows, uint32_t n, const char* const* ids = nullptr)
{
    auto* p = new CProfile(&s->params, s->atp.get());
    for (uint32_t i = 0; i < n; ++i) {
        CGappedSequence gs(ids ? std::string(ids[i]) : "s" + std::to_string(i), std::string(rows[i]), (int)i, nullptr);
        p->AppendRawSequence(gs);
    }
    // AppendRawSequence takes width = gapped_size - 1 for a row that starts with GUARD (profile.cpp:334-337), one short
    // for a row built from a string; Condense, which the refinement calls first, resets it to gapped_size (:387, :427)
    p->width = p->data.front()->gapped_size;
    p->CalculateCountersScores();
    return p;
}

// msa_refinement.cpp:7-18
void refine_random(std::mt19937& rnd, CProfile* p, std::vector<size_t>& dest)
{
    for (size_t i = 0; i < p->data.size(); ++i) dest.emplace_back(rnd() % 2);
    if (std::count(dest.begin(), dest.end(), 0) == 0 || std::count(dest.begin(), dest.end(), 1) == 0) {
        size_t id = rnd() % dest.size();
        dest[id] = !dest[id];
    }
}

// msa_refinement.cpp:21-66; returns the column picked (0: RefineRandom)
size_t refine_column(std::mt19937& rnd, CProfile* p, std::vector<size_t>& dest, std::vector<size_t>& gap_stats, bool valid)
{
    size_t size = p->data.front()->gapped_size;
    size_t card = p->data.size();
    dest.clear();
    if (!valid) p->GetGapStats(gap_stats);
    std::vector<std::pair<size_t, size_t>> tmp;
    for (size_t i = 1; i <= size; ++i) {
        int x = (int)std::min(gap_stats[i], card - gap_stats[i]);
        if (x > 0) tmp.emplace_back(i, x);
    }
    std::stable_sort(tmp.begin(), tmp.end(), [](const std::pair<size_t, size_t>& x, const std::pair<size_t, size_t>& y) {
        return x.second != y.second ? x.second < y.second : x.first < y.first;
    });
    if (tmp.empty()) { refine_random(rnd, p, dest); return 0; }
    size_t col_id = tmp[rnd() % tmp.size()].first;
    int first_prof_id = 0, second_prof_id = 1;
    if (p->data[0]->GetSymbol(col_id) == GAP) std::swap(first_prof_id, second_prof_id);
    for (size_t j = 0; j < card; ++j)
        dest.emplace_back(p->data[j]->GetSymbol(col_id) == GAP ? first_prof_id : second_prof_id);
    return col_id;
}

// RefineAlignment (msa_refinement.cpp:77, 84-92, 113-209) on profile_to_refine, which it consumes: the refined rows by
// sequence number into `refined`, the refined width, totals = {prev_total_score of :114, final total_score}, counts =
// {i_ref, i_succ_ref, n_ref_succ, identical}; trace: per try {i_ref, column (0: RefineRandom), FNV-1a of the split,
// identical, accepted, total}, at most max_trace tries; scores / counters: the final CProfile's tables ((width+1) x 32).
// Rows and tables are written only when the refined width is below stride.
void refine_loop(Session* s, CProfile* profile_to_refine, uint32_t n_refinements, char* refined, uint32_t stride, uint32_t* width,
                 int64_t* totals, uint32_t* counts, int64_t* trace, uint32_t max_trace, int64_t* scores, int32_t* counters)
{
    CParams* params = &s->params;
    // msa_refinement.cpp:77, 84-92
    std::mt19937 rnd_rfn;
    rnd_rfn.seed(5489u);
    size_t n_ref = n_refinements;
    size_t n_seq = profile_to_refine->Size();
    std::vector<size_t> gap_stats;
    if (n_ref > 2 * n_seq) n_ref = 2 * n_seq;
    if (n_ref > 0 && n_ref < 100 && n_seq < 100) n_ref = 100;
    // :113-209
    int n_ref_succ = 0, identical = 0;
    score_t prev_total_score = profile_to_refine->CalculateTotalScore();
    totals[0] = prev_total_score;
    std::sort(profile_to_refine->data.begin(), profile_to_refine->data.end(), [](CGappedSequence* p, CGappedSequence* q) { return p->id < q->id; });
    std::vector<size_t> dest_prof_id;
    std::vector<std::vector<size_t>> old_dest_prof_ids;
    std::vector<int> column_mapping1, column_mapping2;
    size_t i_ref, i_succ_ref;
    bool valid_gap_stats = false;
    for (i_ref = i_succ_ref = 0; i_succ_ref < n_ref && i_ref < 20 * n_ref; ++i_ref) {
        CProfile profile1(params, s->atp.get()), profile2(params, s->atp.get());
        const size_t col = refine_column(rnd_rfn, profile_to_refine, dest_prof_id, gap_stats, valid_gap_stats);
        valid_gap_stats = true;
        uint32_t hash = 2166136261u;
        for (size_t d : dest_prof_id) hash = (hash ^ (uint32_t)d) * 16777619u;
        int64_t* tr = i_ref < max_trace ? trace + 6 * i_ref : nullptr;
        if (tr) { tr[0] = (int64_t)i_ref; tr[1] = (int64_t)col; tr[2] = hash; tr[3] = -1; tr[4] = 0; tr[5] = 0; }
        if (std::find(old_dest_prof_ids.begin(), old_dest_prof_ids.end(), dest_prof_id) != old_dest_prof_ids.end()) continue;
        for (size_t i = 0; i < profile_to_refine->data.size(); ++i)
            if (dest_prof_id[i]) profile1.AppendRawSequence(*profile_to_refine->data[i]);
            else profile2.AppendRawSequence(*profile_to_refine->data[i]);
        profile1.Condense(column_mapping1);
        profile2.Condense(column_mapping2);
        profile1.OptimizeGaps();
        profile2.OptimizeGaps();
        CProfile* prof = new CProfile(params, s->atp.get());
        prof->Align(&profile1, &profile2, s->no_threads, 4, &column_mapping1, &column_mapping2);
        std::sort(prof->data.begin(), prof->data.end(), [](CGappedSequence* p, CGappedSequence* q) { return p->id < q->id; });
        const bool same = *prof == *profile_to_refine;
        if (tr) tr[3] = same;
        if (!same) {
            prof->CalculateTotalScore();
            if (tr) tr[5] = prof->total_score;
            if (prof->total_score >= prev_total_score) {
                prev_total_score = prof->total_score;
                std::swap(profile_to_refine, prof);
                ++n_ref_succ;
                old_dest_prof_ids.clear();
                valid_gap_stats = false;
                if (tr) tr[4] = 1;
            }
        } else
            ++identical;
        delete prof;
        old_dest_prof_ids.emplace_back(dest_prof_id);
        i_succ_ref++;
    }
    *width = (uint32_t)profile_to_refine->width;
    totals[1] = prev_total_score;
    counts[0] = (uint32_t)i_ref; counts[1] = (uint32_t)i_succ_ref; counts[2] = (uint32_t)n_ref_succ; counts[3] = (uint32_t)identical;
    if (profile_to_refine->width >= stride) { delete profile_to_refine; return; }   // no room: the caller sees *width >= stride
    for (auto* gs : profile_to_refine->data) render(gs, refined + (size_t)gs->sequence_no * stride);
    for (size_t c = 0; c <= profile_to_refine->width; ++c)         // the final profile's tables, (width+1) x 32 each
        for (size_t r = 0; r < NO_SYMBOLS; ++r) {
            scores[c * NO_SYMBOLS + r] = profile_to_refine->scores.get_value(c, r);
            counters[c * NO_SYMBOLS + r] = profile_to_refine->counters.get_value(c, r);
        }
    delete profile_to_refine;
}

} // namespace

extern "C" {

// sm: 24 x 24 scores, gaps = {open, ext, term_open, term_ext}; flags as famsa_prof_refine's (1: -dgo, 2: -dsp);
// no_threads: what RefineAlignment passes to Align (> 1: the unbanded ParAlign* paths)
void* rr_create(const int64_t* sm, const int64_t* gaps, int flags, int no_threads)
{
    auto* s = new Session();
    CParams& P = s->params;
    P.score_matrix.assign(NO_AMINOACIDS, std::vector<score_t>());
    P.score_vector.clear();
    for (int i = 0; i < NO_AMINOACIDS; ++i) {
        P.score_vector.push_back(sm[i * 24 + i]);
        for (int j = 0; j < NO_AMINOACIDS; ++j) P.score_matrix[i].push_back(sm[i * 24 + j]);
    }
    P.gap_open = gaps[0]; P.gap_ext = gaps[1]; P.gap_term_open = gaps[2]; P.gap_term_ext = gaps[3];
    P.enable_gap_optimization = !(flags & 1);
    P.enable_total_score_calculation = !(flags & 2);
    P.instruction_set = instruction_set_t::avx2;
    P.n_threads = no_threads;
    s->no_threads = (uint32_t)no_threads;
    s->atp.reset(new refresh::active_thread_pool_v2(no_threads, no_threads));
    return s;
}
void rr_destroy(void* h) { delete static_cast<Session*>(h); }

// CalculateTotalScore of the profile whose rows are given (counters from CalculateCountersScores)
int64_t rr_total_score(void* h, const char* const* rows, uint32_t n)
{
    CProfile* p = from_rows(static_cast<Session*>(h), rows, n);
    const int64_t t = p->CalculateTotalScore();
    delete p;
    return t;
}

// OptimizeGaps of the rows given; out: n x (width + 1) characters, NUL-terminated rows
void rr_optimize_gaps(void* h, const char* const* rows, uint32_t n, char* out)
{
    CProfile* p = from_rows(static_cast<Session*>(h), rows, n);
    p->OptimizeGaps();
    const size_t stride = p->width + 1;
    for (uint32_t i = 0; i < n; ++i) render(p->data[i], out + i * stride);
    delete p;
}

// The progressive alignment of `letters` (FASTA ids `ids`) along `merges` ((n-1) x 2 node ids, leaves 0..n-1, node n+k = merge k), then
// RefineAlignment on its root.  Rows come out by sequence number, `stride` bytes each (NUL-terminated).
// widths = {unrefined, refined}, totals = {prev_total_score of :114, final total_score}, counts = {i_ref, i_succ_ref,
// n_ref_succ, identical}; trace: per try {i_ref, column (0: RefineRandom), FNV-1a of the split, identical, accepted,
// total}, at most max_trace tries; scores / counters: the final CProfile's tables ((width+1) x 32, room for stride
// columns).
void rr_align_refine(void* h, const char* const* letters, const char* const* ids, uint32_t n, const int* merges, uint32_t n_refinements,
                     char* unrefined, char* refined, uint32_t stride, uint32_t* widths, int64_t* totals, uint32_t* counts, int64_t* trace,
                     uint32_t max_trace, int64_t* scores, int32_t* counters)
{
    auto* s = static_cast<Session*>(h);
    CParams* params = &s->params;
    std::vector<CProfile*> node(2 * n - 1, nullptr);
    for (uint32_t i = 0; i < n; ++i) {
        CSequence seq(ids[i], std::string(letters[i]), (int)i, nullptr);
        CGappedSequence gs(std::move(seq));
        node[i] = new CProfile(gs, params);
    }
    for (uint32_t k = 0; k + 1 < n; ++k) {
        CProfile *a = node[merges[2 * k]], *b = node[merges[2 * k + 1]];
        node[n + k] = new CProfile(a, b, params, 1, 4, s->atp.get());
        delete a; delete b;
    }
    CProfile* profile_to_refine = node[2 * n - 2];
    widths[0] = (uint32_t)profile_to_refine->width;
    for (auto* gs : profile_to_refine->data) render(gs, unrefined + (size_t)gs->sequence_no * stride);
    refine_loop(s, profile_to_refine, n_refinements, refined, stride, widths + 1, totals, counts, trace, max_trace, scores, counters);
}

// RefineAlignment of the alignment given as n NUL-terminated rows of letters ('-': gap) with FASTA ids `ids` (sequence
// number = index), built as rr_total_score builds it; outputs as rr_align_refine's, widths[0] = the input's width.
void rr_refine_rows(void* h, const char* const* rows, const char* const* ids, uint32_t n, uint32_t n_refinements, char* refined,
                    uint32_t stride, uint32_t* widths, int64_t* totals, uint32_t* counts, int64_t* trace, uint32_t max_trace,
                    int64_t* scores, int32_t* counters)
{
    auto* s = static_cast<Session*>(h);
    CProfile* p = from_rows(s, rows, n, ids);
    widths[0] = (uint32_t)p->width;
    refine_loop(s, p, n_refinements, refined, stride, widths + 1, totals, counts, trace, max_trace, scores, counters);
}

} // extern "C"
