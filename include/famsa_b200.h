/*
 * famsa_b200.h -- C ABI of libfamsa_b200.so, the H100 (sm_90a) replacement for FAMSA's two
 * data-parallel hot paths.  Plain pointers and sizes only; no C++ or torch types.
 *
 * Every entry point names the reference interface it replaces (paths relative to the FAMSA
 * source tree, v2.5.0).  INTEGRATION.md shows the C++ shims a FAMSA maintainer would add so that
 * src/tree/ *, src/msa.cpp and src/msa_refinement.cpp compile and run unchanged on top of this.
 *
 * Conventions
 *   - All functions return 0 on success and a non-zero FAMSA_E_* code on failure;
 *     famsa_last_error() returns a human-readable message for the calling thread's last failure
 *     (the reference has no status codes: errors are std::runtime_error caught in main(),
 *     src/famsa.cpp:160-165 -- the C++ shim rethrows the message).
 *   - There is NO CPU fallback: without an sm_90 (H100) device every compute entry point fails.
 *   - A context is bound to one device.  Calls on one context are serialised internally, so the
 *     reference's concurrent per-thread CLCSBP instances may share one context.
 *   - Residue codes are the reference's: 0..23 = "ARNDCQEGHILKMFPSTWYVBZX*" (src/core/sequence.cpp:17),
 *     22 = unknown / padding.  Only codes < 20 can match (sequence.cpp:199).
 */
#ifndef FAMSA_B200_H
#define FAMSA_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FAMSA_B200_ABI_VERSION 1

enum {
    FAMSA_OK = 0,
    FAMSA_E_INVALID = 1,   /* bad argument */
    FAMSA_E_NO_DEVICE = 2, /* no usable CUDA device (there is no CPU fallback) */
    FAMSA_E_CUDA = 3,      /* CUDA runtime / kernel failure */
    FAMSA_E_STATE = 4,     /* call order violated (e.g. LCS before upload) */
    FAMSA_E_NOMEM = 5,
    FAMSA_E_SINK = 6       /* a caller's write callback refused bytes (famsa_dist_export) */
};

typedef struct famsa_ctx famsa_ctx;

/* ------------------------------------------------------------------ context */

int famsa_abi_version(void);

/* device = CUDA ordinal, or -1 for the current device. */
int famsa_create(int device, famsa_ctx** out_ctx);
void famsa_destroy(famsa_ctx* ctx);

/* Message for the last failure on the calling thread ("" if none). Never NULL. */
const char* famsa_last_error(void);

/* Number of kernels this context has launched since creation (bench.py's gpu_launches). */
uint64_t famsa_kernel_launches(const famsa_ctx* ctx);

/* ------------------------------------------------------------------ HP-1: all-pairs LCS length
 *
 * Replaces, per worker thread of every guide-tree builder:
 *   CSequence::ComputeBitMasks                 src/core/sequence.cpp:190-201
 *   MSTPrim::prepare_sequences_view/bit_masks  src/tree/MSTPrim.cpp:554-566, 837-852
 *   CLCSBP::GetLCSBP (4 overloads)             src/lcs/lcsbp.h:38-46, lcsbp.cpp:48-368
 *   CLCSBP_{Classic,AVX,AVX2,AVX512,NEON}      src/lcs/lcsbp_classic.h, src/simd/lcsbp_*_intr.h
 * behind the four batch drivers
 *   AbstractTreeGenerator::calculateDistanceVector / Range / RangeSV / Matrix
 *                                              src/tree/AbstractTreeGenerator.hpp:131,191,288,379
 * Results are the raw LCS lengths (what GetLCSBP writes to `dist`); the LCS -> distance
 * Transform (AbstractTreeGenerator.hpp:28-82) stays on the host so distances are bit-identical.
 * Lengths are bit-exact against the reference, including its dropped-carry corner
 * (lcsbp_classic.h:55-56): which sequence is the row (`seq0`, supplies the bit masks) matters.
 */

/* Upload a sequence set.  Sequence i is codes[offsets[i] .. offsets[i]+lens[i]) (no padding
 * needed).  Replaces any previously uploaded set.  Builds the device-side bit-mask tables. */
int famsa_lcs_upload(famsa_ctx* ctx, const int8_t* codes, const uint64_t* offsets,
                     const uint32_t* lens, uint32_t n_seqs);

/* The same, for a set that is NOT in the order the reference works on (length descending, src/msa.cpp:245-256 -- e.g.
 * -dist_export in input order, DistanceCalculator.cpp:42) and is to be sharded across GPUs: the library applies that order
 * up front (stable: ties keep the caller's order) and every index of the calls that follow -- rows, columns, ids, the layout
 * of the triangle -- is a POSITION IN THAT ORDER.  Row shards are then contiguous runs of the kernel's 32-sequence mask
 * groups and a rank launches only its own tiles (with famsa_lcs_upload on unsorted input a row range cannot select tiles
 * and every rank computes all of them).  famsa_lcs_sorted_order returns sorted_to_caller[position] = caller index
 * (the identity after a plain famsa_lcs_upload); element (i, j) of the caller's order is element (pos[i], pos[j]).  Only
 * the row/column roles of the dropped-carry corner (lcsbp_classic.h:55-56) follow positions instead of caller indices. */
int famsa_lcs_upload_sorted(famsa_ctx* ctx, const int8_t* codes, const uint64_t* offsets, const uint32_t* lens, uint32_t n_seqs);
int famsa_lcs_sorted_order(famsa_ctx* ctx, uint32_t* sorted_to_caller);
/* tiles (32 mask sequences x 64 streamed sequences) launched by the most recent triangle call: the unit of LCS work */
uint64_t famsa_lcs_last_tiles(const famsa_ctx* ctx);

uint32_t famsa_lcs_n_seqs(const famsa_ctx* ctx);

/* Lower triangle, rows [row_begin, row_end): for each row i and each j < i the LCS length with
 * sequence i as the row (seq0).  Layout = TriangleMatrix::access (src/tree/TreeDefs.h:114-119):
 *   out[ i(i-1)/2 - row_begin(row_begin-1)/2 + j ].
 * elem_bytes is 2 (uint16_t, requires every length < 65536) or 4 (uint32_t, the type GetLCSBP
 * writes).  `out` is HOST memory in famsa_lcs_triangle and DEVICE memory in the _device variant;
 * `stream` is a cudaStream_t (NULL = the context's own stream; the call then also synchronises). */
int famsa_lcs_triangle(famsa_ctx* ctx, uint32_t row_begin, uint32_t row_end, void* out,
                       int elem_bytes);
int famsa_lcs_triangle_device(famsa_ctx* ctx, uint32_t row_begin, uint32_t row_end, void* d_out,
                              int elem_bytes, void* stream);

/* The triangle on several GPUs (SURVEY 8e row 1: "rows are sharded, one all-gather at the end"), with the exchange step
 * folded into the computation.  One process per GPU; every rank holds a buffer for the FULL packed triangle of all n_seqs
 * rows (famsa_device_alloc, layout as famsa_lcs_triangle_device writes it for rows 0..n_seqs) and has opened its peers'
 * buffers (famsa_ipc_export -> hand the 64 bytes to the other processes by any means -> famsa_ipc_open).  This call
 * computes rows [row_begin, row_end) into their place of d_full in n_pieces pieces (<= 8, equal numbers of pairs) and, as
 * soon as a piece is finished, copies it into the same place of every d_peer_full[k] over NVLink (copy engines; no SM time,
 * no collective kernel) while the next pieces are being computed.  Work queued on `stream` after the call runs after the
 * last copy has landed; once every rank has got there (any barrier, e.g. a one-element NCCL all-reduce on that stream) all
 * buffers hold the whole triangle.  stream: cudaStream_t or NULL (the context's stream, synchronised). */
int famsa_device_alloc(famsa_ctx* ctx, uint64_t bytes, void** d_ptr);
int famsa_device_free(famsa_ctx* ctx, void* d_ptr);
int famsa_ipc_export(famsa_ctx* ctx, void* d_ptr, uint8_t handle[64]);             /* cudaIpcGetMemHandle */
int famsa_ipc_open(famsa_ctx* ctx, const uint8_t handle[64], void** d_ptr);        /* another process's buffer, mapped here */
int famsa_ipc_close(famsa_ctx* ctx, void* d_ptr);
int famsa_lcs_triangle_exchange(famsa_ctx* ctx, uint32_t row_begin, uint32_t row_end, void* d_full,
                                void* const* d_peer_full, uint32_t n_peers, int elem_bytes, uint32_t n_pieces, void* stream);

/* n_ref reference rows against a column list: out[r * n_col + k] = LCS length with sequence
 * ref_ids[r] as the row (seq0) and sequence col_ids[k] streamed.  col_ids == NULL means columns
 * 0..n_col-1 (calculateDistanceVector's prefix shape).  This is calculateDistanceRange /
 * RangeSV (Prim vertex vs unvisited set, medoid seed vs members) with any number of rows. */
int famsa_lcs_rows(famsa_ctx* ctx, const uint32_t* ref_ids, uint32_t n_ref,
                   const uint32_t* col_ids, uint32_t n_col, void* out, int elem_bytes);
int famsa_lcs_rows_device(famsa_ctx* ctx, const uint32_t* d_ref_ids, uint32_t n_ref,
                          const uint32_t* d_col_ids, uint32_t n_col, void* d_out, int elem_bytes,
                          void* stream);

/* Medoid assignment, the inner loop of the -medoidtree / -parttree heuristic
 * (FastTree<>::makeEvaluation, src/tree/FastTree.cpp:309-324): seed k's row of float distances
 * (calculateDistanceVector with sequences[seed_ids[k]] as the row, Transform<float, distance>) is folded into a
 * running minimum,   if (row_k[j] < best[j]) { best[j] = row_k[j]; assignments[j] = k; }   for k = 0..n_seeds-1
 * (strict <, so the first seed wins ties; starting from seed 0 is what the reference's pre-filled dist_row
 * amounts to).  Computed entirely on the device -- LCS rows, the float Transform (pow table shipped from the
 * host so it is the host libm's), the arg-min -- and only assignments[n_seqs] / min_dist[n_seqs] come back
 * instead of n_seeds x n_seqs distances.  The cost (std::accumulate over min_dist, float, left to right) is
 * left to the caller so that its summation order stays the reference's.  distance_kind as in
 * famsa_transform_f32.  HOST pointers. */
int famsa_lcs_assign(famsa_ctx* ctx, const uint32_t* seed_ids, uint32_t n_seeds, int distance_kind,
                     uint32_t* assignments, float* min_dist);

/* The same assignment sharded across GPUs (SURVEY 8e: "row-vs-all splits the column range G ways"): the context of rank
 * `shard` of `n_shards` -- every rank has uploaded the same set -- answers only for its slice of the sequences (a contiguous
 * run of the 32-sequence mask groups of the length-sorted order, i.e. 1/n_shards of the LCS work) and writes
 *   d_packed[j] = ((int64) float bits of min_dist[j] << 32) | assignments[j]      for its sequences j (caller order),
 *   d_packed[j] = INT64_MAX                                                       for everybody else's,
 * into a DEVICE array of n_seqs int64.  One element-wise MIN all-reduce over the ranks (NCCL) completes it everywhere:
 * distances are >= 0, so the packed values order like (distance, seed index) and ties go to the lowest seed exactly like
 * the strict < of the sequential loop.  stream: cudaStream_t or NULL (the context's stream, synchronised). */
int famsa_lcs_assign_shard(famsa_ctx* ctx, const uint32_t* seed_ids, uint32_t n_seeds, int distance_kind,
                           uint32_t shard, uint32_t n_shards, int64_t* d_packed, void* stream);

/* The default guide tree (-gt sl): the vertex loop of MSTPrim<>::run_view (src/tree/MSTPrim.cpp:280-549) on the
 * device.  Per step: distances from the current vertex (as the row, seq0) to every unvisited sequence through
 * Transform<double, distance>, the relaxation  s = {d, ~ids_to_uint64(v, j)};  if (d <= best[j].first && s < best[j])
 * best[j] = s  (MSTPrim.cpp:492-503), and the election of the unvisited vertex with the smallest pair
 * (:366-386), including the lower-bound skip of :450-467 (a candidate whose distance with LCS = the shorter length
 * cannot beat its current one is not computed: a no-op for true LCS values, decisive in the dropped-carry corner).
 * Because the pair is a strict total order on the edges, the tree is the unique MST under it: the library finds it with
 * parallel Boruvka rounds over a float64 distance triangle and replays Prim's visiting order on the n-1 tree edges
 * (the sequential loop itself runs when a sequence has orientation-dependent LCS values, the dropped-carry corner of
 * lcsbp_classic.h:85-92, or when FAMSA_PRIM_SEQUENTIAL is set).
 * Runs on the LCS triangle kept in HBM, so no n^2 data leaves the device: the n-1 MST edges come back in Prim
 * order -- edge k joins edge_from[k] < edge_to[k] at distance edge_dist[k] (positive; the reference stores the
 * negated value) and was added with the (k+1)-th vertex -- plus prim_order[i], the visiting position of every
 * sequence.  The caller hands them to the unchanged mst_to_dendogram (MSTPrim.cpp:784-833).
 * distance_kind 0 (indel075_div_lcs) or 1 (indel_div_lcs), the two MSTPrim instantiations.  HOST pointers. */
int famsa_lcs_prim(famsa_ctx* ctx, int distance_kind, int32_t* edge_from, int32_t* edge_to, double* edge_dist,
                   int32_t* prim_order);

/* The UPGMA guide tree (-gt upgma / -gt upgma_modified): UPGMA<>::run (src/tree/UPGMA.cpp:39-51) = computeDistances (:75-109, the
 * float Transform of every pair of the triangle) + computeTree<MODIFIED> (:114-295, MUSCLE's nearest-neighbour-cache
 * agglomeration with the plain or the MAFFT-style "modified" average, :24-35), on the LCS triangle kept in HBM: no n^2 data
 * leaves the device, only the n-1 merges return.  tree[2k], tree[2k+1] = children of internal node n_seqs + k (node ids as
 * in tree_structure: leaves 0..n-1 in caller order, which must be the order the reference builds the tree on -- length
 * descending, src/msa.cpp:245-256); the result is the reference's tree pair for pair, including the stale-cache behaviour
 * of its scans.  distance_kind 0 (indel075_div_lcs) or 1 (indel_div_lcs), the two UPGMA instantiations; 2 (pairwise
 * identity, a similarity) is rejected with FAMSA_E_INVALID.  When no live row has a finite cached distance left (e.g. a
 * sequence without a common residue with any other; there the reference would index out of range) the call returns
 * FAMSA_E_INVALID and the context stays usable.  HOST pointer. */
int famsa_lcs_upgma(famsa_ctx* ctx, int distance_kind, int modified, int32_t* tree);
/* Same on a packed LCS triangle that is already in HBM (DEVICE pointer; layout and elem_bytes as famsa_lcs_triangle_device
 * writes it for rows 0..n_seqs) -- e.g. the triangle a multi-GPU run has just all-gathered.  The values are not checked:
 * they must be LCS lengths of the uploaded set (distance kind 0 looks up pow(indel, 0.75) in a table sized by its lengths). */
int famsa_lcs_upgma_from_triangle(famsa_ctx* ctx, int distance_kind, int modified, const void* d_triangle, int elem_bytes,
                                  int32_t* tree);

/* The single-linkage guide tree (-gt slink): SingleLinkage<distance>::run (src/tree/SingleLinkage.cpp:30-189) on the
 * device.  SLINK reads row i (sequence i as the row, seq0) against 0..i-1 through Transform<double, distance> and, with
 * SLINK_HANDLE_TIES (SingleLinkage.h:16-38), orders distances by (distance ascending, ids_to_uint64 descending): the
 * strict total order famsa_lcs_prim uses.  Under a strict order the single-linkage hierarchy is the unique minimum
 * spanning tree merged in Kruskal order, and SLINK's output (stable_sort of lambda, then index[pi[j]] = n + k, :166-188)
 * names each merge by the largest member of its two sides.  So the library finds that MST on the LCS triangle kept in
 * HBM -- with the Boruvka rounds over a float64 distance triangle when it fits beside the LCS triangle, else with the
 * sequential vertex loop (also when FAMSA_PRIM_SEQUENTIAL is set; without MSTPrim's lower-bound skip, which SLINK does
 * not have) -- and labels it on the host.  Only the n-1 merges leave the device.  tree[2k], tree[2k+1] = children of
 * internal node n_seqs + k, leaves 0..n-1 in caller order, which must be FAMSA's length-descending order
 * (src/msa.cpp:245-256) for the reference's tree; the result is that tree pair for pair.  n_seqs = 1 gives no merges
 * (tree may then be NULL).  distance_kind 0 (indel075_div_lcs) or 1 (indel_div_lcs), the two SingleLinkage
 * instantiations.  famsa_lcs_last_timing: n_pairs = the whole triangle.  HOST pointer. */
int famsa_lcs_slink(famsa_ctx* ctx, int distance_kind, int32_t* tree);

/* The neighbour-joining guide tree (-gt nj): NeighborJoining<distance>::run (src/tree/NeighborJoining.cpp:10-21) =
 * calculateDistanceMatrix (the float Transform of the triangle famsa_lcs_upgma reads) + computeTree (:33-118), on the
 * triangle kept in HBM: only the n-1 merges leave the device.  Every step picks the first pair (a, b), a < b in position
 * order, with the smallest q = ((m - 2) D(a,b) - s_a) - s_b (:69, each operation rounded on its own; NaN and values
 * >= FLT_MAX never win), and updates the distances and row sums as :79-113 do.  tree[2k], tree[2k+1] = children of
 * internal node n_seqs + k, leaves 0..n-1 in caller order, which must be FAMSA's length-descending order
 * (src/msa.cpp:245-256) for the reference's tree; the result is that tree pair for pair.  distance_kind 0
 * (indel075_div_lcs) or 1 (indel_div_lcs), the two NeighborJoining instantiations (:124-125); needs at least 2 sequences.
 * A step without any candidate pair (every q NaN or >= FLT_MAX, e.g. four or more sequences no two of which share a
 * residue; the reference would then merge cluster 0 with itself) returns FAMSA_E_INVALID and the context stays usable.
 * FAMSA_E_NOMEM when the LCS triangle, the float triangle and the compaction buffer (1/4 of the float triangle) do not
 * fit.  famsa_lcs_last_timing: n_pairs = the whole triangle.  HOST pointer. */
int famsa_lcs_nj(famsa_ctx* ctx, int distance_kind, int32_t* tree);

/* The distance-matrix export (-dist_export [-square_matrix] [-pid]): DistanceCalculator<distance>::run
 * (src/tree/DistanceCalculator.cpp:10-122) with its text formatting, num2str / NumericConversions::Double2PChar
 * (src/utils/conversion.h:52-119), on the device.  Works on the set of the last famsa_lcs_upload, in the caller's
 * order (the reference exports in input order: no sorting, no duplicate removal, msa.cpp:518-526); after
 * famsa_lcs_upload_sorted, or without a set, it returns FAMSA_E_STATE.
 *   cell (r, c) = Transform(LCS with sequence r as the row (seq0), len_r, len_c) as float: pid != 0 gives
 *   Transform<float, pairwise_identity> (distance_kind is then ignored), else Transform<double, distance_kind> rounded
 *   to float (0 indel075_div_lcs, 1 indel_div_lcs).  square == 0: row r holds columns 0..r-1; square != 0: a header line
 *   (',' + each id) and all n columns per row, the diagonal included (computed, and not symmetric in the dropped-carry
 *   corner of lcsbp_classic.h:55-56).  Row text: id, ',', every value followed by ',', the last byte replaced by '\n'.
 * ids: the FASTA headers without '>', id i = ids[id_offsets[i] .. id_offsets[i+1]) (n+1 offsets), written verbatim.
 * The text is handed to `write` in order (header first), in chunks of whole rows of about chunk_bytes (0 = 32 MiB; a
 * chunk grows to the widest row): the device formats and copies chunk k+1 while `write` consumes chunk k from a pinned
 * buffer that stays valid until `write` returns.  `write` returns 0 to accept; anything else stops the call with
 * FAMSA_E_SINK, no further writes, and a message naming the byte offset; the context stays usable.  `write` must not
 * call into the same context.  *bytes_written (may be NULL) = bytes accepted.  The LCS triangle stays resident in HBM
 * for the call; if it and the chunk buffers do not fit, FAMSA_E_NOMEM.  famsa_lcs_last_timing: total = all kernels of
 * the call, main = the LCS tile kernels, n_pairs = cells exported. */
typedef int (*famsa_write_fn)(void* user, const char* bytes, uint64_t n);        /* 0 = accepted */
int famsa_dist_export(famsa_ctx* ctx, int distance_kind, int square, int pid,
                      const char* ids, const uint64_t* id_offsets /* n+1 */, uint64_t chunk_bytes /* 0 = default */,
                      famsa_write_fn write, void* user, uint64_t* bytes_written);

/* Host-side Transform<T, Distance> (AbstractTreeGenerator.hpp:28-82), provided so bindings that
 * are not C++ get bit-identical distances.  kind: 0 indel075_div_lcs, 1 indel_div_lcs,
 * 2 pairwise_identity. */
double famsa_transform_f64(int kind, uint32_t lcs, uint32_t len1, uint32_t len2);
float famsa_transform_f32(int kind, uint32_t lcs, uint32_t len1, uint32_t len2);

/* Timing of the most recent LCS call on this context, measured with CUDA events on the stream the
 * kernels ran on: total = all kernels of the call, main = from its first lcs tile kernel to the end of
 * its last (an empty span in a call without one), n_pairs = the pairs the call computes (the whole
 * triangle for famsa_lcs_prim and famsa_lcs_upgma). */
int famsa_lcs_last_timing(const famsa_ctx* ctx, float* total_ms, float* main_kernel_ms,
                          uint64_t* n_pairs);

/* ------------------------------------------------------------------ HP-2: profile alignment DP
 *
 * Replaces the body of
 *   void CProfile::Align(CProfile* profile1, CProfile* profile2, uint32_t no_threads,
 *                        uint32_t no_rows_per_box, ...)            src/core/profile.cpp:244-305
 * i.e. the variant/orientation choice and the six cell loops
 *   AlignSeqSeq / AlignSeqProf / AlignProfProf                    src/core/profile_seq.cpp:24,165,495
 *   ParAlignSeqProf / ParAlignProfProf                            src/core/profile_par.cpp:26,441
 * with their helpers DP_SolveGapsProblemWhenStarting/Continuing    src/core/profile.cpp:1223-1315
 * and the traceback at the top of ConstructProfile                 src/core/profile.cpp:727-782,
 * for MANY independent merges per call (all ready nodes of the guide tree: what CProfileQueue,
 * src/core/queues.cpp:127-187, hands to the worker threads one at a time).
 * The merged-profile construction (rest of ConstructProfile, profile.cpp:784-1002) stays on the
 * host and consumes `path`; the unbanded variants are implemented (what every no_threads > 1
 * call and every progressive-alignment call uses; the banded refinement calls pass NULL
 * column mappings only when unguided -- see INTEGRATION.md).
 * Scores are int64 (score_t, src/core/defs.h:36-40): results are bit-exact, not "within 1 ulp".
 */

typedef struct {
    const int64_t* scores;   /* CProfileValues<score_t,32>: (width+1) columns x 32 rows, column c at scores + 32*c */
    const int32_t* counters; /* CProfileValues<counter_t,32>: same shape */
    uint32_t width;          /* CProfile::width */
    uint32_t card;           /* CProfile::data.size() */
} famsa_dp_profile;

typedef struct {
    famsa_dp_profile p1, p2; /* the two arguments of CProfile::Align, in call order */
} famsa_dp_job;

typedef struct {
    int64_t total_score;     /* CProfile::total_score of the merged profile */
    int64_t last[3];         /* dp_row_elem_t {D,H,V} at (W_rows, W_cols), ConstructProfile's last_elem */
    uint64_t path_offset;    /* this job's path starts at path_buf + path_offset */
    uint64_t dirs_offset;    /* this job's CDPMatrix bytes start at dirs_buf + dirs_offset (if requested) */
    uint32_t path_len;       /* = width of the merged profile */
    uint32_t rows_width, cols_width; /* after orientation */
    uint8_t swapped;         /* 1: rows of the DP matrix = p2 (Align called the cell loop as (p2, p1)) */
    uint8_t variant;         /* 0 AlignSeqSeq, 1 AlignSeqProf, 2 AlignProfProf */
    uint8_t pad[2];
} famsa_dp_result;

/* gaps[4] = {gap_open, gap_ext, gap_term_open, gap_term_ext} (CParams, already rescaled,
 * src/msa.cpp:83-106).  path_buf receives, per job, path_len direction_t bytes in forward order
 * (0 D: a row and a column are consumed, 1 H: column only, 2 V: row only) == ConstructProfile's
 * path[1..width]; job k starts at offset sum_{m<k}(p1.width + p2.width) (also reported).
 * dirs_buf may be NULL; otherwise it receives each job's (rows_width+1) x (cols_width+1)
 * CDPMatrix bytes (dirD | dirH<<2 | dirV<<4, src/core/profile.h:93-142) at offset
 * sum_{m<k}(p1.width+1)(p2.width+1).  All pointers are HOST memory. */
int famsa_dp_align_batch(famsa_ctx* ctx, const famsa_dp_job* jobs, uint32_t n_jobs, const int64_t gaps[4],
                         famsa_dp_result* results, uint8_t* path_buf, uint8_t* dirs_buf);

/* Same, but with the profile tables already resident in HBM (famsa_dp_profile pointers are DEVICE
 * pointers, 16-byte aligned; results/path/dirs are DEVICE buffers); used to time the kernels without PCIe.
 * Variant/orientation are then decided on the device too.  stream: cudaStream_t or NULL. */
int famsa_dp_align_batch_device(famsa_ctx* ctx, const famsa_dp_job* h_jobs_with_device_ptrs, uint32_t n_jobs,
                                const int64_t gaps[4], famsa_dp_result* d_results, uint8_t* d_path_buf,
                                uint8_t* d_dirs_buf, void* stream);

/* Timing of the most recent DP call: total device time and the DP kernel alone (CUDA events on the
 * launch stream), and the number of DP cells (sum of rows_width * cols_width). */
int famsa_dp_last_timing(const famsa_ctx* ctx, float* total_ms, float* kernel_ms, uint64_t* n_cells);

/* ---------------------------------------------------------------------------------------------
 * Resident profiles: ConstructProfile's merge part on the device (SURVEY 8f-2).
 *
 * Replaces, for a whole level of the guide tree, CProfile::Align + the table-building half of
 * CProfile::ConstructProfile (src/core/profile.cpp:244-305 and :784-1002: InsertColumn :1107-1111,
 * InsertGaps :1005-1050, SolveGapsProblemWhenStarting/Continuing :1114-1220, column 0 :998-1001).
 * scores/counters of every profile stay in HBM between levels; per merge only the traceback path
 * (<= W1+W2 bytes) returns to the host, where FinalizeGaps (profile.cpp:1053-1104) applies its H runs
 * to the members of the row profile and its V runs to the members of the column profile.
 * Leaves are materialised on the device from the sequences of famsa_lcs_upload
 * (CProfile::CalculateCountersScores for one sequence, profile.cpp:101-231).
 */
#define FAMSA_PROF_LEAF 0x80000000u   /* child = FAMSA_PROF_LEAF | sequence id (caller order of famsa_lcs_upload) */

typedef struct {
    uint32_t child1, child2;  /* the two arguments of CProfile::Align, in call order: resident profile id or leaf */
} famsa_prof_merge;

/* CParams::score_matrix (src/core/params.h), 24 x 24 row-major, needed to materialise leaves. */
int famsa_prof_set_scoring(famsa_ctx* ctx, const int64_t score_matrix[24 * 24]);

/* Uploads n host profiles (same layout as famsa_dp_profile for famsa_dp_align_batch) as resident ones. */
int famsa_prof_put(famsa_ctx* ctx, const famsa_dp_profile* profiles, uint32_t n, uint32_t* ids_out);

/* A resident profile from a finished (gapped) alignment: CProfile::AppendRawSequence for every row +
 * CalculateCountersScores (src/core/profile.cpp:101-235, :329-350), as CFAMSA::alignProfiles builds its two inputs
 * (src/msa.cpp:675-691): no Condense, no OptimizeGaps, all-gap columns kept.  rows: n_rows x width bytes, row-major, in the
 * order AppendRawSequence sees them; each byte a residue code 0..23 or GAP = 30 (no GUARD), as for famsa_prof_refine.
 * gaps = {gap_open, gap_ext, gap_term_open, gap_term_ext}, the rescaled costs the merge will also use (for the
 * profile-profile mode: adjustParams(n1 + n2), src/famsa.cpp:94).  *id_out: an ordinary resident profile of card n_rows,
 * for famsa_prof_merge_batch, famsa_prof_get, famsa_prof_drop, or as a famsa_prof_refine root.  Its width is `width`, and
 * width - 1 with FAMSA_PUT_ROWS_FROM_TEXT.
 * FAMSA_PUT_ROWS_FROM_TEXT: the profile the reference builds from rows read as text.  Such a CGappedSequence already starts
 * with GUARD (sequence.cpp:234), so AppendRawSequence sets the profile's width to gapped_size - 1 (profile.cpp:333-336)
 * while CalculateCounters still reads every residue and internal gap of the whole row: the profile is the flag-free one
 * without its last column (a gap run up to a residue in that column stays an internal one).  CalculateCountersScores
 * still sizes the counters gapped_size + 1, so they keep that column's residues, and the ProfProf orientation test
 * (get_num_of_non_zeros, profile.cpp:283) counts them: the entry keeps them too and the merge counts them the same way.
 * The DP never aligns that column; FinalizeGaps keeps it at the end of every merged row.  This is what
 * famsa in1 in2 out computes.
 * FAMSA's profile-profile mode is two of these calls with FAMSA_PUT_ROWS_FROM_TEXT and one
 * famsa_prof_merge_batch({id1, id2}); the merged rows are the column profile's rows, then the row profile's
 * (famsa_dp_result.swapped tells which is which), each with the path's gap columns inserted (INTEGRATION.md).
 * Does not touch the state of famsa_prof_refine: famsa_prof_refined_rows still returns the last refinement's rows.
 * FAMSA_E_STATE without famsa_prof_set_scoring; FAMSA_E_INVALID for NULL pointers, unknown flags, n_rows == 0 or width == 0
 * (width < 2 with FAMSA_PUT_ROWS_FROM_TEXT), a code that is neither < 24 nor 30, a row without a residue (CalculateCounters
 * would read symbols[0] of an empty sequence) and a one-row alignment with a gap in a column the profile keeps (with
 * FAMSA_PUT_ROWS_FROM_TEXT a gap in the last column is allowed): the reference aligns a one-row profile
 * as a sequence and its Seq* cell loops read the residues as the columns (src/core/profile_seq.cpp:32-33,176), so a gap
 * makes them read past the sequence; FAMSA_E_NOMEM when an allocation fails.  Nothing the call made stays resident after
 * an error, and the context stays usable. */
#define FAMSA_PUT_ROWS_FROM_TEXT 1

int famsa_prof_put_rows(famsa_ctx* ctx, const uint8_t* rows, uint32_t n_rows, uint32_t width, const int64_t gaps[4],
                        int flags, uint32_t* id_out);

/* Aligns and merges n independent pairs.  Resident children are consumed (as ComputeAlignment deletes
 * them, msa.cpp:406-407).  merged_ids_out[k] is the resident id of merge k's profile (width =
 * results[k].path_len, card = sum of the children's).  results/path_buf as in famsa_dp_align_batch
 * (job k's path at path_offset = sum_{m<k}(W1_m + W2_m)); path_cap = bytes available in path_buf. */
int famsa_prof_merge_batch(famsa_ctx* ctx, const famsa_prof_merge* merges, uint32_t n, const int64_t gaps[4],
                           uint32_t* merged_ids_out, famsa_dp_result* results, uint8_t* path_buf, uint64_t path_cap);

/* The whole progressive alignment as ONE call: replaces the worker loop of CFAMSA::ComputeAlignment
 * (src/msa.cpp:360-438) together with CProfileQueue (src/core/queues.cpp:17-187), which hands a merge to a worker
 * thread as soon as both of its children are finished.  Here every merge whose children are finished (or queued) is
 * submitted to the device without the host waiting for earlier batches: widths of queued children travel on the
 * device, so several dependency levels are in flight at once and nothing but the per-merge result records and
 * traceback paths ever returns to the host.
 * tree: the internal nodes of the reference's tree_structure (src/tree/TreeDefs.h:15-16), i.e. guide_tree.data() +
 * n_leaves viewed as int32 pairs: tree[2k], tree[2k+1] = children of node n_leaves + k; leaves 0..n_leaves-1 are the
 * sequences of famsa_lcs_upload in caller order; children precede parents.  Needs famsa_prof_set_scoring.
 * results[k] (k < n_leaves - 1) describes merge k; its path_offset indexes the path buffer fetched afterwards with
 * famsa_prof_tree_paths (*path_bytes_out bytes; offsets are not contiguous).  *root_id_out = resident id of the final
 * profile (famsa_prof_get / famsa_prof_drop). */
typedef struct {
    double wall_ms;               /* host wall clock of the call */
    double device_ms;             /* first to last operation on the stream (CUDA events) */
    uint64_t cells;               /* sum over merges of rows_width * cols_width */
    uint32_t n_batches;           /* submissions of ready merges */
    uint32_t n_drains;            /* times the host had to wait for the device before it could submit more */
    uint32_t max_in_flight;       /* batches queued at once */
    uint32_t pad;
    uint64_t peak_resident_bytes; /* HBM held by resident profiles at the high-water mark */
} famsa_tree_stats;

int famsa_prof_align_tree(famsa_ctx* ctx, const int32_t* tree, uint32_t n_leaves, const int64_t gaps[4],
                          famsa_dp_result* results, uint32_t* root_id_out, uint64_t* path_bytes_out,
                          famsa_tree_stats* stats /* may be NULL */);
int famsa_prof_tree_paths(famsa_ctx* ctx, uint8_t* path_buf, uint64_t path_cap);

/* The final alignment of the most recent famsa_prof_align_tree: FinalizeGaps of every merge (profile.cpp:1053-1104),
 * built on the device and kept there.  Row k is leaf order[k] (order NULL: row k = leaf k), W_root codes, GAP = 30.
 * rows may be NULL (keep on the device only); otherwise n_rows x W_root bytes, row-major, are copied to it (cap bytes).
 * Each merge's H steps are gap columns in the members of the DP's row profile, its V steps in those of the column
 * profile (famsa_dp_result.swapped says which child is which); the leaves' residues are the codes of the sequences
 * already uploaded (famsa_lcs_upload, a code outside 0..23 written as 22, as the leaf profiles count it).  Nothing is
 * uploaded again but the paths, and no host work is done per merge.  *width_out = W_root.
 * The rows describe the most recent SUCCESSFUL famsa_prof_align_tree; a later famsa_lcs_upload / famsa_lcs_upload_sorted
 * or a failed famsa_prof_align_tree leaves none: FAMSA_E_STATE.  FAMSA_E_INVALID: n_rows != the tree's leaves, an order
 * that is not a permutation of 0..n_rows-1, cap < n_rows x W_root with rows != NULL, width_out NULL.  FAMSA_E_NOMEM: an
 * allocation failed.  After an error nothing of the call's own stays allocated and the context stays usable.
 * The rows stay on the device for famsa_prof_refine with FAMSA_REFINE_TREE_ROWS, until the next call of this function. */
int famsa_prof_tree_rows(famsa_ctx* ctx, const uint32_t* order, uint32_t n_rows, uint8_t* rows, uint64_t cap,
                         uint32_t* width_out);

/* width/card of a resident profile; scores ((width+1)*32 int64) / counters ((width+1)*32 int32) are
 * copied to the host when non-NULL. */
int famsa_prof_get(famsa_ctx* ctx, uint32_t id, uint32_t* width, uint32_t* card, int64_t* scores, int32_t* counters);

/* Frees resident profiles that will not be merged (e.g. the root once the alignment is done). */
int famsa_prof_drop(famsa_ctx* ctx, const uint32_t* ids, uint32_t n);

/* Device time of the most recent famsa_prof_merge_batch: whole call and the construct kernel alone;
 * the DP part is reported by famsa_dp_last_timing. */
int famsa_prof_last_timing(famsa_ctx* ctx, float* total_ms, float* construct_ms);

/* Number of resident profiles and the HBM they occupy. */
int famsa_prof_stats(famsa_ctx* ctx, uint64_t* n_live, uint64_t* resident_bytes);

/* Refinement of the final alignment: replaces CFAMSA::RefineAlignment (src/msa_refinement.cpp:73-217, called at
 * src/msa.cpp:615) as it runs with no_threads > 1 (the unbanded Align).  Whether to refine at all (-refine_mode, -rt,
 * msa_refinement.cpp:79-82) stays with the caller; the clamps of n_refinements (:84-92) are applied here.
 * root_id: the resident profile famsa_prof_align_tree returned; it is consumed.  rows: the alignment that profile
 * describes, n_rows x width bytes, row-major, residue codes of src/core/defs.h and GAP = 30 (no GUARD), the rows in the
 * order the refinement loop uses: sorted by CGappedSequence::id, the FASTA id compared byte-wise (:116).  The caller
 * sorts, since ids are strings.  gaps = {gap_open, gap_ext, gap_term_open, gap_term_ext} as for the merges.
 * *refined_id_out: resident id of the final profile (the root's own when no candidate was accepted), for
 * famsa_prof_get / famsa_prof_drop; *width_out, *total_score_out: its width and CalculateTotalScore (0 with
 * FAMSA_REFINE_NO_TOTAL_SCORE).  The rows themselves: famsa_prof_refined_rows.  Needs famsa_prof_set_scoring
 * (FAMSA_E_STATE otherwise); FAMSA_E_INVALID for an unknown root, rows that are not the root's (width, count), fewer
 * than 2 rows, a row without residues, unknown codes or flags, NULL pointers, and an alignment (also a realignment
 * during the loop) wider than 51 199 columns; FAMSA_E_NOMEM when an allocation fails.  Errors found before the loop
 * leave the root resident; once the loop has started, a failing call consumes the root and leaves nothing of its own
 * resident.  The context stays usable after any error. */
#define FAMSA_REFINE_NO_GAP_OPT     1   /* -dgo: CParams::enable_gap_optimization = false */
#define FAMSA_REFINE_NO_TOTAL_SCORE 2   /* -dsp: CParams::enable_total_score_calculation = false */
/* FAMSA_REFINE_TREE_ROWS: rows must be NULL; the alignment is the one the most recent famsa_prof_tree_rows kept on the
 * device, in the order given there -- which must be the id order above, the caller's responsibility as it is for rows.
 * root_id must be that tree's root (still the same resident profile), n_rows and width must be its; anything else,
 * or no kept rows, is FAMSA_E_INVALID.  The rows never pass through the host. */
#define FAMSA_REFINE_TREE_ROWS      4

typedef struct {
    double wall_ms, device_ms;    /* host wall clock of the call; first to last operation on the stream */
    uint32_t n_tries;             /* i_ref at loop exit */
    uint32_t n_realigned;         /* i_succ_ref: distinct splits aligned */
    uint32_t n_accepted;          /* n_ref_succ */
    uint32_t n_identical;         /* realignments equal to the current alignment (not scored) */
    uint64_t cells;               /* sum of DP cells */
} famsa_refine_stats;

int famsa_prof_refine(famsa_ctx* ctx, uint32_t root_id, const uint8_t* rows, uint32_t n_rows, uint32_t width,
                      const int64_t gaps[4], uint32_t n_refinements, int flags,
                      uint32_t* refined_id_out, uint32_t* width_out, int64_t* total_score_out,
                      famsa_refine_stats* stats /* may be NULL */);
/* The rows of the most recent famsa_prof_refine: n_rows x width_out bytes, row-major, in the order they were given. */
int famsa_prof_refined_rows(famsa_ctx* ctx, uint8_t* rows, uint64_t cap);

#ifdef __cplusplus
}
#endif
#endif /* FAMSA_B200_H */
