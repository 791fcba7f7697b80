// famsa_prof_tree_rows: the final alignment of famsa_prof_align_tree built on the device -- FinalizeGaps of every merge
// (src/core/profile.cpp:1053-1104) without the host touching a member row.
//
// Merge k has the path P_k (0 D, 1 H, 2 V) and children (a, b); `swapped` makes b the DP's row profile.  The row
// profile's column j sits in the j-th step of P_k that is not H (an H step is a gap column in its members), the column
// profile's column j in the j-th step that is not V.  With M_v = the root column of each column of node v (M_root = the
// identity), a child's map is  M_child[j] = M_parent[s_j],  so composing from the root down gives every node's map, and a
// leaf's map places its residues: row i is W_root GAP bytes with leaf i's codes at M_i.
//
// One persistent launch.  Blocks take merges from an atomic ticket in top-down order (merge index descending: a parent
// comes after its children in the tree, so it gets an earlier ticket).  A block waits only for its own node's map, which
// the block holding the parent's (earlier) ticket writes and then flags; that block is running already, so any number of
// resident blocks makes progress, and the number of launches does not grow with the depth of the tree.  Per merge the
// block walks its path in tiles of kTRTile steps: one block-wide scan of the two counts (packed into one word) gives each
// step its column in either child, and the step writes M_parent[s] there -- into the child's map, or, for a leaf, the
// leaf's residue into its output row.  Work: the sum of the internal nodes' widths, plus the output.
#include <algorithm>
#include <cstring>
#include <numeric>
#include <vector>

#include "ctx.h"
#include "prof_dev.cuh"

namespace fb {

namespace {

constexpr int kTRTile = 512;      // path steps per block iteration = threads of k_tree_rows

struct TreeRowsMerge {
    uint64_t path_off;            // the merge's path in the device copy of the paths
    uint64_t map_off;             // the merged node's map (path_len entries) in the map storage
    uint32_t len;                 // path_len = width of the merged node
    uint32_t swapped;             // 1: child b is the DP's row profile
    int32_t a, b;                 // children (node ids: leaves < n_leaves)
};

struct TreeRowsArgs {
    const TreeRowsMerge* merges; uint32_t n_merges, n_leaves;
    const uint8_t* paths;
    int* maps;                    // the internal nodes' maps, root excluded
    unsigned* ready;              // ready[k] != 0: node n_leaves + k has its map
    unsigned* ticket;
    const int8_t* codes; const uint64_t* off;   // the uploaded sequences (famsa_lcs_upload, caller order)
    const uint32_t* rowpos;       // leaf -> output row
    uint8_t* rows; uint32_t width;              // n_leaves x width, row-major
    const uint32_t* len;          // the uploaded sequences' lengths
    unsigned* fault;              // set when a step finds an unwritten map entry or a column past its child's width
};

// exclusive prefix sum over the block in thread order; *total = the block's sum.  sh: >= 32 words.
__device__ unsigned tr_excl_scan(unsigned v, unsigned* sh, unsigned* total)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    unsigned x = v;
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    __syncthreads();                                                // sh is free (the previous tile's readers are done)
    if (lane == 31) sh[warp] = x;
    __syncthreads();
    if (warp == 0) {
        unsigned w = lane < nwarps ? sh[lane] : 0;
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned y = __shfl_up_sync(0xffffffffu, w, o);
            if (lane >= o) w += y;
        }
        sh[lane] = w;
    }
    __syncthreads();
    *total = sh[nwarps - 1];
    return (warp ? sh[warp - 1] : 0) + x - v;
}

__global__ void __launch_bounds__(kTRTile) k_tree_rows(const TreeRowsArgs A)
{
    __shared__ unsigned sh[32];
    __shared__ unsigned s_ticket;
    for (;;) {
        if (threadIdx.x == 0) s_ticket = atomicAdd(A.ticket, 1u);
        __syncthreads();
        const unsigned t = s_ticket;
        if (t >= A.n_merges) return;
        const uint32_t k = A.n_merges - 1 - t;
        const TreeRowsMerge m = A.merges[k];
        const bool root = k == A.n_merges - 1;
        const int* pmap = root ? nullptr : A.maps + m.map_off;
        if (!root) {
            if (threadIdx.x == 0) {
                while (!*(volatile unsigned*)(A.ready + k)) __nanosleep(100);
                __threadfence();
            }
            __syncthreads();
        }
        const int32_t side[2] = {m.swapped ? m.b : m.a, m.swapped ? m.a : m.b};   // row profile, column profile
        uint32_t used[2] = {0, 0};                                  // columns of either child placed by the earlier tiles
        for (uint32_t base = 0; base < m.len; base += kTRTile) {
            const uint32_t s = base + threadIdx.x;
            const bool in = s < m.len;
            const uint8_t d = in ? A.paths[m.path_off + s] : 0;
            // the two counts of one tile (< 2^16 each) scanned as the halves of one word
            const unsigned v = in ? (unsigned)(d != 1) | ((unsigned)(d != 2) << 16) : 0u;
            unsigned tot;
            const unsigned ex = tr_excl_scan(v, sh, &tot);
            if (in) {
                const int col = root ? (int)s : __ldcg(pmap + s);
                for (int c = 0; c < 2; ++c) {
                    if (!((v >> (16 * c)) & 1u)) continue;          // an H step is a gap in the row profile, a V step in the column one
                    const uint32_t j = used[c] + ((ex >> (16 * c)) & 0xffffu);
                    const int32_t node = side[c];
                    // The maps start as -1 (memset before the launch): a map entry read before its parent's block wrote
                    // and flagged it, or a path that does not fit its children, is reported instead of written through.
                    const uint32_t wn = (uint32_t)node < A.n_leaves ? A.len[node] : A.merges[node - A.n_leaves].len;
                    if (col < 0 || (uint32_t)col >= A.width || j >= wn) { atomicOr(A.fault, 1u); continue; }
                    if ((uint32_t)node < A.n_leaves) {
                        int sym = A.codes[A.off[node] + j];
                        if (sym < 0 || sym >= kNAA) sym = 22;       // as the leaf profile counts it
                        A.rows[(size_t)A.rowpos[node] * A.width + col] = (uint8_t)sym;
                    } else
                        A.maps[A.merges[node - A.n_leaves].map_off + j] = col;
                }
            }
            used[0] += tot & 0xffffu;
            used[1] += tot >> 16;
        }
        // the children's maps are complete: flag them (the whole block's stores, then one fence, as a grid barrier does)
        __syncthreads();
        if (threadIdx.x == 0) {
            __threadfence();
            for (int c = 0; c < 2; ++c)
                if ((uint32_t)side[c] >= A.n_leaves) atomicExch(A.ready + (side[c] - A.n_leaves), 1u);
        }
    }
}

} // namespace

void tree_state_invalidate(famsa_ctx* ctx) { ctx->prof.tree_valid = false; }

int prof_tree_rows(famsa_ctx* ctx, const uint32_t* order, uint32_t n_rows, uint8_t* rows, uint64_t cap, uint32_t* width_out)
{
    ProfState& P = ctx->prof;
    LcsState& L = ctx->lcs;
    if (!P.tree_valid) {
        set_error("famsa_prof_tree_rows: no alignment to build: famsa_prof_align_tree has not succeeded since the last upload");
        return FAMSA_E_STATE;
    }
    const uint32_t n = (uint32_t)P.tree_res.size() + 1, n_merges = n - 1;
    if (!width_out) { set_error("famsa_prof_tree_rows: width_out is NULL"); return FAMSA_E_INVALID; }
    if (n_rows != n) { set_error("famsa_prof_tree_rows: n_rows is " + std::to_string(n_rows) + ", the tree has " + std::to_string(n) + " leaves"); return FAMSA_E_INVALID; }
    std::vector<uint32_t> rowpos(n, UINT32_MAX);
    for (uint32_t k = 0; k < n; ++k) {
        const uint32_t leaf = order ? order[k] : k;
        if (leaf >= n || rowpos[leaf] != UINT32_MAX) {
            set_error("famsa_prof_tree_rows: order is not a permutation of 0.." + std::to_string(n - 1) + " (entry " + std::to_string(k) + ")");
            return FAMSA_E_INVALID;
        }
        rowpos[leaf] = k;
    }
    const uint32_t W = P.tree_res.back().path_len;
    const uint64_t bytes = (uint64_t)n * W;
    if (rows && cap < bytes) {
        set_error("famsa_prof_tree_rows: " + std::to_string(bytes) + " bytes needed, " + std::to_string(cap) + " given");
        return FAMSA_E_INVALID;
    }
    // per merge: its path, its children, and where its map goes (the root has none: its map is the identity)
    std::vector<TreeRowsMerge> M(n_merges);
    uint64_t map_total = 0;
    for (uint32_t k = 0; k < n_merges; ++k) {
        const famsa_dp_result& r = P.tree_res[k];
        M[k] = TreeRowsMerge{r.path_offset, map_total, r.path_len, r.swapped, P.tree_kept[2 * k], P.tree_kept[2 * k + 1]};
        if (k + 1 < n_merges) map_total += r.path_len;
    }
    cudaStream_t st = ctx->stream;
    P.tree_rows_valid = false;                                      // its buffer is rewritten from here on
    if (P.d_tree_rows.reserve(bytes) != FAMSA_OK) return FAMSA_E_NOMEM;
    Layout Lb;
    const size_t o_m = Lb.add(sizeof(TreeRowsMerge) * n_merges), o_path = Lb.add(std::max<uint64_t>(P.tree_path_bytes, 1));
    const size_t o_map = Lb.add(sizeof(int) * std::max<uint64_t>(map_total, 1)), o_flag = Lb.add(sizeof(unsigned) * (n_merges + 2));
    const size_t o_pos = Lb.add(sizeof(uint32_t) * n);
    char* blob = nullptr;
    {
        const cudaError_t e = cudaMallocAsync(reinterpret_cast<void**>(&blob), Lb.end, st);
        if (e != cudaSuccess) {
            cudaGetLastError();
            P.d_tree_rows.release();
            set_error("famsa_prof_tree_rows: cudaMallocAsync(" + std::to_string(Lb.end) + ") failed: " + cudaGetErrorString(e));
            return FAMSA_E_NOMEM;
        }
    }
    unsigned fault = 0;
    auto body = [&]() -> int {
        int& occupancy = P.tree_rows_occupancy;                     // asked once per context, under its lock
        if (!occupancy) FB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occupancy, k_tree_rows, kTRTile, 0));
        FB_CUDA(cudaMemcpyAsync(blob + o_m, M.data(), sizeof(TreeRowsMerge) * n_merges, cudaMemcpyHostToDevice, st));
        if (P.tree_path_bytes) FB_CUDA(cudaMemcpyAsync(blob + o_path, P.h_tree_paths, P.tree_path_bytes, cudaMemcpyHostToDevice, st));
        FB_CUDA(cudaMemcpyAsync(blob + o_pos, rowpos.data(), sizeof(uint32_t) * n, cudaMemcpyHostToDevice, st));
        FB_CUDA(cudaMemsetAsync(blob + o_flag, 0, sizeof(unsigned) * (n_merges + 2), st));     // ready flags, ticket, fault
        FB_CUDA(cudaMemsetAsync(blob + o_map, 0xff, sizeof(int) * map_total, st));             // every map entry -1 until written
        FB_CUDA(cudaMemsetAsync(P.d_tree_rows.p, kGAP, bytes, st));
        TreeRowsArgs A{reinterpret_cast<const TreeRowsMerge*>(blob + o_m), n_merges, n, reinterpret_cast<const uint8_t*>(blob + o_path),
                       reinterpret_cast<int*>(blob + o_map), reinterpret_cast<unsigned*>(blob + o_flag),
                       reinterpret_cast<unsigned*>(blob + o_flag) + n_merges, L.d_raw_codes.as<int8_t>(), L.d_raw_off.as<uint64_t>(),
                       reinterpret_cast<const uint32_t*>(blob + o_pos), P.d_tree_rows.as<uint8_t>(), W, L.d_raw_len.as<uint32_t>(),
                       reinterpret_cast<unsigned*>(blob + o_flag) + n_merges + 1};
        const unsigned grid = std::min<unsigned>(n_merges, (unsigned)std::max(occupancy, 1) * (unsigned)ctx->sm_count);
        k_tree_rows<<<grid, kTRTile, 0, st>>>(A);
        FB_CUDA(cudaGetLastError());
        ++ctx->launches;
        FB_CUDA(cudaMemcpyAsync(&fault, blob + o_flag + sizeof(unsigned) * (n_merges + 1), sizeof(unsigned), cudaMemcpyDeviceToHost, st));
        if (rows) FB_CUDA(cudaMemcpyAsync(rows, P.d_tree_rows.p, bytes, cudaMemcpyDeviceToHost, st));
        return FAMSA_OK;
    };
    int rc = body();
    const cudaError_t f = cudaFreeAsync(blob, st);
    const cudaError_t s = cudaStreamSynchronize(st);
    if (rc == FAMSA_OK && (f != cudaSuccess || s != cudaSuccess)) {
        set_error(std::string("famsa_prof_tree_rows: ") + cudaGetErrorString(f != cudaSuccess ? f : s));
        rc = FAMSA_E_CUDA;
    }
    if (rc == FAMSA_OK && fault) {
        set_error("famsa_prof_tree_rows: internal: a merge read a column map before it was written, or its path does not fit its children");
        rc = FAMSA_E_CUDA;
    }
    if (rc != FAMSA_OK) { P.d_tree_rows.release(); return rc; }
    P.tree_rows_n = n; P.tree_rows_w = W;
    P.tree_rows_root = P.tree_root; P.tree_rows_root_gen = P.tree_root_gen;
    P.tree_rows_valid = true;
    *width_out = W;
    return FAMSA_OK;
}

} // namespace fb
