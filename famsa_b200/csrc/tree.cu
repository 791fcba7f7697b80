// The device guide trees on the resident LCS triangle: medoid assignment, MST-Prim (the sequential vertex loop and the
// Boruvka rounds), single linkage on the same MST engines, and UPGMA.  The triangle and the side rows come from lcs.cu;
// see DESIGN.md section 6.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <queue>
#include <tuple>
#include <type_traits>

#include <cooperative_groups.h>

#include "ctx.h"
#include "triangle_dev.cuh"

namespace fb {

// ------------------------------------------------------------------------------------------------
// shared pieces: the edge key, candidate reductions, the distance triangle
// ------------------------------------------------------------------------------------------------

// MSTPrim's edge key ~ids_to_uint64(min id, max id) (MSTPrim.h:432-439) and its inverse uint64_to_id (:441-450)
__host__ __device__ __forceinline__ unsigned long long edge_key(uint32_t a, uint32_t b)
{
    const unsigned long long lo = a < b ? a : b, hi = a < b ? b : a;
    return ~((lo << 32) + hi);
}
__host__ __device__ __forceinline__ void edge_ids(unsigned long long key, uint32_t& lo, uint32_t& hi)
{
    lo = (uint32_t)(~key >> 32);
    hi = (uint32_t)(~key & 0xffffffffull);
}

// The reduction candidates and their orders.  Every reduction keeps its own value unless the other one is strictly less,
// so ties go to the value a lane already holds.
struct EdgeMin {                   // (distance, edge key), compared lexicographically
    double d;
    unsigned long long k;
};
struct PrimCand {                  // k_prim's: id < 0 = no candidate
    double dist;
    unsigned long long key;
    int id;
    int pad;
};
__host__ __device__ __forceinline__ bool cand_less(const EdgeMin& x, const EdgeMin& c) { return x.d < c.d || (x.d == c.d && x.k < c.k); }
// (the key test is a non-short-circuit `&`: with `&&` every butterfly level of k_prim gets a branch, and its loop slows)
__device__ __forceinline__ bool cand_less(const PrimCand& x, const PrimCand& c)
{
    return x.id >= 0 && (c.id < 0 || x.dist < c.dist || ((x.dist == c.dist) & (x.key < c.key)));
}
__device__ __forceinline__ bool cand_less(unsigned long long x, unsigned long long c) { return x < c; }
struct NjCand {                    // k_nj's pair (q, a, b), a < b: k = (q in unsigned order << 32) | a; k = ~0 = no candidate
    unsigned long long k;
    uint32_t b;
    uint32_t pad;
};
__device__ __forceinline__ bool cand_less(const NjCand& x, const NjCand& c) { return x.k < c.k || ((x.k == c.k) & (x.b < c.b)); }

__device__ __forceinline__ EdgeMin shfl_xor(const EdgeMin& c, int o)
{
    return EdgeMin{__shfl_xor_sync(0xffffffffu, c.d, o), __shfl_xor_sync(0xffffffffu, c.k, o)};
}
__device__ __forceinline__ PrimCand shfl_xor(const PrimCand& c, int o)
{
    return PrimCand{__shfl_xor_sync(0xffffffffu, c.dist, o), __shfl_xor_sync(0xffffffffu, c.key, o),
                    __shfl_xor_sync(0xffffffffu, c.id, o), 0};
}
__device__ __forceinline__ unsigned long long shfl_xor(unsigned long long c, int o) { return __shfl_xor_sync(0xffffffffu, c, o); }
__device__ __forceinline__ NjCand shfl_xor(const NjCand& c, int o)
{
    return NjCand{__shfl_xor_sync(0xffffffffu, c.k, o), __shfl_xor_sync(0xffffffffu, c.b, o), 0};
}

template <class C>
__device__ __forceinline__ C warp_min(C c)
{
    for (int o = 16; o; o >>= 1) {
        const C x = shfl_xor(c, o);
        if (cand_less(x, c)) c = x;
    }
    return c;
}

// minimum over the block, valid in warp 0; `none` stands in for the warps the block does not have, sh[32] is the
// caller's shared scratch (declared first in the kernel: k_upgma's merge loop is measurably slower with it elsewhere)
template <class C>
__device__ __forceinline__ C block_min(C c, C none, C* sh)
{
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    c = warp_min(c);
    if (lane == 0) sh[warp] = c;
    __syncthreads();
    if (warp == 0) c = warp_min(lane < blockDim.x / 32 ? sh[lane] : none);
    return c;
}

// minimum of v[0..count) for one warp: the cross-block gather of the cooperative kernels
template <class C>
__device__ __forceinline__ C warp_min_of(const C* v, uint32_t count, C none)
{
    C c = none;
    for (uint32_t b = threadIdx.x & 31; b < count; b += 32) {
        const C x = v[b];
        if (cand_less(x, c)) c = x;
    }
    return warp_min(c);
}

// one block per row i: Transform<T, Distance> of (i, j), j < i (AbstractTreeGenerator.hpp:28-82) -- float64 for the
// Boruvka rounds, float32 for UPGMA (computeDistances, UPGMA.cpp:75-109)
template <class T>
__global__ void __launch_bounds__(256) k_dist_tri(const void* __restrict__ tri, int eb, const uint32_t* __restrict__ lens,
                                                  const T* __restrict__ pow075, int kind, T* __restrict__ out)
{
    const uint32_t i = blockIdx.x + 1;
    const size_t base = tri_index(i, 0);
    const uint32_t li = lens[i];
    for (uint32_t j = threadIdx.x; j < i; j += blockDim.x) {
        const uint32_t l = lcs_load(tri, eb, base + j);
        if constexpr (std::is_same<T, float>::value) out[base + j] = transform_f32(kind, l, li, lens[j], pow075);
        else out[base + j] = transform_f64(kind, l, li, lens[j], pow075);
    }
}

// ------------------------------------------------------------------------------------------------
// medoid assignment: float Transform + running arg-min over the seed rows (FastTree.cpp:309-324)
// ------------------------------------------------------------------------------------------------

// Only the sequences whose mask group lies in [g_begin, g_end) are answered; the result is packed as
// (float bits of the distance << 32) | seed index so that an element-wise MIN over the shards (one all-reduce) assembles
// the complete assignment -- distances are >= 0, so their bit patterns order like the values, and among equal distances
// the lowest seed index wins, which is what the strict < of the sequential loop does.  Unanswered entries hold INT64_MAX.
__global__ void k_assign_packed(const void* __restrict__ lcs, int elem_bytes, uint32_t n, uint32_t n_seeds,
                                const uint32_t* __restrict__ seed_ids, const uint32_t* __restrict__ lens,
                                const float* __restrict__ pow075, int kind,
                                const uint32_t* __restrict__ invperm, uint32_t g_begin, uint32_t g_end,
                                long long* __restrict__ packed)
{
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const uint32_t g = invperm[j] / 32;
    if (g < g_begin || g >= g_end) { packed[j] = 0x7fffffffffffffffll; return; }
    const uint32_t lj = lens[j];
    float best = 0.f;
    uint32_t a = 0;
    for (uint32_t k = 0; k < n_seeds; ++k) {
        const float d = transform_f32(kind, lcs_load(lcs, elem_bytes, (size_t)k * n + j), lens[seed_ids[k]], lj, pow075);
        if (k == 0 || d < best) { best = d; a = k; }
    }
    packed[j] = (long long)(((unsigned long long)__float_as_uint(best) << 32) | a);
}

// ------------------------------------------------------------------------------------------------
// MST-Prim vertex loop (MSTPrim<>::run_view, MSTPrim.cpp:280-549) on the resident LCS triangle
// ------------------------------------------------------------------------------------------------

struct PrimState {                 // per sequence: best known connection to the tree
    double dist;
    unsigned long long key;        // edge_key(from, j)
};

// Cooperative grid (one block per SM, all co-resident): per step every thread relaxes its own unvisited sequences
// against the current vertex (one triangle lookup + one pow-table lookup each, all independent), blocks publish their
// best (dist, key) pair, ONE grid-wide barrier, and every block reduces the published candidates itself, so all
// blocks agree on the next vertex without a second barrier.  Candidate slots are double-buffered by step parity.
// Lookups go through lcs_seq0 on the true-LCS triangle and the side rows (lcs_side_rows), the representation the square
// distance export reads too.
// kSlink (famsa_lcs_slink): tri is the triangle SLINK reads (row = seq0, dropped-carry rows exact), every lookup reads
// it (side_idx and side are not read), and there is no lower-bound skip -- SingleLinkage has none.
template <bool kSlink>
__global__ void __launch_bounds__(1024) k_prim(const void* __restrict__ tri, int eb, uint32_t n,
                                               const uint32_t* __restrict__ lens, const double* __restrict__ pow075,
                                               int kind, const int* __restrict__ side_idx,
                                               const uint32_t* __restrict__ side, PrimState* __restrict__ st,
                                               unsigned char* __restrict__ visited, PrimCand* __restrict__ cand,
                                               int* __restrict__ out_from, int* __restrict__ out_to,
                                               double* __restrict__ out_dist, int* __restrict__ order)
{
    namespace cg = cooperative_groups;
    cg::grid_group grid = cg::this_grid();
    __shared__ PrimCand sh[32];
    __shared__ int sh_v;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t gtid = blockIdx.x * blockDim.x + tid, gthreads = gridDim.x * blockDim.x;
    const uint32_t nblk = gridDim.x;
    const PrimCand none{0.0, 0, -1, 0};
    for (uint32_t j = gtid; j < n; j += gthreads) {
        st[j].dist = 1.7976931348623157e308;        // numeric_limits<double>::max()
        st[j].key = 0;
        visited[j] = j == 0;
        order[j] = j == 0 ? 0 : (int)n;
    }
    // the first sequence a thread owns lives in registers (with n <= gridDim.x * 1024 that is all of them)
    const bool has0 = gtid < n;
    const uint32_t len0 = has0 ? lens[gtid] : 0;
    bool vis0 = gtid == 0;
    double d0 = 1.7976931348623157e308;
    unsigned long long k0 = 0;
    uint32_t v = 0;
    const Seq0View L{tri, eb, n, side_idx, side};
    grid.sync();
    for (uint32_t step = 1; step < n; ++step) {
        const uint32_t lv = lens[v];
        const int sv = side_row<!kSlink>(L, v);
        PrimCand b = none;
        // MSTPrim.cpp:450-467: a candidate is only computed when the distance it would have with LCS = the shorter length
        // does not exceed its current one.  A no-op for a true LCS (<= the shorter length); with the dropped-carry corner the
        // reference's LCS can be larger, and then the skip decides whether the candidate is relaxed.
        if (has0 && !vis0) {
            const uint32_t j = gtid;
            const bool tried = kSlink || transform_f64(kind, lv < len0 ? lv : len0, lv, len0, pow075) <= d0;
            const double d = tried ? transform_f64(kind, lcs_seq0(L, sv, v, j), lv, len0, pow075) : 1.7976931348623157e308;
            if (tried && d <= d0) {
                const unsigned long long k = edge_key(v, j);
                if (d < d0 || k < k0) { d0 = d; k0 = k; }                                  // pair <, given d <= d0
            }
            b = PrimCand{d0, k0, (int)j, 0};
        }
        for (uint32_t j = gtid + gthreads; j < n; j += gthreads) {                         // only when n > grid size
            if (visited[j]) continue;
            double cd = st[j].dist;
            unsigned long long ck = st[j].key;
            const uint32_t lj = lens[j];
            const bool tried = kSlink || transform_f64(kind, lv < lj ? lv : lj, lv, lj, pow075) <= cd;
            const double d = tried ? transform_f64(kind, lcs_seq0(L, sv, v, j), lv, lj, pow075) : 1.7976931348623157e308;
            if (tried && d <= cd) {
                const unsigned long long k = edge_key(v, j);
                if (d < cd || k < ck) { cd = d; ck = k; st[j].dist = cd; st[j].key = ck; }
            }
            const PrimCand c{cd, ck, (int)j, 0};
            if (cand_less(c, b)) b = c;
        }
        // block-wide minimum, one grid barrier, then every block reduces the published candidates for itself
        b = block_min(b, none, sh);
        if (tid == 0) cand[(step & 1) * nblk + blockIdx.x] = b;
        grid.sync();
        if (warp == 0) {
            b = warp_min_of(cand + (step & 1) * nblk, nblk, none);
            if (lane == 0) {
                sh_v = b.id;
                if (blockIdx.x == 0) {
                    uint32_t lo, hi;
                    edge_ids(b.key, lo, hi);
                    out_from[step - 1] = (int)lo;
                    out_to[step - 1] = (int)hi;
                    out_dist[step - 1] = b.dist;
                    order[b.id] = (int)step;
                }
                if ((uint32_t)b.id >= gthreads && (uint32_t)b.id % gthreads / blockDim.x == blockIdx.x) visited[b.id] = 1;   // its owner block
            }
        }
        __syncthreads();
        v = (uint32_t)sh_v;
        if (v == gtid) vis0 = true;
    }
}

// ------------------------------------------------------------------------------------------------
// Parallel MST (Boruvka rounds) under MSTPrim's edge order.
//
// MSTPrim relaxes and elects with the pair (distance, edge_key(min id, max id)) compared lexicographically
// (MSTPrim.cpp:366-386, 492-503).  The key is unique per edge, so the pairs are a strict total order and the minimum
// spanning tree under it is unique: any algorithm finds the edges Prim finds.  What Prim adds is the visiting order
// from vertex 0, and that can be replayed on the n-1 tree edges alone (at every step Prim takes the smallest edge
// leaving the visited set, which is a tree edge).  So: distances once into a float64 triangle, then log2(n) rounds in
// which every vertex finds its smallest edge into another component -- two streaming passes over the triangle, rows
// and columns, both coalesced -- while the host merges components (union-find over n entries) and finally replays
// Prim's order with a heap.  Used when no sequence has orientation-dependent LCS values (the dropped-carry corner);
// otherwise the sequential loop above runs.  famsa_b200/mst.py + tests/test_mst_host.py pin the argument on the CPU.
// ------------------------------------------------------------------------------------------------
constexpr double kEdgeNone = __builtin_huge_val();      // +inf: no candidate (distances are finite)

// row pass: vertex i against its lower neighbours j < i in other components
__global__ void __launch_bounds__(256) k_mst_rows(const double* __restrict__ dtri, uint32_t n, const uint32_t* __restrict__ comp,
                                                  EdgeMin* __restrict__ best)
{
    __shared__ EdgeMin sh[32];
    const uint32_t i = blockIdx.x;
    const size_t base = tri_index(i, 0);
    const uint32_t ci = comp[i];
    EdgeMin e{kEdgeNone, 0};
    for (uint32_t j = threadIdx.x; j < i; j += blockDim.x) {
        if (comp[j] == ci) continue;
        const EdgeMin c{dtri[base + j], edge_key(i, j)};
        if (cand_less(c, e)) e = c;
    }
    e = block_min(e, EdgeMin{kEdgeNone, 0}, sh);
    if (threadIdx.x == 0) best[i] = e;
}

// column pass: vertex j against its upper neighbours i > j; block = 32 columns x a chunk of kMstChunk rows, every row
// contributes a coalesced 256-byte segment.  part[chunk][j] receives the chunk's minimum.
constexpr uint32_t kMstChunk = 1024;
__global__ void __launch_bounds__(256) k_mst_cols(const double* __restrict__ dtri, uint32_t n, const uint32_t* __restrict__ comp,
                                                  EdgeMin* __restrict__ part)
{
    __shared__ EdgeMin sh[8][32];
    const uint32_t x = threadIdx.x & 31, y = threadIdx.x >> 5;
    const uint32_t j = blockIdx.x * 32 + x;
    const uint32_t r0 = blockIdx.y * kMstChunk, r1 = r0 + kMstChunk < n ? r0 + kMstChunk : n;
    EdgeMin e{kEdgeNone, 0};
    if (j < n) {
        const uint32_t cj = comp[j];
        uint32_t i = r0 + y;
        if (i <= j) i += ((j + 1 - i) + 7) / 8 * 8;                 // first row of this thread's residue class above j
        for (; i < r1; i += 8) {
            if (comp[i] == cj) continue;
            const EdgeMin c{dtri[tri_index(i, j)], edge_key(i, j)};
            if (cand_less(c, e)) e = c;
        }
    }
    sh[y][x] = e;
    __syncthreads();
    if (y == 0 && j < n) {
        for (int q = 1; q < 8; ++q)
            if (cand_less(sh[q][x], e)) e = sh[q][x];
        part[(size_t)blockIdx.y * n + j] = e;
    }
}

// best[j] = min(best[j] (row pass), part[*][j])
__global__ void __launch_bounds__(256) k_mst_combine(uint32_t n, uint32_t n_chunks, const EdgeMin* __restrict__ part, EdgeMin* __restrict__ best)
{
    const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= n) return;
    EdgeMin e = best[j];
    for (uint32_t c = j / kMstChunk; c < n_chunks; ++c)              // chunks that end at or below row j hold nothing for j
        if (cand_less(part[(size_t)c * n + j], e)) e = part[(size_t)c * n + j];
    best[j] = e;
}

// ------------------------------------------------------------------------------------------------
// UPGMA on the resident triangle (UPGMA<>::computeTree, UPGMA.cpp:114-295; SURVEY 8f-1).
//
// The reference's agglomeration is MUSCLE's nearest-neighbour-cache UPGMA: every live row keeps (MinDist, NearestNeighbor);
// an iteration picks the live row with the smallest MinDist (first such row), merges it with its cached neighbour,
// overwrites the row of the left child with the averaged distances and re-labels -- but does not re-evaluate -- the
// caches of the other rows (UPGMA.cpp:229-262: a row whose neighbour was the right child now points at the left child
// and keeps the OLD distance).  Results depend on that, so it is reproduced step for step; what is parallel is the inside
// of a step: both scans (arg-min over the rows, update + arg-min over the new row) are grid-wide reductions of packed
// (float bits, index) words -- distances are >= 0, so unsigned order is value order and ties go to the lowest index,
// exactly what the strict < of the sequential scans does.  One cooperative kernel, two grid barriers per merge.
// ------------------------------------------------------------------------------------------------
constexpr float kUpgmaBig = 1e29f;                                  // UPGMA::BIG_DIST (UPGMA.h:82)
constexpr unsigned long long kNoCand = ~0ull;

__device__ __forceinline__ unsigned long long pack_cand(float d, uint32_t j) { return ((unsigned long long)__float_as_uint(d) << 32) | j; }

// initial (MinDist, NearestNeighbor) of every row (UPGMA.cpp:183-203): partners are met in ascending index order and
// only a strictly smaller distance replaces the cache, so the cache is the arg-min with the lowest partner on ties
__global__ void __launch_bounds__(256) k_upgma_init(const float* __restrict__ dist, uint32_t n, float* __restrict__ mind, uint32_t* __restrict__ nn,
                                                    int* __restrict__ node)
{
    __shared__ unsigned long long sh[32];
    const uint32_t r = blockIdx.x;
    unsigned long long best = kNoCand;
    for (uint32_t p = threadIdx.x; p < n; p += blockDim.x) {
        if (p == r) continue;
        const float d = dist[p < r ? tri_index(r, p) : tri_index(p, r)];
        if (d < kUpgmaBig) { const unsigned long long c = pack_cand(d, p); best = c < best ? c : best; }
    }
    best = block_min(best, kNoCand, sh);
    if (threadIdx.x == 0) {
        mind[r] = best == kNoCand ? kUpgmaBig : __uint_as_float((unsigned)(best >> 32));
        nn[r] = best == kNoCand ? 0x7fffffffu : (uint32_t)best;
        node[r] = (int)r;
    }
}

template <bool MODIFIED>
__global__ void __launch_bounds__(1024) k_upgma(float* __restrict__ dist, uint32_t n, float* __restrict__ mind, uint32_t* __restrict__ nn,
                                                int* __restrict__ node, unsigned long long* __restrict__ cand, int* __restrict__ out_tree,
                                                int* __restrict__ status)
{
    namespace cg = cooperative_groups;
    cg::grid_group grid = cg::this_grid();
    __shared__ unsigned long long sh[32];
    __shared__ unsigned long long sh_pick;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t gtid = blockIdx.x * blockDim.x + tid, gthreads = gridDim.x * blockDim.x, nblk = gridDim.x;
    auto tri_at = [](uint32_t a, uint32_t b) { return tri_index(a > b ? a : b, a > b ? b : a); };
    // every block reduces the nblk published candidates of buffer `buf` for itself: all agree without a second barrier
    auto gather = [&](uint32_t buf) -> unsigned long long {
        if (warp == 0) {
            const unsigned long long v = warp_min_of(cand + (size_t)buf * nblk, nblk, kNoCand);
            if (lane == 0) sh_pick = v;
        }
        __syncthreads();
        return sh_pick;
    };
    // what the previous merge changed (row L got a new cache, row R died): every thread knows it from the reductions, so the
    // scan below does not have to wait for thread 0's writes to become visible -- two grid barriers per merge, not three
    uint32_t pL = 0xffffffffu, pR = 0xffffffffu;
    unsigned long long pN = kNoCand;
    for (uint32_t it = 0; it + 1 < n; ++it) {
        // ---- the live row with the smallest cached distance (first such row)
        unsigned long long best = kNoCand;
        for (uint32_t j = gtid; j < n; j += gthreads) {
            if (j == pR) continue;
            float d;
            if (j == pL) { if (pN == kNoCand) continue; d = __uint_as_float((unsigned)(pN >> 32)); }
            else { if (node[j] < 0) continue; d = mind[j]; }
            if (d < kUpgmaBig) { const unsigned long long c = pack_cand(d, j); best = c < best ? c : best; }
        }
        best = block_min(best, kNoCand, sh);
        if (tid == 0) cand[(size_t)0 * nblk + blockIdx.x] = best;
        grid.sync();
        const unsigned long long pick = gather(0);
        if (pick == kNoCand) { if (gtid == 0) *status = 1; return; }     // no finite distance left: the reference would index out of range
        const uint32_t L = (uint32_t)pick, R = nn[L];
        // ---- distances to the new node overwrite the row of L; the arg-min of the new row becomes L's cache
        unsigned long long nbest = kNoCand;
        for (uint32_t j = gtid; j < n; j += gthreads) {
            if (j == L || j == R || node[j] < 0) continue;
            const size_t vL = tri_at(L, j), vR = tri_at(R, j);
            const float dL = dist[vL], dR = dist[vR];
            const float nd = MODIFIED ? __fadd_rn(__fmul_rn(0.05f, __fadd_rn(dL, dR)), __fmul_rn(0.9f, dR < dL ? dR : dL))
                                      : __fmul_rn(__fadd_rn(dL, dR), 0.5f);
            if (nn[j] == R) nn[j] = L;
            dist[vL] = nd;
            if (nd < kUpgmaBig) { const unsigned long long c = pack_cand(nd, j); nbest = c < nbest ? c : nbest; }
        }
        nbest = block_min(nbest, kNoCand, sh);
        if (tid == 0) cand[(size_t)1 * nblk + blockIdx.x] = nbest;
        grid.sync();
        const unsigned long long npick = gather(1);
        if (gtid == 0) {
            out_tree[2 * it] = node[L];
            out_tree[2 * it + 1] = node[R];
            node[L] = (int)(n + it);
            nn[L] = npick == kNoCand ? 0x7fffffffu : (uint32_t)npick;
            mind[L] = npick == kNoCand ? kUpgmaBig : __uint_as_float((unsigned)(npick >> 32));
            node[R] = -1;                                                // (visible to everybody after the next barrier)
        }
        pL = L; pR = R; pN = npick;
    }
}

// ------------------------------------------------------------------------------------------------
// Neighbour joining on the resident triangle (NeighborJoining<>::computeTree, NeighborJoining.cpp:33-118).
//
// The reference keeps the live clusters in ascending original order (erase only, the merged cluster keeps its slot), so
// a slot order that only ever loses dead slots is its position order, and its first-found tie rule is the lexicographic
// minimum of (q, a, b).  Per merge, one cooperative kernel with two grid barriers:
//   1. the Q scan over the live pairs (one warp per row, lanes along it) and its arg-min per block;
//   2. every block reduces the block candidates itself, then row a, the sums s_k and the node table are updated.
// The new s_a is a chain of dependent float adds in ascending slot order (:104); it runs in one warp (the last of the
// grid) during the NEXT scan, which leaves row a and column a to that warp: it sums, then scans the pairs of a.
// When the live rows fall to half of the stored ones the triangle, s and node are compacted, order preserved, into the
// other of two buffers (the second a quarter of the first), so each scan reads ~the live triangle only.
// Dead slots have s = NaN: their q is NaN and never wins, so the scan needs no liveness test per element.
// ------------------------------------------------------------------------------------------------
constexpr float kFltMax = 3.40282347e+38f;                       // numeric_limits<float>::max(), min_q's start (:59)
constexpr uint32_t kNjNone = 0xffffffffu;

// q as an unsigned key that orders like the float (negative values included); -0 and +0 are one key, as they are one value
__device__ __forceinline__ uint32_t nj_qkey(float q)
{
    const uint32_t u = __float_as_uint(__fadd_rn(q, 0.f));       // -0 + 0 = +0
    return (u >> 31) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ NjCand nj_cand(float q, uint32_t a, uint32_t b)
{
    return q < kFltMax ? NjCand{((unsigned long long)nj_qkey(q) << 32) | a, b, 0} : NjCand{~0ull, kNjNone, 0};
}
// q of the pair at positions a < b (:69): product, then the earlier position's sum, then the later one's, each rounded
__device__ __forceinline__ float nj_q(float f, float d, float s_lo, float s_hi) { return __fsub_rn(__fsub_rn(__fmul_rn(f, d), s_lo), s_hi); }

// initial sums (:45-55): s_i = 0, then + D(i, j) for j = 0..n-1, j != i, one add at a time.  One thread per row, 32 rows
// per warp; tiles left of the diagonal are rows of the warp's own rows, staged through shared memory so the loads stay
// coalesced, tiles right of it are columns of later rows and coalesced as they are.  Also node[i] = i.
__global__ void __launch_bounds__(128) k_nj_sums(const float* __restrict__ D, uint32_t n, float* __restrict__ s, int* __restrict__ node)
{
    __shared__ float tile[4][32][33];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t i0 = (blockIdx.x * 4 + warp) * 32, i = i0 + lane;
    if (i0 >= n) return;
    float acc = 0.f;
    for (uint32_t j0 = 0; j0 < n; j0 += 32) {
        if (j0 < i0) {                                           // j < i for every lane
            for (uint32_t r = 0; r < 32; ++r) tile[warp][r][lane] = i0 + r < n ? D[tri_index(i0 + r, j0 + lane)] : 0.f;
            __syncwarp();
            for (uint32_t jj = 0; jj < 32; ++jj) acc = __fadd_rn(acc, tile[warp][lane][jj]);
            __syncwarp();
        } else {
            for (uint32_t j = j0; j < j0 + 32 && j < n; ++j)
                if (i < n && j != i) acc = __fadd_rn(acc, D[j < i ? tri_index(i, j) : tri_index(j, i)]);
        }
    }
    if (i < n) { s[i] = acc; node[i] = (int)i; }
}

// The chain of s_a for the slot merged last, then the pairs of a, by one warp: the candidate of those pairs for lane 0.
// Lanes load 128 slots at a time, one chunk ahead, and every lane adds them in slot order (the same chain in each lane).
__device__ __forceinline__ NjCand nj_chain(const float* __restrict__ D, float* __restrict__ s, const int* __restrict__ node,
                                           uint32_t R, uint32_t pa, float f, uint32_t lane)
{
    constexpr uint32_t U = 4;
    auto dist = [&](uint32_t k) { return D[k < pa ? tri_index(pa, k) : tri_index(k, pa)]; };
    auto load = [&](uint32_t k0, float (&v)[U], unsigned (&live)[U]) {
#pragma unroll
        for (uint32_t u = 0; u < U; ++u) {
            const uint32_t k = k0 + u * 32 + lane;
            const bool l = k < R && k != pa && node[k] >= 0;
            v[u] = l ? dist(k) : 0.f;
            live[u] = __ballot_sync(0xffffffffu, l);
        }
    };
    float sa = 0.f;
    float v[U], nv[U];
    unsigned live[U], nlive[U];
    load(0, v, live);
    for (uint32_t k0 = 0; k0 < R; k0 += 32 * U) {
        if (k0 + 32 * U < R) load(k0 + 32 * U, nv, nlive);
#pragma unroll
        for (uint32_t u = 0; u < U; ++u)
#pragma unroll
            for (uint32_t j = 0; j < 32; ++j) {
                const float x = __shfl_sync(0xffffffffu, v[u], j);
                sa = (live[u] >> j & 1) ? __fadd_rn(sa, x) : sa;
            }
#pragma unroll
        for (uint32_t u = 0; u < U; ++u) { v[u] = nv[u]; live[u] = nlive[u]; }
    }
    // pairs (k, a) and (a, k) in ascending k per lane, i.e. in lexicographic order: a strict < keeps the first
    float bq = kFltMax;
    uint32_t ba = 0, bb = 0;
    for (uint32_t k = lane; k < R; k += 32) {
        if (k == pa || node[k] < 0) continue;
        const float q = k < pa ? nj_q(f, dist(k), s[k], sa) : nj_q(f, dist(k), sa, s[k]);
        if (q < bq) { bq = q; ba = k < pa ? k : pa; bb = k < pa ? pa : k; }
    }
    if (lane == 0) s[pa] = sa;
    return nj_cand(bq, ba, bb);
}

// D0: the float triangle of n rows; D1: room for the triangle of n/2 + 1 rows; s/node: two buffers of n each; map: n
// entries; misc[0]: the new slot of the pending row after a compaction.  out_tree: the n - 1 merges; *status = 1 when an
// iteration has no candidate (every q NaN or >= FLT_MAX), where the reference would merge cluster 0 with itself.
__global__ void __launch_bounds__(1024) k_nj(float* __restrict__ D0, float* __restrict__ D1, uint32_t n, float* __restrict__ s0,
                                             float* __restrict__ s1, int* __restrict__ node0, int* __restrict__ node1,
                                             uint32_t* __restrict__ map, uint32_t* __restrict__ misc, NjCand* __restrict__ cand,
                                             int* __restrict__ out_tree, int* __restrict__ status)
{
    namespace cg = cooperative_groups;
    cg::grid_group grid = cg::this_grid();
    __shared__ NjCand sh[32];
    __shared__ NjCand sh_pick;
    __shared__ uint32_t sh_cnt[32];
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t gtid = blockIdx.x * blockDim.x + tid, gthreads = gridDim.x * blockDim.x, nblk = gridDim.x;
    const uint32_t gw = blockIdx.x * 32 + warp, n_warps = nblk * 32;
    const bool chain_warp = gw == n_warps - 1;                   // the scan runs on the other n_warps - 1 warps
    const NjCand none{~0ull, kNjNone, 0};
    float* D = D0; float* Dn = D1; float* s = s0; float* sn = s1; int* node = node0; int* noden = node1;
    uint32_t R = n, pa = kNjNone;                                // stored rows; slot whose s_a chain is pending
    for (uint32_t it = 0; n - it > 2; ++it) {
        const uint32_t m = n - it;
        if (2 * m <= R) {
            // ---- compaction: block 0 ranks the live slots (map: new -> old) and moves s and node; then all copy the rows
            if (blockIdx.x == 0) {
                uint32_t base = 0;
                for (uint32_t k0 = 0; k0 < R; k0 += blockDim.x) {
                    const uint32_t k = k0 + tid;
                    const bool l = k < R && node[k] >= 0;
                    const unsigned bal = __ballot_sync(0xffffffffu, l);
                    if (lane == 0) sh_cnt[warp] = __popc(bal);
                    __syncthreads();
                    uint32_t pre = 0, total = 0;
                    for (uint32_t w = 0; w < blockDim.x / 32; ++w) { pre += w < warp ? sh_cnt[w] : 0; total += sh_cnt[w]; }
                    if (l) {
                        const uint32_t nk = base + pre + __popc(bal & ((1u << lane) - 1));
                        map[nk] = k; sn[nk] = s[k]; noden[nk] = node[k];
                        if (k == pa) misc[0] = nk;
                    }
                    base += total;
                    __syncthreads();
                }
            }
            grid.sync();
            for (uint32_t r = 1 + gw; r < m; r += n_warps) {
                const float* src = D + tri_index(map[r], 0);
                float* dst = Dn + tri_index(r, 0);
                for (uint32_t c = lane; c < r; c += 32) dst[c] = src[map[c]];
            }
            grid.sync();
            { float* t = D; D = Dn; Dn = t; }
            { float* t = s; s = sn; sn = t; }
            { int* t = node; node = noden; noden = t; }
            R = m;
            if (pa != kNjNone) pa = misc[0];
        }
        // ---- Q scan: every live pair but those of the pending slot, whose sum the chain warp computes meanwhile
        const float f = (float)(m - 2);
        NjCand best = none;
        if (chain_warp) {
            if (pa != kNjNone) best = nj_chain(D, s, node, R, pa, f, lane);
        } else {
            // per lane, rows ascending and columns ascending within a row: (q, c) decides, and an equal (q, c) came first
            float bq = kFltMax;
            uint32_t bc = 0, bb = 0;
            for (uint32_t b = 1 + gw; b < R; b += n_warps - 1) {
                const float sb = s[b];
                if (b == pa || isnan(sb)) continue;              // dead row, or every q of the row NaN
                const float* row = D + tri_index(b, 0);
                for (uint32_t c = lane; c < b; c += 32) {
                    if (c == pa) continue;
                    const float q = nj_q(f, row[c], s[c], sb);
                    if (q < bq || ((q == bq) & (c < bc))) { bq = q; bc = c; bb = b; }
                }
            }
            best = nj_cand(bq, bc, bb);
        }
        best = block_min(best, none, sh);
        if (tid == 0) cand[blockIdx.x] = best;
        grid.sync();
        if (warp == 0) {
            const NjCand v = warp_min_of(cand, nblk, none);
            if (lane == 0) sh_pick = v;
        }
        __syncthreads();
        const NjCand pick = sh_pick;
        if (pick.k == ~0ull) { if (gtid == 0) *status = 1; return; }
        // ---- merge (:79-113): row a gets (D(a,k) + D(b,k) - D(a,b)) / 2, every other live sum loses D(a,k) + D(b,k) and
        // gains the new distance; b dies
        const uint32_t a = (uint32_t)pick.k, b = pick.b;
        const float dab = D[tri_index(b, a)];
        for (uint32_t k = gtid; k < R; k += gthreads) {
            if (k == a || k == b || node[k] < 0) continue;
            const size_t ia = k < a ? tri_index(a, k) : tri_index(k, a), ib = k < b ? tri_index(b, k) : tri_index(k, b);
            const float t = __fadd_rn(D[ia], D[ib]);
            const float nd = __fmul_rn(__fsub_rn(t, dab), 0.5f);
            s[k] = __fadd_rn(__fsub_rn(s[k], t), nd);
            D[ia] = nd;
        }
        if (gtid == 0) {
            out_tree[2 * it] = node[a];
            out_tree[2 * it + 1] = node[b];
            node[a] = (int)(n + it);
            node[b] = -1;
            s[b] = __int_as_float(0x7fc00000);                    // NaN: no pair of b is a candidate any more
        }
        pa = a;
        grid.sync();
    }
    // the last two clusters, in position order (:117)
    if (gtid == 0) {
        int first = -1;
        for (uint32_t k = 0; k < R; ++k) {
            if (node[k] < 0) continue;
            if (first < 0) first = node[k];
            else { out_tree[2 * (n - 2)] = first; out_tree[2 * (n - 2) + 1] = node[k]; break; }
        }
    }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------

struct UnionFind {
    std::vector<uint32_t> parent;
    explicit UnionFind(uint32_t n) : parent(n) { std::iota(parent.begin(), parent.end(), 0u); }
    uint32_t find(uint32_t x)
    {
        while (parent[x] != x) { parent[x] = parent[parent[x]]; x = parent[x]; }
        return x;
    }
};

// Development knobs, read on every call.  FAMSA_TREE_MAX_BLOCKS=<k> caps the cooperative grids of k_prim, k_upgma and
// k_nj at k blocks, so that a few thousand sequences reach what otherwise only sets above ~135 k do on an H100: threads
// that own several sequences, warps that scan dozens of NJ rows.  It only ever lowers a grid; unset, 0 or unparsable
// changes nothing.  FAMSA_TREE_DEBUG: one `[coop] <kernel> n=<n> blocks=<grid>` line per cooperative launch on stderr.
static uint32_t coop_cap(uint32_t nblk)
{
    const char* e = getenv("FAMSA_TREE_MAX_BLOCKS");
    if (!e) return nblk;
    char* end = nullptr;
    const long k = strtol(e, &end, 10);
    if (end == e || *end || k <= 0) return nblk;
    return (uint32_t)std::min<long>(nblk, k);
}
static void coop_debug(const char* kernel, uint32_t n, uint32_t nblk)
{
    if (getenv("FAMSA_TREE_DEBUG")) fprintf(stderr, "[coop] %s n=%u blocks=%u\n", kernel, n, nblk);
}

// Blocks of 1024 threads for a cooperative kernel over n items: all co-resident, no more than the items need
static int coop_blocks(famsa_ctx* ctx, const void* fn, uint32_t n, uint32_t& nblk)
{
    int per_sm = 0;
    FB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, 1024, 0));
    nblk = coop_cap(std::max(1u, std::min((uint32_t)(ctx->sm_count * std::max(per_sm, 1)), (n + 1023) / 1024)));
    return FAMSA_OK;
}

// The distance triangle of d_tri (width eb) into d_dist_tri, which the caller has reserved
template <class T>
static int dist_triangle(famsa_ctx* ctx, const void* d_tri, int eb, int kind, const T* d_pow, cudaStream_t st)
{
    LcsState& S = ctx->lcs;
    const uint32_t n = S.n;
    k_dist_tri<T><<<n - 1, 256, 0, st>>>(d_tri, eb, S.d_raw_len.as<uint32_t>(), d_pow, kind, S.d_dist_tri.as<T>());
    FB_CUDA(cudaGetLastError());
    ctx->launches++;
    return FAMSA_OK;
}

// The seed rows against the sequences of mask groups [g_begin, g_end), packed (k_assign_packed) into d_packed
static int assign_packed(famsa_ctx* ctx, const uint32_t* h_seed_ids, uint32_t n_seeds, int kind, uint32_t g_begin, uint32_t g_end,
                         long long* d_packed, cudaStream_t st)
{
    LcsState& S = ctx->lcs;
    const uint32_t n = S.n;
    const int eb = S.elem_bytes();
    FB_TRY(S.d_assign_lcs.reserve((size_t)eb * n * n_seeds));
    FB_TRY(S.d_ids_a.reserve(sizeof(uint32_t) * n_seeds));
    FB_CUDA(cudaMemcpyAsync(S.d_ids_a.p, h_seed_ids, sizeof(uint32_t) * n_seeds, cudaMemcpyHostToDevice, st));
    // seed k is the row (seq0) of its distance vector, every sequence a column: exactly famsa_lcs_rows
    FB_TRY(lcs_rows(ctx, h_seed_ids, n_seeds, nullptr, n, S.d_assign_lcs.p, eb, st, g_begin, g_end));
    k_assign_packed<<<(n + 255) / 256, 256, 0, st>>>(S.d_assign_lcs.p, eb, n, n_seeds, S.d_ids_a.as<uint32_t>(),
                                                    S.d_raw_len.as<uint32_t>(), S.d_pow075.as<float>(), kind,
                                                    S.d_invperm.as<uint32_t>(), g_begin, g_end, d_packed);
    FB_CUDA(cudaGetLastError());
    ctx->launches++;
    return FAMSA_OK;
}

int lcs_assign(famsa_ctx* ctx, const uint32_t* h_seed_ids, uint32_t n_seeds, int kind, uint32_t* h_assign, float* h_mind)
{
    LcsState& S = ctx->lcs;
    cudaStream_t st = ctx->stream;
    const uint32_t n = S.n;
    FB_TRY(S.d_out_stage.reserve(sizeof(unsigned long long) * n));
    FB_TRY(assign_packed(ctx, h_seed_ids, n_seeds, kind, 0, S.n_groups, S.d_out_stage.as<long long>(), st));
    std::vector<unsigned long long> packed(n);
    FB_CUDA(cudaMemcpyAsync(packed.data(), S.d_out_stage.p, sizeof(unsigned long long) * n, cudaMemcpyDeviceToHost, st));
    FB_CUDA(cudaStreamSynchronize(st));
    for (uint32_t j = 0; j < n; ++j) {
        const uint32_t bits = (uint32_t)(packed[j] >> 32);
        h_assign[j] = (uint32_t)packed[j];
        memcpy(&h_mind[j], &bits, sizeof(float));
    }
    return FAMSA_OK;
}

// famsa_lcs_assign_shard: the seed rows against this shard's slice of the mask groups only, packed for a MIN all-reduce
int lcs_assign_shard(famsa_ctx* ctx, const uint32_t* h_seed_ids, uint32_t n_seeds, int kind, uint32_t shard, uint32_t n_shards,
                     long long* d_packed, cudaStream_t st)
{
    LcsState& S = ctx->lcs;
    const uint32_t g_begin = (uint32_t)((unsigned long long)S.n_groups * shard / n_shards);
    const uint32_t g_end = (uint32_t)((unsigned long long)S.n_groups * (shard + 1) / n_shards);
    FB_TRY(assign_packed(ctx, h_seed_ids, n_seeds, kind, g_begin, g_end, d_packed, st));
    S.last_pairs = 0;
    for (uint32_t g = g_begin; g < g_end; ++g) S.last_pairs += (uint64_t)std::min(32u, S.n - g * 32) * n_seeds;
    return FAMSA_OK;
}

// Parallel MST (see the kernels above) into `edges`; prim_replay then gives Prim's visiting order.  Expects the
// triangle in d_lcs_tri and the pow table in d_pow075_f64.
static int prim_boruvka(famsa_ctx* ctx, int kind, int eb, std::vector<MstEdge>& edges)
{
    LcsState& S = ctx->lcs;
    cudaStream_t st = ctx->stream;
    const uint32_t n = S.n;
    const uint32_t n_chunks = (n + kMstChunk - 1) / kMstChunk;
    FB_TRY(S.d_dist_tri.reserve(tri_index(n, 0) * sizeof(double)));
    FB_TRY(S.d_mst_comp.reserve(sizeof(uint32_t) * n));
    FB_TRY(S.d_mst_best.reserve(sizeof(EdgeMin) * n));
    FB_TRY(S.d_mst_part.reserve(sizeof(EdgeMin) * (size_t)n_chunks * n));
    FB_TRY(dist_triangle<double>(ctx, S.d_lcs_tri.p, eb, kind, S.d_pow075_f64.as<double>(), st));
    double* d_dtri = S.d_dist_tri.as<double>();
    uint32_t* d_comp = S.d_mst_comp.as<uint32_t>();
    EdgeMin* d_best = S.d_mst_best.as<EdgeMin>();
    EdgeMin* d_part = S.d_mst_part.as<EdgeMin>();

    UnionFind uf(n);
    std::vector<uint32_t> comp(n);
    std::iota(comp.begin(), comp.end(), 0u);
    edges.clear();
    edges.reserve(n - 1);
    std::vector<EdgeMin> best(n), cbest(n);
    uint32_t n_comp = n;
    while (n_comp > 1) {
        FB_CUDA(cudaMemcpyAsync(d_comp, comp.data(), sizeof(uint32_t) * n, cudaMemcpyHostToDevice, st));
        k_mst_rows<<<n, 256, 0, st>>>(d_dtri, n, d_comp, d_best);
        k_mst_cols<<<dim3((n + 31) / 32, n_chunks), 256, 0, st>>>(d_dtri, n, d_comp, d_part);
        k_mst_combine<<<(n + 255) / 256, 256, 0, st>>>(n, n_chunks, d_part, d_best);
        FB_CUDA(cudaGetLastError());
        ctx->launches += 3;
        FB_CUDA(cudaMemcpyAsync(best.data(), d_best, sizeof(EdgeMin) * n, cudaMemcpyDeviceToHost, st));
        FB_CUDA(cudaStreamSynchronize(st));
        // every component's smallest outgoing edge ...
        for (uint32_t v = 0; v < n; ++v) cbest[v].d = kEdgeNone;
        for (uint32_t v = 0; v < n; ++v) {
            if (!(best[v].d < kEdgeNone)) continue;
            EdgeMin& c = cbest[comp[v]];
            if (cand_less(best[v], c)) c = best[v];
        }
        // ... joins two components (the edge order is strict, so no cycle can close)
        const uint32_t before = n_comp;
        for (uint32_t c = 0; c < n; ++c) {
            if (!(cbest[c].d < kEdgeNone)) continue;
            uint32_t a, b;
            edge_ids(cbest[c].k, a, b);
            const uint32_t ra = uf.find(a), rb = uf.find(b);
            if (ra == rb) continue;                                 // both sides elected the same edge
            uf.parent[ra] = rb;
            edges.push_back(MstEdge{a, b, cbest[c].d});
            --n_comp;
        }
        if (n_comp == before) { set_error("famsa_lcs_prim: no progress in a Boruvka round"); return FAMSA_E_CUDA; }
        for (uint32_t v = 0; v < n; ++v) comp[v] = uf.find(v);
    }
    return FAMSA_OK;
}

// Prim's visiting order from vertex 0, replayed on the tree (MSTPrim.cpp:366-386 restricted to tree edges)
int prim_replay(const std::vector<MstEdge>& edges, int32_t* h_from, int32_t* h_to, double* h_dist, int32_t* h_order)
{
    const uint32_t n = (uint32_t)edges.size() + 1;
    using Item = std::tuple<double, unsigned long long, uint32_t>;
    std::vector<std::vector<Item>> adj(n);
    for (const MstEdge& e : edges) {
        const unsigned long long key = edge_key(e.a, e.b);
        adj[e.a].emplace_back(e.d, key, e.b);
        adj[e.b].emplace_back(e.d, key, e.a);
    }
    std::priority_queue<Item, std::vector<Item>, std::greater<Item>> heap;
    for (uint32_t v = 0; v < n; ++v) h_order[v] = (int32_t)n;
    h_order[0] = 0;
    for (const Item& it : adj[0]) heap.push(it);
    uint32_t step = 0;
    while (!heap.empty()) {
        const Item it = heap.top();
        heap.pop();
        const uint32_t v = std::get<2>(it);
        if (h_order[v] != (int32_t)n) continue;
        uint32_t lo, hi;
        edge_ids(std::get<1>(it), lo, hi);
        h_from[step] = (int32_t)lo;
        h_to[step] = (int32_t)hi;
        h_dist[step] = std::get<0>(it);
        h_order[v] = (int32_t)++step;
        for (const Item& nx : adj[v])
            if (h_order[std::get<2>(nx)] == (int32_t)n) heap.push(nx);
    }
    if (step != n - 1) { set_error("famsa_lcs_prim: the replay did not reach every sequence"); return FAMSA_E_CUDA; }
    return FAMSA_OK;
}

// The MST of d_lcs_tri under MSTPrim's edge order.  The Boruvka rounds fill `edges` when `parallel` is set and
// FAMSA_PRIM_SEQUENTIAL is not; otherwise, or when their float64 triangle does not fit, the sequential vertex loop
// k_prim<kSlink> runs (on the side rows too for MSTPrim) and `edges` stays empty: edge k joins from[k] < to[k] at
// dist[k] and was added with the (k+1)-th vertex, order[i] = visiting position (not copied when order is NULL).
template <bool kSlink>
static int mst(famsa_ctx* ctx, int kind, bool parallel, std::vector<MstEdge>& edges, int32_t* from, int32_t* to, double* dist,
               int32_t* order)
{
    LcsState& S = ctx->lcs;
    cudaStream_t st = ctx->stream;
    const uint32_t n = S.n;
    const int eb = S.elem_bytes();
    edges.clear();
    if (parallel && n >= 2 && !getenv("FAMSA_PRIM_SEQUENTIAL")) {
        const int rc = prim_boruvka(ctx, kind, eb, edges);
        if (rc != FAMSA_E_NOMEM) return rc;                         // no room for the float64 triangle: sequential loop
        edges.clear();
        set_error("");                                              // the failed reservation is not this call's outcome
    }
    FB_TRY(S.d_tree_state.reserve((sizeof(PrimState) + 1) * (size_t)n + 64));
    FB_TRY(S.d_tree_out.reserve((sizeof(int) * 3 + sizeof(double)) * (size_t)n + 64));
    PrimState* d_state = S.d_tree_state.as<PrimState>();
    unsigned char* d_vis = reinterpret_cast<unsigned char*>(d_state + n);
    double* d_dist = S.d_tree_out.as<double>();
    int* d_from = reinterpret_cast<int*>(d_dist + n);
    int* d_to = d_from + n;
    int* d_order = d_to + n;
    uint32_t nblk = 0;
    FB_TRY(coop_blocks(ctx, (const void*)k_prim<kSlink>, n, nblk));
    FB_TRY(S.d_tree_cand.reserve(sizeof(PrimCand) * 2 * nblk));
    const void* a_tri = S.d_lcs_tri.p; int a_eb = eb; uint32_t a_n = n;
    const uint32_t* a_len = S.d_raw_len.as<uint32_t>(); const double* a_pow = S.d_pow075_f64.as<double>();
    int a_kind = kind;
    const int* a_sidx = kSlink ? nullptr : S.d_side_idx.as<int>();
    const uint32_t* a_side = kSlink ? nullptr : S.d_side_rows.as<uint32_t>();
    PrimCand* a_cand = S.d_tree_cand.as<PrimCand>();
    void* args[] = {&a_tri, &a_eb, &a_n, &a_len, &a_pow, &a_kind, &a_sidx, &a_side, &d_state, &d_vis,
                    &a_cand, &d_from, &d_to, &d_dist, &d_order};
    coop_debug(kSlink ? "k_prim<1>" : "k_prim<0>", n, nblk);
    FB_CUDA(cudaLaunchCooperativeKernel((void*)k_prim<kSlink>, dim3(nblk), dim3(1024), args, 0, st));
    ctx->launches++;
    if (n > 1) {
        FB_CUDA(cudaMemcpyAsync(from, d_from, sizeof(int) * (n - 1), cudaMemcpyDeviceToHost, st));
        FB_CUDA(cudaMemcpyAsync(to, d_to, sizeof(int) * (n - 1), cudaMemcpyDeviceToHost, st));
        FB_CUDA(cudaMemcpyAsync(dist, d_dist, sizeof(double) * (n - 1), cudaMemcpyDeviceToHost, st));
    }
    if (order) FB_CUDA(cudaMemcpyAsync(order, d_order, sizeof(int) * n, cudaMemcpyDeviceToHost, st));
    FB_CUDA(cudaStreamSynchronize(st));
    return FAMSA_OK;
}

int lcs_prim(famsa_ctx* ctx, int kind, int32_t* h_from, int32_t* h_to, double* h_dist, int32_t* h_order,
             std::vector<MstEdge>& tree)
{
    LcsState& S = ctx->lcs;
    cudaStream_t st = ctx->stream;
    const uint32_t n = S.n;
    const int eb = S.elem_bytes();
    FB_TRY(S.d_lcs_tri.reserve(std::max<size_t>(tri_index(n, 0), 1) * eb));
    // the true-LCS triangle (orientation-free) plus the own rows of the flagged sequences
    FB_TRY(lcs_triangle(ctx, 0, n, S.d_lcs_tri.p, eb, st, nullptr, 1, nullptr, /*quirk_fixups=*/false));
    FB_TRY(lcs_side_rows(ctx, st));
    FB_TRY(lcs_pow075_f64(ctx, st));
    // with flagged sequences the distances are not symmetric: only the sequential loop follows MSTPrim then
    return mst<false>(ctx, kind, S.h_quirky.empty(), tree, h_from, h_to, h_dist, h_order);
}

// famsa_lcs_slink: SingleLinkage<>::run (SingleLinkage.cpp:30-189) orders distances by (distance, ids_to_uint64
// descending), the strict order of the MST engines above, so its hierarchy is the unique MST merged in Kruskal order.
// The triangle is the one SLINK reads (row i = seq0 against j < i, dropped-carry rows exact), so the distances are
// symmetric and the Boruvka rounds serve whatever the set.  `edges` gets the n-1 MST edges in no particular order;
// slink_labels names them.
int lcs_slink(famsa_ctx* ctx, int kind, std::vector<MstEdge>& edges)
{
    LcsState& S = ctx->lcs;
    cudaStream_t st = ctx->stream;
    const uint32_t n = S.n;
    const int eb = S.elem_bytes();
    edges.clear();
    if (n < 2) return FAMSA_OK;
    FB_TRY(S.d_lcs_tri.reserve(tri_index(n, 0) * eb));
    FB_TRY(lcs_triangle(ctx, 0, n, S.d_lcs_tri.p, eb, st, nullptr, 1, nullptr, /*quirk_fixups=*/true));
    FB_TRY(lcs_pow075_f64(ctx, st));
    std::vector<int32_t> from(n - 1), to(n - 1);
    std::vector<double> dist(n - 1);
    FB_TRY(mst<true>(ctx, kind, true, edges, from.data(), to.data(), dist.data(), nullptr));
    if (edges.empty())
        for (uint32_t k = 0; k + 1 < n; ++k) edges.push_back(MstEdge{(uint32_t)from[k], (uint32_t)to[k], dist[k]});
    return FAMSA_OK;
}

// SLINK's tree from its MST (famsa_b200/mst.py slink_tree is the same in numpy): the edges in (distance, key) order; for
// the edge joining clusters whose largest members are a < b, emit (node(a), node(b)) as merge k and key the merged
// cluster, node n + k, by b.  This is what SLINK's stable_sort of lambda and its index relabelling produce (:166-188).
void slink_labels(std::vector<MstEdge> edges, uint32_t n, int32_t* tree)
{
    std::sort(edges.begin(), edges.end(), [](const MstEdge& x, const MstEdge& y) {
        return x.d < y.d || (x.d == y.d && edge_key(x.a, x.b) < edge_key(y.a, y.b));
    });
    UnionFind uf(n);
    std::vector<uint32_t> top(n), node(n);
    std::iota(top.begin(), top.end(), 0u);
    std::iota(node.begin(), node.end(), 0u);
    for (size_t k = 0; k < edges.size(); ++k) {
        const uint32_t ra = uf.find(edges[k].a), rb = uf.find(edges[k].b);
        const uint32_t lo = std::min(top[ra], top[rb]), hi = std::max(top[ra], top[rb]);
        tree[2 * k] = (int32_t)node[lo];
        tree[2 * k + 1] = (int32_t)node[hi];
        node[hi] = n + (uint32_t)k;
        uf.parent[ra] = rb;
        top[rb] = hi;
    }
}

// famsa_lcs_upgma: LCS triangle (row = seq0, as calculateDistanceVector builds it) -> float distances -> the agglomeration
int lcs_upgma(famsa_ctx* ctx, int kind, int modified, int32_t* h_tree, const void* d_tri_in, int tri_eb)
{
    LcsState& S = ctx->lcs;
    cudaStream_t st = ctx->stream;
    const uint32_t n = S.n;
    const int eb = d_tri_in ? tri_eb : S.elem_bytes();
    const void* d_tri = d_tri_in;
    if (!d_tri) {
        FB_TRY(S.d_lcs_tri.reserve(std::max<size_t>(tri_index(n, 0), 1) * eb));
        FB_TRY(lcs_triangle(ctx, 0, n, S.d_lcs_tri.p, eb, st));
        d_tri = S.d_lcs_tri.p;
    }
    FB_TRY(S.d_dist_tri.reserve(std::max<size_t>(tri_index(n, 0), 1) * sizeof(float)));
    FB_TRY(S.d_tree_state.reserve((sizeof(float) + sizeof(uint32_t) + sizeof(int)) * (size_t)n + 64));
    FB_TRY(S.d_tree_out.reserve(sizeof(int) * 2 * (size_t)n + 64));
    float* d_mind = S.d_tree_state.as<float>();
    uint32_t* d_nn = reinterpret_cast<uint32_t*>(d_mind + n);
    int* d_node = reinterpret_cast<int*>(d_nn + n);
    int* d_tree = S.d_tree_out.as<int>();
    int* d_status = d_tree + 2 * (size_t)(n - 1);
    FB_TRY(dist_triangle<float>(ctx, d_tri, eb, kind, S.d_pow075.as<float>(), st));
    float* d_dist = S.d_dist_tri.as<float>();
    k_upgma_init<<<n, 256, 0, st>>>(d_dist, n, d_mind, d_nn, d_node);
    FB_CUDA(cudaGetLastError());
    FB_CUDA(cudaMemsetAsync(d_status, 0, sizeof(int), st));
    ctx->launches++;
    {
        const void* fn = modified ? (const void*)k_upgma<true> : (const void*)k_upgma<false>;
        uint32_t nblk = 0;
        FB_TRY(coop_blocks(ctx, fn, n, nblk));
        FB_TRY(S.d_tree_cand.reserve(sizeof(unsigned long long) * 2 * nblk));
        uint32_t a_n = n;
        unsigned long long* a_cand = S.d_tree_cand.as<unsigned long long>();
        void* args[] = {&d_dist, &a_n, &d_mind, &d_nn, &d_node, &a_cand, &d_tree, &d_status};
        coop_debug(modified ? "k_upgma<1>" : "k_upgma<0>", n, nblk);
        FB_CUDA(cudaLaunchCooperativeKernel(fn, dim3(nblk), dim3(1024), args, 0, st));
        ctx->launches++;
    }
    int status = 0;
    FB_CUDA(cudaMemcpyAsync(h_tree, d_tree, sizeof(int) * 2 * (size_t)(n - 1), cudaMemcpyDeviceToHost, st));
    FB_CUDA(cudaMemcpyAsync(&status, d_status, sizeof(int), cudaMemcpyDeviceToHost, st));
    FB_CUDA(cudaStreamSynchronize(st));
    if (status) { set_error("famsa_lcs_upgma: no finite distance left between two clusters (sequences without a common residue)"); return FAMSA_E_INVALID; }
    return FAMSA_OK;
}

// famsa_lcs_nj: the LCS triangle UPGMA reads -> float distances (calculateDistanceMatrix, NeighborJoining.cpp:14-18) ->
// the initial sums -> the agglomeration.  Needs n >= 2.
int lcs_nj(famsa_ctx* ctx, int kind, int32_t* h_tree)
{
    LcsState& S = ctx->lcs;
    cudaStream_t st = ctx->stream;
    const uint32_t n = S.n;
    const int eb = S.elem_bytes();
    FB_TRY(S.d_lcs_tri.reserve(tri_index(n, 0) * eb));
    FB_TRY(S.d_dist_tri.reserve(tri_index(n, 0) * sizeof(float)));
    FB_TRY(S.d_nj_half.reserve(tri_index(n / 2 + 1, 0) * sizeof(float)));
    FB_TRY(S.d_tree_state.reserve((sizeof(float) * 2 + sizeof(int) * 2 + sizeof(uint32_t)) * (size_t)n + 64));
    FB_TRY(S.d_tree_out.reserve(sizeof(int) * 2 * (size_t)n + 64));
    float* d_s0 = S.d_tree_state.as<float>();
    float* d_s1 = d_s0 + n;
    int* d_node0 = reinterpret_cast<int*>(d_s1 + n);
    int* d_node1 = d_node0 + n;
    uint32_t* d_map = reinterpret_cast<uint32_t*>(d_node1 + n);
    uint32_t* d_misc = d_map + n;
    int* d_tree = S.d_tree_out.as<int>();
    int* d_status = d_tree + 2 * (size_t)(n - 1);
    FB_TRY(lcs_triangle(ctx, 0, n, S.d_lcs_tri.p, eb, st));
    FB_TRY(dist_triangle<float>(ctx, S.d_lcs_tri.p, eb, kind, S.d_pow075.as<float>(), st));
    float* d_dist = S.d_dist_tri.as<float>();
    float* d_half = S.d_nj_half.as<float>();
    k_nj_sums<<<(n + 127) / 128, 128, 0, st>>>(d_dist, n, d_s0, d_node0);
    FB_CUDA(cudaGetLastError());
    FB_CUDA(cudaMemsetAsync(d_status, 0, sizeof(int), st));
    ctx->launches++;
    // the scan of the first merges reads the whole triangle: blocks for every 64 rows, all co-resident
    int per_sm = 0;
    FB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, (const void*)k_nj, 1024, 0));
    const uint32_t nblk = coop_cap(std::max(1u, std::min((uint32_t)(ctx->sm_count * std::max(per_sm, 1)), (n + 63) / 64)));
    FB_TRY(S.d_tree_cand.reserve(sizeof(NjCand) * nblk));
    uint32_t a_n = n;
    NjCand* a_cand = S.d_tree_cand.as<NjCand>();
    void* args[] = {&d_dist, &d_half, &a_n, &d_s0, &d_s1, &d_node0, &d_node1, &d_map, &d_misc, &a_cand, &d_tree, &d_status};
    coop_debug("k_nj", n, nblk);
    FB_CUDA(cudaLaunchCooperativeKernel((const void*)k_nj, dim3(nblk), dim3(1024), args, 0, st));
    ctx->launches++;
    int status = 0;
    FB_CUDA(cudaMemcpyAsync(h_tree, d_tree, sizeof(int) * 2 * (size_t)(n - 1), cudaMemcpyDeviceToHost, st));
    FB_CUDA(cudaMemcpyAsync(&status, d_status, sizeof(int), cudaMemcpyDeviceToHost, st));
    FB_CUDA(cudaStreamSynchronize(st));
    if (status) {
        set_error("famsa_lcs_nj: a step without a candidate pair (every Q is NaN or >= FLT_MAX: sequences without a common residue)");
        return FAMSA_E_INVALID;
    }
    return FAMSA_OK;
}

} // namespace fb
