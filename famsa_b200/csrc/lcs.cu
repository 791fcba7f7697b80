// HP-1: all-pairs bit-parallel LCS length on sm_90a.
//
// Replaces CLCSBP::GetLCSBP and its scalar/AVX/AVX2/AVX512/NEON back-ends
// (reference src/lcs/lcsbp.cpp:48-368, src/lcs/lcsbp_classic.h:67-221,
// src/simd/lcsbp_avx2_intr.h:127-395) together with CSequence::ComputeBitMasks
// (src/core/sequence.cpp:190-201) behind the batch drivers of
// src/tree/AbstractTreeGenerator.hpp:131-398.  See DESIGN.md section 3 for the layout.
//
// Design (not a translation of the CPU code):
//   * Sequences are re-ordered by descending length and cut into MASK GROUPS of 32.  A group's
//     per-symbol position bit-vectors are stored lane-interleaved in 32-bit limbs ("blob"), so
//     that lane L of a warp owns sequence L of the group and every mask fetch of the warp is one
//     conflict-free LDS.128/LDS.64/LDS.32.
//   * One CTA = one tile = (mask group, a run of streamed sequences).  The blob is staged to
//     shared memory with one TMA bulk copy (cp.async.bulk + mbarrier).  Each warp streams one
//     sequence at a time: the residue is warp-uniform, each lane advances the Hyyro recurrence
//     for its own (mask sequence, streamed sequence) pair with the bit-vector X[] held in
//     registers and the carry rippling through an add.cc/addc.cc chain.  32 pairs per warp.
//   * The tile kernel computes the TRUE LCS, which is symmetric, so either sequence of a pair may
//     be the mask side.  The reference's result differs from the true LCS only when its row
//     sequence (seq0) owns an all-ones 64-bit mask word (dropped carry, lcsbp_classic.h:55-56);
//     those rows -- and rows too long for the register-resident kernel -- are recomputed by
//     k_lcs_exact, which follows the reference recurrence word for word.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <numeric>

#include "ctx.h"
#include "triangle_dev.cuh"

namespace fb {

constexpr int kMaskRows = 21;     // symbols 0..19 + one all-zero row shared by every other code
constexpr int kNoMatch = 20;      // device residue code for "never matches" (B, Z, X, *, padding)
constexpr int kTileWarps = 4;
constexpr int kSeqPerWarp = 8;
constexpr int kTileQ = kTileWarps * kSeqPerWarp;   // streamed sequences per tile
constexpr int kMaxNL = 64;        // limbs the register-resident kernel is instantiated for (2048 aa)

__host__ __device__ inline uint32_t blob_words(uint32_t nl) { return kMaskRows * 32u * nl; }

// word index of (symbol c, limb w, lane) inside a group's blob: limbs are grouped in fours
// (LDS.128), the remaining 1..3 limbs as LDS.32 / LDS.64 / LDS.64+LDS.32.
__host__ __device__ inline uint32_t blob_index(uint32_t nl, uint32_t c, uint32_t w, uint32_t lane)
{
    const uint32_t nq = nl / 4, tail = nl % 4;
    const uint32_t base = c * 32u * nl;
    if (w < 4 * nq) return base + ((w / 4) * 32 + lane) * 4 + (w % 4);
    const uint32_t k = w - 4 * nq;
    const uint32_t tb = base + nq * 128;
    if (tail == 1) return tb + lane;
    if (tail == 2) return tb + lane * 2 + k;
    return k < 2 ? tb + lane * 2 + k : tb + 64 + lane;
}

static uint32_t nl_for_len(uint32_t max_len)
{
    uint32_t req = (max_len + 31) / 32;
    if (req == 0) req = 1;
    if (req <= 32) return req;
    if (req <= kMaxNL) return (req + 3) / 4 * 4;
    return 0;
}

// ------------------------------------------------------------------------------------------------
// upload-time kernels
// ------------------------------------------------------------------------------------------------

// One warp per sequence (sorted position): copy residues into the 16-byte padded device layout,
// mapping every code outside 0..19 to kNoMatch.
__global__ void k_repack(const int8_t* __restrict__ raw, const uint64_t* __restrict__ raw_off,
                         const uint32_t* __restrict__ raw_len, const uint32_t* __restrict__ perm,
                         const uint32_t* __restrict__ code_off, uint8_t* __restrict__ codes,
                         uint32_t n)
{
    const uint32_t p = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32;
    if (p >= n) return;
    const uint32_t lane = threadIdx.x % 32;
    const uint32_t a = perm[p];
    const uint32_t len = raw_len[a];
    const int8_t* src = raw + raw_off[a];
    uint8_t* dst = codes + (size_t)code_off[p] * 16;
    const uint32_t padded = (len + 15) / 16 * 16;
    for (uint32_t i = lane; i < padded; i += 32) {
        int c = i < len ? src[i] : kNoMatch;
        dst[i] = (c >= 0 && c < 20) ? (uint8_t)c : (uint8_t)kNoMatch;
    }
}

// One CTA per mask group: build the lane-interleaved blob in shared memory, write it out.
__global__ void k_build_blob(const uint8_t* __restrict__ codes, const uint32_t* __restrict__ code_off,
                             const uint32_t* __restrict__ len_sorted,
                             const uint64_t* __restrict__ group_blob, const uint32_t* __restrict__ group_nl,
                             uint32_t* __restrict__ blob, uint32_t n)
{
    extern __shared__ uint32_t sm[];
    const uint32_t g = blockIdx.x;
    const uint32_t nl = group_nl[g];
    if (nl == 0) return;
    const uint32_t words = blob_words(nl);
    for (uint32_t i = threadIdx.x; i < words; i += blockDim.x) sm[i] = 0;
    __syncthreads();
    const uint32_t warp = threadIdx.x / 32, lane = threadIdx.x % 32, nwarps = blockDim.x / 32;
    for (uint32_t s = warp; s < 32; s += nwarps) {
        const uint32_t p = g * 32 + s;
        if (p >= n) continue;
        const uint32_t len = len_sorted[p];
        const uint8_t* src = codes + (size_t)code_off[p] * 16;
        for (uint32_t pos = lane; pos < len; pos += 32) {
            const uint32_t c = src[pos];
            if (c < 20) atomicOr(&sm[blob_index(nl, c, pos / 32, s)], 1u << (pos % 32));
        }
    }
    __syncthreads();
    uint32_t* dst = blob + group_blob[g];
    for (uint32_t i = threadIdx.x; i < words; i += blockDim.x) dst[i] = sm[i];
}

// flag[p] = 1 if some 64-bit mask word of sequence p is all ones, i.e. 64 identical matching
// residues starting at a multiple of 64 (the dropped-carry corner needs exactly that).
__global__ void k_quirky(const uint8_t* __restrict__ codes, const uint32_t* __restrict__ code_off,
                         const uint32_t* __restrict__ len_sorted, uint8_t* __restrict__ flag, uint32_t n)
{
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    const uint32_t len = len_sorted[p];
    const uint8_t* src = codes + (size_t)code_off[p] * 16;
    uint8_t f = 0;
    for (uint32_t w = 0; w + 64 <= len; w += 64) {
        const uint8_t c = src[w];
        if (c >= 20) continue;
        bool all = true;
        for (uint32_t k = 1; k < 64; ++k) all &= (src[w + k] == c);
        if (all) f = 1;
    }
    flag[p] = f;
}

// ------------------------------------------------------------------------------------------------
// the tile kernel
// ------------------------------------------------------------------------------------------------

struct TileParams {
    const uint32_t* blob;
    const uint64_t* group_blob;
    const uint3* tiles;            // {group, q_begin, q_end}
    const uint8_t* codes;
    const uint32_t* code_off;
    const uint32_t* len_sorted;
    const uint32_t* perm;
    const uint32_t* refpos;        // rows mode: streamed item q -> sorted position
    void* out;
    uint64_t tri_base;
    uint32_t n;
    uint32_t row_begin, row_end;
    uint32_t ld_res;
    int elem_bytes;
    int rows_mode;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p)
{
    return (uint32_t)__cvta_generic_to_shared(p);
}

// Shared-memory byte addresses of the lane's words in symbol row 0 of the blob (blob_index with c = 0): the quads,
// the 1- or 2-limb tail and, for TAIL == 3, the third tail limb.  Row c is these plus c * row bytes: one IMAD per
// address and residue, on the FMA pipe, instead of shifts and adds on the integer ALU pipe, which the recurrence keeps busy.
template <int NL>
struct BlobLaneAddr {
    uint32_t quad, tail, tail3;
    __device__ __forceinline__ BlobLaneAddr(uint32_t sm_base, uint32_t lane)
    {
        constexpr uint32_t NQ = NL / 4, TAIL = NL % 4;
        quad = sm_base + lane * 16;
        tail = sm_base + NQ * 512 + lane * (TAIL == 1 ? 4 : 8);
        tail3 = sm_base + NQ * 512 + 256 + lane * 4;
    }
};

__device__ __forceinline__ uint4 lds128(uint32_t a)
{
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
    return v;
}
__device__ __forceinline__ uint2 lds64(uint32_t a)
{
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a));
    return v;
}
__device__ __forceinline__ uint32_t lds32(uint32_t a)
{
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
}

// One Hyyro step for 32*NL cells of one pair: X' = (X + (X & M)) | (X & ~M), true carries.  c = the streamed residue.
template <int NL>
__device__ __forceinline__ void lcs_step(uint32_t (&X)[NL], const BlobLaneAddr<NL>& A, uint32_t c)
{
    constexpr int NQ = NL / 4, TAIL = NL % 4;
    constexpr uint32_t kRowBytes = 32u * NL * 4u;
    uint32_t m[NL];
    const uint32_t qa = c * kRowBytes + A.quad;
#pragma unroll
    for (int q = 0; q < NQ; ++q) {
        const uint4 v = lds128(qa + q * 512);
        m[4 * q] = v.x; m[4 * q + 1] = v.y; m[4 * q + 2] = v.z; m[4 * q + 3] = v.w;
    }
    if (TAIL == 1) m[4 * NQ] = lds32(c * kRowBytes + A.tail);
    if (TAIL >= 2) {
        const uint2 v = lds64(c * kRowBytes + A.tail);
        m[4 * NQ] = v.x; m[4 * NQ + 1] = v.y;
    }
    if (TAIL == 3) m[4 * NQ + 2] = lds32(c * kRowBytes + A.tail3);

    uint32_t tb[NL], s[NL];
#pragma unroll
    for (int w = 0; w < NL; ++w) tb[w] = X[w] & m[w];
    // carry chain: one IADD3 + (NL-1) IADD3.X; the carry out of the last limb is discarded
    asm volatile("add.cc.u32 %0, %1, %2;" : "=r"(s[0]) : "r"(X[0]), "r"(tb[0]));
#pragma unroll
    for (int w = 1; w < NL; ++w)
        asm volatile("addc.cc.u32 %0, %1, %2;" : "=r"(s[w]) : "r"(X[w]), "r"(tb[w]));
#pragma unroll
    for (int w = 0; w < NL; ++w) X[w] = s[w] | (X[w] ^ tb[w]);
}

template <int NL>
__global__ void __launch_bounds__(kTileWarps * 32) k_lcs_tile(const TileParams P)
{
    extern __shared__ __align__(128) uint32_t sm[];
    __shared__ __align__(8) uint64_t bar;

    const uint3 tile = P.tiles[blockIdx.x];
    const uint32_t g = tile.x;
    constexpr uint32_t kBlobBytes = kMaskRows * 32u * NL * 4u;

    // stage the group's mask blob: one TMA bulk copy, completion on an mbarrier
    if (threadIdx.x == 0) {
        const uint32_t b = smem_u32(&bar);
        asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(b));
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"(kBlobBytes) : "memory");
        asm volatile(
            "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                smem_u32(sm)),
            "l"(P.blob + P.group_blob[g]), "r"(kBlobBytes), "r"(b)
            : "memory");
    }
    __syncthreads();
    {
        const uint32_t b = smem_u32(&bar);
        uint32_t done = 0;
        while (!done) {
            asm volatile(
                "{\n\t.reg .pred p;\n\t"
                "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\t"
                "selp.u32 %0, 1, 0, p;\n\t}"
                : "=r"(done)
                : "r"(b)
                : "memory");
        }
    }

    const uint32_t lane = threadIdx.x % 32, warp = threadIdx.x / 32;
    const uint32_t p = g * 32 + lane;
    const uint32_t a = p < P.n ? P.perm[p] : 0xffffffffu;
    const BlobLaneAddr<NL> addr(smem_u32(sm), lane);

    for (uint32_t q = tile.y + warp; q < tile.z; q += kTileWarps) {
        const uint32_t sq = P.rows_mode ? P.refpos[q] : q;
        const uint32_t len = P.len_sorted[sq];
        const uint8_t* sp = P.codes + (size_t)P.code_off[sq] * 16;
        const uint32_t nwords = (len + 3) / 4;

        uint32_t X[NL];
#pragma unroll
        for (int w = 0; w < NL; ++w) X[w] = 0xffffffffu;

        // One warp-uniform byte load per residue (MIO pipe) instead of one word load and a shift and mask per residue
        // (ALU pipe).  Padding residues (code kNoMatch, all-zero mask row) leave X unchanged; the code buffer has
        // 16 bytes of slack for the prefetch of the last round.
        uint32_t c[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) c[k] = __ldg(sp + k);
        for (uint32_t t = 0; t < nwords; ++t) {
            sp += 4;
            uint32_t nxt[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) nxt[k] = __ldg(sp + k);
#pragma unroll
            for (int k = 0; k < 4; ++k) lcs_step<NL>(X, addr, c[k]);
#pragma unroll
            for (int k = 0; k < 4; ++k) c[k] = nxt[k];
        }
        uint32_t lcs = 0;
#pragma unroll
        for (int w = 0; w < NL; ++w) lcs += __popc(~X[w]);

        if (P.rows_mode) {
            lcs_store(P.out, P.elem_bytes, (size_t)q * P.ld_res + p, lcs);
        } else if (a != 0xffffffffu && sq < p) {
            const uint32_t b = P.perm[sq];
            const uint32_t i = a > b ? a : b, j = a > b ? b : a;
            if (i >= P.row_begin && i < P.row_end) lcs_store(P.out, P.elem_bytes, tri_index(i, 0) - P.tri_base + j, lcs);
        }
    }
}

// rows mode: res[r][sorted position] -> out[r][k] in the caller's column order
__global__ void k_gather_rows(const void* __restrict__ res, uint32_t ld_res, int res_bytes,
                              const uint32_t* __restrict__ col_ids, const uint32_t* __restrict__ invperm,
                              uint32_t n_col, void* __restrict__ out, int elem_bytes)
{
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t r = blockIdx.y;
    if (k >= n_col) return;
    const uint32_t c = col_ids ? col_ids[k] : k;
    const uint32_t v = lcs_load(res, res_bytes, (size_t)r * ld_res + invperm[c]);
    lcs_store(out, elem_bytes, (size_t)r * n_col + k, v);
}

// ------------------------------------------------------------------------------------------------
// exact path: the reference recurrence word for word (64-bit words, carry = (sum < V))
// ------------------------------------------------------------------------------------------------

// masks[c * nw + w], c in 0..20 (row 20 all zero), for the sequence at sorted position sp
__global__ void k_masks64(const uint8_t* __restrict__ codes, const uint32_t* __restrict__ code_off,
                          const uint32_t* __restrict__ len_sorted, uint32_t sp, uint32_t nw,
                          unsigned long long* __restrict__ masks)
{
    const uint32_t idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= kMaskRows * nw) return;
    const uint32_t c = idx / nw, w = idx % nw;
    const uint32_t len = len_sorted[sp];
    const uint8_t* src = codes + (size_t)code_off[sp] * 16;
    unsigned long long m = 0;
    if (c < 20)
        for (uint32_t b = 0; b < 64; ++b) {
            const uint32_t pos = w * 64 + b;
            if (pos < len && src[pos] == c) m |= 1ull << b;
        }
    masks[idx] = m;
}

// one thread per column; X lives in global scratch, word-major so the warp's accesses coalesce
__global__ void k_lcs_exact(const uint8_t* __restrict__ codes, const uint32_t* __restrict__ code_off,
                            const uint32_t* __restrict__ len_sorted, const uint32_t* __restrict__ invperm,
                            const unsigned long long* __restrict__ masks, uint32_t nw,
                            const uint32_t* __restrict__ col_ids, uint32_t n_col,
                            const uint32_t* __restrict__ group_nl, int only_long_cols,
                            unsigned long long* __restrict__ xs, void* __restrict__ out,
                            size_t out_base, int elem_bytes)
{
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_col) return;
    const uint32_t col = col_ids ? col_ids[k] : k;
    const uint32_t sq = invperm[col];
    if (only_long_cols && group_nl[sq / 32] != 0) return;
    const uint32_t len = len_sorted[sq];
    const uint8_t* src = codes + (size_t)code_off[sq] * 16;
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    unsigned long long* x = xs + k;
    for (uint32_t w = 0; w < nw; ++w) x[w * stride] = ~0ull;
    for (uint32_t t = 0; t < len; ++t) {
        const uint32_t c = src[t];
        if (c >= 20) continue;
        const unsigned long long* m = masks + (size_t)c * nw;
        unsigned long long carry = 0;
        for (uint32_t w = 0; w < nw; ++w) {
            const unsigned long long v = x[w * stride];
            const unsigned long long tb = v & m[w];
            const unsigned long long sum = v + tb + carry;
            carry = sum < v;
            x[w * stride] = sum | (v - tb);
        }
    }
    uint32_t lcs = 0;
    for (uint32_t w = 0; w < nw; ++w) lcs += __popcll(~x[w * stride]);
    lcs_store(out, elem_bytes, out_base + k, lcs);
}

// All special rows of a call in ONE launch: blockIdx.y = the row, its 64-bit masks are built in shared memory by the
// block itself, X[] lives in the thread (local memory, L1-resident) -- for rows of at most kExactWords * 64 residues.
// rows[r] = {sorted position of the row, out_base (element offset of the row's first result), n_col, only_long_cols}.
constexpr int kExactWords = 64;
struct ExactRow { uint32_t sp, n_col, only_long, pad; unsigned long long out_base; };
__global__ void __launch_bounds__(128) k_lcs_exact_batch(const uint8_t* __restrict__ codes, const uint32_t* __restrict__ code_off,
                                                         const uint32_t* __restrict__ len_sorted, const uint32_t* __restrict__ invperm,
                                                         const ExactRow* __restrict__ rows, const uint32_t* __restrict__ col_ids,
                                                         const uint32_t* __restrict__ group_nl, void* __restrict__ out, int elem_bytes)
{
    __shared__ unsigned long long masks[kMaskRows * kExactWords];
    const ExactRow R = rows[blockIdx.y];
    if (blockIdx.x * blockDim.x >= R.n_col) return;
    const uint32_t rlen = len_sorted[R.sp], nw = rlen ? (rlen + 63) / 64 : 1;
    const uint8_t* rsrc = codes + (size_t)code_off[R.sp] * 16;
    for (uint32_t i = threadIdx.x; i < kMaskRows * nw; i += blockDim.x) masks[i] = 0;
    __syncthreads();
    for (uint32_t pos = threadIdx.x; pos < rlen; pos += blockDim.x) {
        const uint32_t c = rsrc[pos];
        if (c < 20) atomicOr(&masks[c * nw + pos / 64], 1ull << (pos % 64));
    }
    __syncthreads();
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= R.n_col) return;
    const uint32_t col = col_ids ? col_ids[k] : k;
    const uint32_t sq = invperm[col];
    if (R.only_long && group_nl[sq / 32] != 0) return;
    const uint32_t len = len_sorted[sq];
    const uint8_t* src = codes + (size_t)code_off[sq] * 16;
    unsigned long long x[kExactWords];
    for (uint32_t w = 0; w < nw; ++w) x[w] = ~0ull;
    for (uint32_t t = 0; t < len; ++t) {
        const uint32_t c = src[t];
        if (c >= 20) continue;
        const unsigned long long* m = masks + c * nw;
        unsigned long long carry = 0;
        for (uint32_t w = 0; w < nw; ++w) {
            const unsigned long long v = x[w];
            const unsigned long long tb = v & m[w];
            const unsigned long long sum = v + tb + carry;
            carry = sum < v;
            x[w] = sum | (v - tb);
        }
    }
    uint32_t lcs = 0;
    for (uint32_t w = 0; w < nw; ++w) lcs += __popcll(~x[w]);
    lcs_store(out, elem_bytes, R.out_base + k, lcs);
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------

// (T) pow(i, 0.75) for every possible indel count, computed by the host libm like the reference's table
template <class T>
static int upload_pow075(famsa_ctx* ctx, DevBuf& buf, cudaStream_t st)
{
    std::vector<T> pw((size_t)2 * ctx->lcs.max_len + 2);
    for (size_t v = 0; v < pw.size(); ++v) pw[v] = (T)pow((double)v, 0.75);
    FB_TRY(buf.reserve(sizeof(T) * pw.size()));
    FB_CUDA(cudaMemcpyAsync(buf.p, pw.data(), sizeof(T) * pw.size(), cudaMemcpyHostToDevice, st));
    FB_CUDA(cudaStreamSynchronize(st));          // pw goes out of scope
    return FAMSA_OK;
}

template <int NL>
static int launch_tile(famsa_ctx* ctx, const TileParams& P, uint32_t n_tiles, cudaStream_t st)
{
    static std::atomic<bool> configured[64];       // per device ordinal; setting the attribute twice is harmless
    const size_t smem = (size_t)blob_words(NL) * 4;
    if (!configured[ctx->device & 63].load(std::memory_order_acquire)) {
        FB_CUDA(cudaFuncSetAttribute(k_lcs_tile<NL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        configured[ctx->device & 63].store(true, std::memory_order_release);
    }
    k_lcs_tile<NL><<<n_tiles, kTileWarps * 32, smem, st>>>(P);
    FB_CUDA(cudaGetLastError());
    ctx->launches++;
    return FAMSA_OK;
}

static int launch_tile_nl(famsa_ctx* ctx, uint32_t nl, const TileParams& P, uint32_t n_tiles, cudaStream_t st)
{
    switch (nl) {
#define FB_CASE(N) case N: return launch_tile<N>(ctx, P, n_tiles, st);
        FB_CASE(1) FB_CASE(2) FB_CASE(3) FB_CASE(4) FB_CASE(5) FB_CASE(6) FB_CASE(7) FB_CASE(8)
        FB_CASE(9) FB_CASE(10) FB_CASE(11) FB_CASE(12) FB_CASE(13) FB_CASE(14) FB_CASE(15) FB_CASE(16)
        FB_CASE(17) FB_CASE(18) FB_CASE(19) FB_CASE(20) FB_CASE(21) FB_CASE(22) FB_CASE(23) FB_CASE(24)
        FB_CASE(25) FB_CASE(26) FB_CASE(27) FB_CASE(28) FB_CASE(29) FB_CASE(30) FB_CASE(31) FB_CASE(32)
        FB_CASE(36) FB_CASE(40) FB_CASE(44) FB_CASE(48) FB_CASE(52) FB_CASE(56) FB_CASE(60) FB_CASE(64)
#undef FB_CASE
    default:
        set_error("internal: no tile kernel for nl=" + std::to_string(nl));
        return FAMSA_E_INVALID;
    }
}

static int lcs_upload_impl(famsa_ctx* ctx, const int8_t* codes, const uint64_t* offsets, const uint32_t* lens, uint32_t n);

// A failed upload leaves the context without a sequence set (n = 0) rather than with a half-replaced one.
int lcs_upload(famsa_ctx* ctx, const int8_t* codes, const uint64_t* offsets, const uint32_t* lens, uint32_t n)
{
    const int rc = lcs_upload_impl(ctx, codes, offsets, lens, n);
    if (rc != FAMSA_OK) {
        LcsState& S = ctx->lcs;
        S.n = S.n_groups = 0;
        S.max_len = 0;
        S.groups.clear(); S.h_quirky.clear(); S.h_long.clear();
    }
    return rc;
}

static int lcs_upload_impl(famsa_ctx* ctx, const int8_t* codes, const uint64_t* offsets, const uint32_t* lens, uint32_t n)
{
    LcsState& S = ctx->lcs;
    cudaStream_t st = ctx->stream;
    S.n = n;
    S.n_groups = (n + 31) / 32;
    S.h_quirky.clear();
    S.h_long.clear();
    if (n == 0) return FAMSA_OK;
    const uint32_t npad = S.n_groups * 32;

    // length-descending order (stable), as CFAMSA::sortAndExtendSequences leaves it (msa.cpp:245-279)
    S.h_perm.resize(n);
    std::iota(S.h_perm.begin(), S.h_perm.end(), 0u);
    S.identity_perm = std::is_sorted(lens, lens + n, [](uint32_t x, uint32_t y) { return x > y; });
    if (!S.identity_perm)
        std::stable_sort(S.h_perm.begin(), S.h_perm.end(), [&](uint32_t x, uint32_t y) { return lens[x] > lens[y]; });
    S.h_invperm.resize(n);
    for (uint32_t p = 0; p < n; ++p) S.h_invperm[S.h_perm[p]] = p;

    S.h_len_sorted.assign(npad, 0);
    std::vector<uint32_t> code_off(npad + 1, 0);
    uint64_t units = 0, raw_lo = UINT64_MAX, raw_hi = 0;
    S.max_len = 0;
    for (uint32_t p = 0; p < n; ++p) {
        const uint32_t a = S.h_perm[p];
        S.h_len_sorted[p] = lens[a];
        S.max_len = std::max(S.max_len, lens[a]);
        code_off[p] = (uint32_t)units;
        units += (lens[a] + 15) / 16;
        if (units > 0xfffffff0ull) { set_error("sequence set too large (> 64 GiB of residues)"); return FAMSA_E_INVALID; }
        if (lens[a]) { raw_lo = std::min(raw_lo, offsets[a]); raw_hi = std::max(raw_hi, offsets[a] + lens[a]); }
    }
    for (uint32_t p = n; p <= npad; ++p) code_off[p] = (uint32_t)units;
    if (raw_lo == UINT64_MAX) raw_lo = raw_hi = 0;

    S.groups.assign(S.n_groups, LcsGroupInfo{0, 0});
    std::vector<uint64_t> group_blob(S.n_groups);
    std::vector<uint32_t> group_nl(S.n_groups);
    uint64_t words = 0;
    uint32_t max_nl = 1;
    for (uint32_t g = 0; g < S.n_groups; ++g) {
        const uint32_t nl = nl_for_len(S.h_len_sorted[g * 32]);   // first of the group is the longest
        S.groups[g].nl = nl;
        S.groups[g].blob_word = words;
        group_blob[g] = words;
        group_nl[g] = nl;
        words += blob_words(nl);
        max_nl = std::max(max_nl, nl);
        if (nl == 0)
            for (uint32_t p = g * 32; p < std::min(n, g * 32 + 32); ++p) S.h_long.push_back(S.h_perm[p]);
    }

    // shifted offsets so that only the used byte range of the caller's buffer is copied
    std::vector<uint64_t> off_shift(n);
    for (uint32_t a = 0; a < n; ++a) off_shift[a] = lens[a] ? offsets[a] - raw_lo : 0;

    FB_TRY(S.d_perm.reserve(sizeof(uint32_t) * n));
    FB_TRY(S.d_invperm.reserve(sizeof(uint32_t) * n));
    FB_TRY(S.d_len_sorted.reserve(sizeof(uint32_t) * npad));
    FB_TRY(S.d_code_off.reserve(sizeof(uint32_t) * (npad + 1)));
    FB_TRY(S.d_codes.reserve(units * 16 + 64));
    FB_TRY(S.d_blob.reserve(std::max<uint64_t>(words, 1) * 4));
    FB_TRY(S.d_group_blob.reserve(sizeof(uint64_t) * S.n_groups + sizeof(uint32_t) * S.n_groups));
    FB_TRY(S.d_raw_codes.reserve(raw_hi - raw_lo + 16));
    FB_TRY(S.d_raw_off.reserve(sizeof(uint64_t) * n));
    FB_TRY(S.d_raw_len.reserve(sizeof(uint32_t) * n));
    FB_TRY(S.d_flags.reserve(n));

    uint32_t* d_group_nl = reinterpret_cast<uint32_t*>(S.d_group_blob.as<uint64_t>() + S.n_groups);
    FB_CUDA(cudaMemcpyAsync(S.d_perm.p, S.h_perm.data(), sizeof(uint32_t) * n, cudaMemcpyHostToDevice, st));
    FB_CUDA(cudaMemcpyAsync(S.d_invperm.p, S.h_invperm.data(), sizeof(uint32_t) * n, cudaMemcpyHostToDevice, st));
    FB_CUDA(cudaMemcpyAsync(S.d_len_sorted.p, S.h_len_sorted.data(), sizeof(uint32_t) * npad, cudaMemcpyHostToDevice, st));
    FB_CUDA(cudaMemcpyAsync(S.d_code_off.p, code_off.data(), sizeof(uint32_t) * (npad + 1), cudaMemcpyHostToDevice, st));
    FB_CUDA(cudaMemcpyAsync(S.d_group_blob.p, group_blob.data(), sizeof(uint64_t) * S.n_groups, cudaMemcpyHostToDevice, st));
    FB_CUDA(cudaMemcpyAsync(d_group_nl, group_nl.data(), sizeof(uint32_t) * S.n_groups, cudaMemcpyHostToDevice, st));
    if (raw_hi > raw_lo)
        FB_CUDA(cudaMemcpyAsync(S.d_raw_codes.p, codes + raw_lo, raw_hi - raw_lo, cudaMemcpyHostToDevice, st));
    FB_CUDA(cudaMemcpyAsync(S.d_raw_off.p, off_shift.data(), sizeof(uint64_t) * n, cudaMemcpyHostToDevice, st));
    FB_CUDA(cudaMemcpyAsync(S.d_raw_len.p, lens, sizeof(uint32_t) * n, cudaMemcpyHostToDevice, st));
    FB_CUDA(cudaMemsetAsync(S.d_codes.p, kNoMatch, units * 16 + 64, st));

    FB_TRY(upload_pow075<float>(ctx, S.d_pow075, st));
    k_repack<<<(n + 7) / 8, 256, 0, st>>>(S.d_raw_codes.as<int8_t>(), S.d_raw_off.as<uint64_t>(),
                                          S.d_raw_len.as<uint32_t>(), S.d_perm.as<uint32_t>(),
                                          S.d_code_off.as<uint32_t>(), S.d_codes.as<uint8_t>(), n);
    FB_CUDA(cudaGetLastError());
    const size_t build_smem = (size_t)blob_words(max_nl) * 4;
    FB_CUDA(cudaFuncSetAttribute(k_build_blob, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)build_smem));
    k_build_blob<<<S.n_groups, 256, build_smem, st>>>(S.d_codes.as<uint8_t>(), S.d_code_off.as<uint32_t>(),
                                                      S.d_len_sorted.as<uint32_t>(), S.d_group_blob.as<uint64_t>(),
                                                      d_group_nl, S.d_blob.as<uint32_t>(), n);
    FB_CUDA(cudaGetLastError());
    k_quirky<<<(n + 127) / 128, 128, 0, st>>>(S.d_codes.as<uint8_t>(), S.d_code_off.as<uint32_t>(),
                                              S.d_len_sorted.as<uint32_t>(), S.d_flags.as<uint8_t>(), n);
    FB_CUDA(cudaGetLastError());
    ctx->launches += 3;
    std::vector<uint8_t> flags(n);
    FB_CUDA(cudaMemcpyAsync(flags.data(), S.d_flags.p, n, cudaMemcpyDeviceToHost, st));
    FB_CUDA(cudaStreamSynchronize(st));
    for (uint32_t p = 0; p < n; ++p)
        if (flags[p]) S.h_quirky.push_back(S.h_perm[p]);
    std::sort(S.h_quirky.begin(), S.h_quirky.end());
    std::sort(S.h_long.begin(), S.h_long.end());
    return FAMSA_OK;
}

static TileParams base_params(famsa_ctx* ctx)
{
    LcsState& S = ctx->lcs;
    TileParams P{};
    P.blob = S.d_blob.as<uint32_t>();
    P.group_blob = S.d_group_blob.as<uint64_t>();
    P.codes = S.d_codes.as<uint8_t>();
    P.code_off = S.d_code_off.as<uint32_t>();
    P.len_sorted = S.d_len_sorted.as<uint32_t>();
    P.perm = S.d_perm.as<uint32_t>();
    P.n = S.n;
    return P;
}

// exact recomputation of one row (caller id `row`) against a column list
static int exact_row(famsa_ctx* ctx, uint32_t row, const uint32_t* d_col_ids, uint32_t n_col,
                     int only_long_cols, void* d_out, size_t out_base, int elem_bytes, cudaStream_t st)
{
    LcsState& S = ctx->lcs;
    if (n_col == 0) return FAMSA_OK;
    const uint32_t sp = S.h_invperm[row];
    const uint32_t len = S.h_len_sorted[sp];
    const uint32_t nw = std::max(1u, (len + 63) / 64);
    const uint32_t threads = 128, blocks = (n_col + threads - 1) / threads;
    FB_TRY(S.d_masks64.reserve(sizeof(uint64_t) * kMaskRows * nw));
    FB_TRY(S.d_x64.reserve(sizeof(uint64_t) * (size_t)nw * blocks * threads));
    k_masks64<<<(kMaskRows * nw + 127) / 128, 128, 0, st>>>(
        S.d_codes.as<uint8_t>(), S.d_code_off.as<uint32_t>(), S.d_len_sorted.as<uint32_t>(), sp, nw,
        S.d_masks64.as<unsigned long long>());
    FB_CUDA(cudaGetLastError());
    const uint32_t* d_group_nl = reinterpret_cast<const uint32_t*>(S.d_group_blob.as<uint64_t>() + S.n_groups);
    k_lcs_exact<<<blocks, threads, 0, st>>>(
        S.d_codes.as<uint8_t>(), S.d_code_off.as<uint32_t>(), S.d_len_sorted.as<uint32_t>(),
        S.d_invperm.as<uint32_t>(), S.d_masks64.as<unsigned long long>(), nw, d_col_ids, n_col, d_group_nl,
        only_long_cols, S.d_x64.as<unsigned long long>(), d_out, out_base, elem_bytes);
    FB_CUDA(cudaGetLastError());
    ctx->launches += 2;
    return FAMSA_OK;
}

// The exact recomputation of many rows: rows of at most kExactWords * 64 residues go through one launch of
// k_lcs_exact_batch (masks in shared memory, X[] in the thread); longer ones keep the per-row global-memory path.
struct ExactReq { uint32_t row, n_col; int only_long; size_t out_base; };
static int exact_rows(famsa_ctx* ctx, const std::vector<ExactReq>& reqs, const uint32_t* d_col_ids, void* d_out, int elem_bytes, cudaStream_t st)
{
    LcsState& S = ctx->lcs;
    std::vector<ExactRow> batch;
    uint32_t max_cols = 0;
    for (const ExactReq& q : reqs) {
        if (!q.n_col) continue;
        const uint32_t sp = S.h_invperm[q.row];
        if (S.h_len_sorted[sp] <= (uint32_t)kExactWords * 64) {
            batch.push_back(ExactRow{sp, q.n_col, (uint32_t)q.only_long, 0, (unsigned long long)q.out_base});
            max_cols = std::max(max_cols, q.n_col);
        } else FB_TRY(exact_row(ctx, q.row, d_col_ids, q.n_col, q.only_long, d_out, q.out_base, elem_bytes, st));
    }
    if (batch.empty()) return FAMSA_OK;
    const uint32_t* d_group_nl = reinterpret_cast<const uint32_t*>(S.d_group_blob.as<uint64_t>() + S.n_groups);
    for (size_t b0 = 0; b0 < batch.size(); b0 += 65535) {            // gridDim.y limit
        const size_t nb = std::min<size_t>(65535, batch.size() - b0);
        FB_TRY(S.d_exact_rows.reserve(sizeof(ExactRow) * nb));
        FB_CUDA(cudaMemcpyAsync(S.d_exact_rows.p, batch.data() + b0, sizeof(ExactRow) * nb, cudaMemcpyHostToDevice, st));
        k_lcs_exact_batch<<<dim3((max_cols + 127) / 128, (unsigned)nb), 128, 0, st>>>(
            S.d_codes.as<uint8_t>(), S.d_code_off.as<uint32_t>(), S.d_len_sorted.as<uint32_t>(), S.d_invperm.as<uint32_t>(),
            S.d_exact_rows.as<ExactRow>(), d_col_ids, d_group_nl, d_out, elem_bytes);
        FB_CUDA(cudaGetLastError());
        ctx->launches++;
    }
    return FAMSA_OK;
}

void lcs_row_pieces(uint32_t row_begin, uint32_t row_end, int n_pieces, const double* frac, uint32_t* bounds)
{
    const uint64_t pairs = tri_index(row_end, 0) - tri_index(row_begin, 0);
    bounds[0] = row_begin;
    for (int b = 1; b < n_pieces; ++b) {
        const double share = frac ? (double)pairs * frac[b] : (double)pairs * b / n_pieces;
        uint32_t r = (uint32_t)((1.0 + std::sqrt(1.0 + 8.0 * ((double)tri_index(row_begin, 0) + share))) / 2.0);
        r = (r + 16) / 32 * 32;
        bounds[b] = std::min(std::max(r, bounds[b - 1]), row_end);
    }
    bounds[n_pieces] = row_end;
}

// The span of the tile kernels within the entry point's call: ev[1] at the first tile launch, ev[2] after the last
static int mark_tiles_begin(famsa_ctx* ctx, cudaStream_t st)
{
    if (ctx->lcs.tiles_marked) return FAMSA_OK;
    FB_CUDA(cudaEventRecord(ctx->ev[1], st));
    ctx->lcs.tiles_marked = true;
    return FAMSA_OK;
}

// The tiles of one call, per piece and limb-count class (index NL).  upload() copies all of them into d_tiles in one
// go, piece after piece and class after class, and marks the start of the tile span; launch(b), called for the pieces
// in order, issues piece b's classes in ascending NL on the given stream.
struct TilePlan {
    std::vector<std::vector<std::vector<uint3>>> lists;
    size_t total = 0, at = 0;
    explicit TilePlan(int n_pieces) : lists(n_pieces, std::vector<std::vector<uint3>>(kMaxNL + 1)) {}
    // mask group g against the streamed items [0, q_end), kTileQ per tile
    void add(int b, uint32_t g, uint32_t nl, uint32_t q_end)
    {
        for (uint32_t q0 = 0; q0 < q_end; q0 += kTileQ, ++total)
            lists[b][nl].push_back(make_uint3(g, q0, std::min(q_end, q0 + (uint32_t)kTileQ)));
    }
    int upload(famsa_ctx* ctx, cudaStream_t st) const
    {
        std::vector<uint3> flat;
        flat.reserve(total);
        for (auto& piece : lists)
            for (auto& v : piece) flat.insert(flat.end(), v.begin(), v.end());
        FB_TRY(ctx->lcs.d_tiles.reserve(sizeof(uint3) * std::max<size_t>(total, 1)));
        if (total) FB_CUDA(cudaMemcpyAsync(ctx->lcs.d_tiles.p, flat.data(), sizeof(uint3) * total, cudaMemcpyHostToDevice, st));
        return mark_tiles_begin(ctx, st);
    }
    int launch(famsa_ctx* ctx, int b, TileParams P, cudaStream_t st)
    {
        for (uint32_t nl = 1; nl <= (uint32_t)kMaxNL; ++nl) {
            const auto& v = lists[b][nl];
            if (v.empty()) continue;
            P.tiles = ctx->lcs.d_tiles.as<uint3>() + at;
            FB_TRY(launch_tile_nl(ctx, nl, P, (uint32_t)v.size(), st));
            at += v.size();
        }
        return FAMSA_OK;
    }
};

// Rows [row_begin, row_end) of the packed triangle.  With `bounds` (n_blocks + 1 ascending row indices spanning the
// range) the work is issued block by block and block_events[b] is recorded after block b, so that a caller can
// start copying finished blocks while later ones are still being computed; every tile list is uploaded up front.
int lcs_triangle(famsa_ctx* ctx, uint32_t row_begin, uint32_t row_end, void* d_out, int elem_bytes, cudaStream_t st,
                 const uint32_t* bounds, int n_blocks, cudaEvent_t* block_events, bool quirk_fixups, bool piece_streams)
{
    LcsState& S = ctx->lcs;
    const uint32_t n = S.n;
    const uint32_t whole[2] = {row_begin, row_end};
    if (!bounds || !S.identity_perm) { bounds = whole; n_blocks = 1; }

    TilePlan tiles(n_blocks);
    for (int b = 0; b < n_blocks; ++b)
        for (uint32_t g = 0; g < S.n_groups; ++g) {
            if (S.groups[g].nl == 0) continue;
            if (S.identity_perm && (g * 32 + 32 <= bounds[b] || g * 32 >= bounds[b + 1])) continue;
            tiles.add(b, g, S.groups[g].nl, std::min(n, g * 32 + 31));
        }
    S.last_tiles = tiles.total;
    FB_TRY(tiles.upload(ctx, st));
    TileParams P = base_params(ctx);
    P.out = d_out;
    P.elem_bytes = elem_bytes;
    P.rows_mode = 0;
    P.tri_base = tri_index(row_begin, 0);
    std::vector<uint32_t> special;      // rows the tile kernel may not answer for: dropped-carry and over-long rows
    if (quirk_fixups) std::set_union(S.h_quirky.begin(), S.h_quirky.end(), S.h_long.begin(), S.h_long.end(), std::back_inserter(special));
    else special = S.h_long;         // true LCS everywhere: only the rows the tile kernel cannot reach
    // Blocks in one stream would each end with a partly filled last wave (half a wave of tiles per block boundary: 0.4 ms at
    // C2).  Issued round-robin on the auxiliary streams instead, the block scheduler fills the tail of block b with the first
    // tiles of block b+1 and the blocks still finish in order.  (The exact kernels share one scratch: single stream then.)
    constexpr int kAux = sizeof(ctx->aux_stream) / sizeof(ctx->aux_stream[0]);
    const bool fan = piece_streams && n_blocks > 1 && special.empty();
    if (fan) {
        FB_CUDA(cudaEventRecord(ctx->ev_fork, st));
        for (int a = 0; a < std::min(kAux, n_blocks); ++a) FB_CUDA(cudaStreamWaitEvent(ctx->aux_stream[a], ctx->ev_fork, 0));
    }
    for (int b = 0; b < n_blocks; ++b) {
        const cudaStream_t bst = fan ? ctx->aux_stream[b % kAux] : st;
        P.row_begin = bounds[b];
        P.row_end = bounds[b + 1];
        FB_TRY(tiles.launch(ctx, b, P, bst));
        // rows the tile kernel cannot answer for: dropped-carry rows entirely; over-long rows only against over-long columns
        // (their pairs with shorter sequences were computed with the shorter one as the mask side -- the true LCS is symmetric)
        std::vector<ExactReq> reqs;
        for (uint32_t row : special) {
            if (row < bounds[b] || row >= bounds[b + 1] || row == 0) continue;
            const bool quirky = quirk_fixups && std::binary_search(S.h_quirky.begin(), S.h_quirky.end(), row);
            reqs.push_back(ExactReq{row, row, quirky ? 0 : 1, tri_index(row, 0) - (size_t)P.tri_base});
        }
        FB_TRY(exact_rows(ctx, reqs, nullptr, d_out, elem_bytes, bst));
        if (block_events) FB_CUDA(cudaEventRecord(block_events[b], bst));
    }
    if (fan)
        for (int a = 0; a < std::min(kAux, n_blocks); ++a) {
            FB_CUDA(cudaEventRecord(ctx->ev_join[a], ctx->aux_stream[a]));
            FB_CUDA(cudaStreamWaitEvent(st, ctx->ev_join[a], 0));
        }
    FB_CUDA(cudaEventRecord(ctx->ev[2], st));
    return FAMSA_OK;
}

int lcs_rows(famsa_ctx* ctx, const uint32_t* h_ref_ids, uint32_t n_ref, const uint32_t* d_col_ids, uint32_t n_col, void* d_out,
             int elem_bytes, cudaStream_t st, uint32_t g_begin, uint32_t g_end)
{
    LcsState& S = ctx->lcs;
    const uint32_t npad = S.n_groups * 32;
    const int res_bytes = S.elem_bytes();

    // streamed side = the reference rows (true LCS is symmetric); mask side = every group
    std::vector<uint32_t> refpos(n_ref);
    for (uint32_t r = 0; r < n_ref; ++r) refpos[r] = S.h_invperm[h_ref_ids[r]];
    FB_TRY(S.d_refpos.reserve(sizeof(uint32_t) * std::max(1u, n_ref)));
    FB_CUDA(cudaMemcpyAsync(S.d_refpos.p, refpos.data(), sizeof(uint32_t) * n_ref, cudaMemcpyHostToDevice, st));
    FB_TRY(S.d_res.reserve((size_t)res_bytes * npad * std::max(1u, n_ref)));

    TilePlan tiles(1);
    g_end = std::min(g_end, S.n_groups);
    for (uint32_t g = g_begin; g < g_end; ++g)                       // the mask groups (= columns) this call answers for
        if (S.groups[g].nl) tiles.add(0, g, S.groups[g].nl, n_ref);
    FB_TRY(tiles.upload(ctx, st));
    TileParams P = base_params(ctx);
    P.out = S.d_res.p;
    P.elem_bytes = res_bytes;
    P.rows_mode = 1;
    P.refpos = S.d_refpos.as<uint32_t>();
    P.ld_res = npad;
    FB_TRY(tiles.launch(ctx, 0, P, st));
    FB_CUDA(cudaEventRecord(ctx->ev[2], st));
    if (n_col && n_ref) {
        dim3 grid((n_col + 255) / 256, n_ref);
        k_gather_rows<<<grid, 256, 0, st>>>(S.d_res.p, npad, res_bytes, d_col_ids, S.d_invperm.as<uint32_t>(),
                                            n_col, d_out, elem_bytes);
        FB_CUDA(cudaGetLastError());
        ctx->launches++;
    }
    // exact fix-ups: dropped-carry / over-long reference rows entirely, over-long columns for the rest
    {
        std::vector<ExactReq> reqs;
        for (uint32_t r = 0; r < n_ref; ++r) {
            const uint32_t row = h_ref_ids[r];
            const bool quirky = std::binary_search(S.h_quirky.begin(), S.h_quirky.end(), row);
            const bool is_long = std::binary_search(S.h_long.begin(), S.h_long.end(), row);
            // (an over-long reference row is the streamed side of the tiles, so only its over-long columns are missing)
            if (quirky) reqs.push_back(ExactReq{row, n_col, 0, (size_t)r * n_col});
            else if (is_long || !S.h_long.empty()) reqs.push_back(ExactReq{row, n_col, 1, (size_t)r * n_col});
        }
        FB_TRY(exact_rows(ctx, reqs, d_col_ids, d_out, elem_bytes, st));
    }
    return FAMSA_OK;
}

// (double) pow(i, 0.75) for every possible indel count into d_pow075_f64, like Transform<double, indel075_div_lcs>'s table
int lcs_pow075_f64(famsa_ctx* ctx, cudaStream_t st) { return upload_pow075<double>(ctx, ctx->lcs.d_pow075_f64, st); }

// The sequences whose LCS depends on which side is the row (the dropped-carry corner, h_quirky) and every over-long
// sequence before the last flagged over-long one: lcs_triangle computes a pair of two over-long sequences with the later
// one as seq0, so the true triangle holds a flagged one's orientation there.  d_side_idx[caller id] = their row in
// d_side_rows or -1, and d_side_rows = those rows (u32, n wide) with the sequence as seq0 -- what lcs_seq0 reads.
int lcs_side_rows(famsa_ctx* ctx, cudaStream_t st)
{
    LcsState& S = ctx->lcs;
    const uint32_t n = S.n;
    uint32_t long_end = 0;
    for (uint32_t x : S.h_long)
        if (std::binary_search(S.h_quirky.begin(), S.h_quirky.end(), x)) long_end = x;
    std::vector<uint32_t> ids;
    std::set_union(S.h_quirky.begin(), S.h_quirky.end(), S.h_long.begin(),
                   std::lower_bound(S.h_long.begin(), S.h_long.end(), long_end), std::back_inserter(ids));
    const uint32_t nq = (uint32_t)ids.size();
    std::vector<int> side_idx(n, -1);
    for (uint32_t q = 0; q < nq; ++q) side_idx[ids[q]] = (int)q;
    FB_TRY(S.d_side_idx.reserve(sizeof(int) * n));
    FB_CUDA(cudaMemcpyAsync(S.d_side_idx.p, side_idx.data(), sizeof(int) * n, cudaMemcpyHostToDevice, st));
    FB_TRY(S.d_side_rows.reserve(std::max<size_t>((size_t)nq * n, 1) * sizeof(uint32_t)));
    if (nq) FB_TRY(lcs_rows(ctx, ids.data(), nq, nullptr, n, S.d_side_rows.p, 4, st));
    return FAMSA_OK;
}

} // namespace fb
