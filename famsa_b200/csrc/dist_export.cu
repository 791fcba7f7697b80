// The distance-matrix export (-dist_export [-square_matrix] [-pid]) on sm_90a.
//
// Replaces DistanceCalculator<distance>::run (reference src/tree/DistanceCalculator.cpp:10-122): the per-row LCS +
// Transform of its worker threads and the single-threaded gather loop that prints every value with
// NumericConversions::Double2PChar (src/utils/conversion.h:52-119).  See DESIGN.md section 3.
//
//   * LCS: the packed triangle of the caller's order, computed once by the tile kernel and kept in HBM.  Triangle mode
//     reads it with row = seq0 (the dropped-carry rows recomputed by the exact path).  Square mode reads what k_prim
//     reads, through lcs_seq0: the true-LCS triangle and the side rows (lcs_side_rows) of the sequences whose value
//     depends on being seq0; the diagonal of the others is the number of residues that can match (codes < 20).
//   * Text: pass 1 sums every row's byte count (the width of a value depends on it alone); the host cuts the rows into
//     chunks and prefix-sums the row offsets; pass 2, one block per row, formats 1024 values at a time: per-value
//     lengths, a block scan, the characters into shared memory at the destination's 16-byte phase, then aligned 16-byte
//     stores (bytes at the two ragged ends).  Every byte has one writer and one value, so the text is deterministic.
#include <cmath>
#include <cstring>
#include <string>
#include <vector>

#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include "ctx.h"
#include "triangle_dev.cuh"

namespace fb {

constexpr int kFmtThreads = 256;
constexpr int kFmtPerThread = 4;                                  // consecutive columns per thread: contiguous text
constexpr int kFmtTile = kFmtThreads * kFmtPerThread;             // columns per block iteration
constexpr int kMaxValueChars = 40;                                // "9223372036854775808.223372036854775808" + ','
constexpr uint64_t kDefaultChunk = 32ull << 20;

struct DistParams {
    Seq0View lcs;                  // square; triangle: tri is the packed triangle with row = seq0, no side rows
    const uint32_t* lens;          // caller order
    const double* pow075;          // (double) pow(i, 0.75), host libm
    int kind, pid, square;
    const uint32_t* diag;          // square: LCS of a sequence with itself (those without a side row)
    const char* ids;
    const unsigned long long* id_off;   // n + 1
};

// ------------------------------------------------------------------------------------------------
// NumericConversions::Double2PChar((double) v, 6) (conversion.h:109-119), as the reference's x86-64 build runs it
// ------------------------------------------------------------------------------------------------

// (int64_t) x on x86-64 (cvttsd2si): NaN and out-of-range values give 0x8000000000000000; PTX's cvt would saturate.
__device__ __forceinline__ long long x86_trunc_i64(double x)
{
    return (x >= -0x1p63 && x < 0x1p63) ? (long long)x : (long long)0x8000000000000000ull;
}

__device__ __forceinline__ int ndigits_u64(unsigned long long v)
{
    int d = 1;
    while (v >= 10) { v /= 10; ++d; }
    return d;
}

// a = (int64) v, b = (int64) ((1.0 + (v - a)) * 10^6 + 0.5), each rounded on its own (no FMA contraction)
__device__ __forceinline__ void split_value(float v, unsigned long long& a, unsigned long long& b)
{
    const double d = (double)v;
    const long long ia = x86_trunc_i64(d);
    const double t = __dadd_rn(__dmul_rn(__dadd_rn(1.0, __dsub_rn(d, (double)ia)), 1000000.0), 0.5);
    a = (unsigned long long)ia;
    b = (unsigned long long)x86_trunc_i64(t);
}

// Int2PChar(a) then Int2PChar(b) with b's first digit overwritten by '.'; returns the length
__device__ __forceinline__ int value_chars(unsigned long long a, unsigned long long b)
{
    return ndigits_u64(a) + ndigits_u64(b);
}

__device__ __forceinline__ void put_u64(char* dst, int nd, unsigned long long v)
{
    if (v < 0x100000000ull) {                                     // 32-bit division for every ordinary value
        uint32_t w = (uint32_t)v;
        for (int i = nd - 1; i >= 0; --i) { dst[i] = (char)('0' + w % 10); w /= 10; }
    } else {
        for (int i = nd - 1; i >= 0; --i) { dst[i] = (char)('0' + v % 10); v /= 10; }
    }
}

__device__ __forceinline__ void put_value(char* dst, unsigned long long a, unsigned long long b)
{
    const int na = ndigits_u64(a), nb = ndigits_u64(b);
    put_u64(dst, na, a);
    put_u64(dst + na, nb, b);
    dst[na] = '.';
}

// ------------------------------------------------------------------------------------------------
// cells
// ------------------------------------------------------------------------------------------------

// LCS with r as seq0 and c streamed (c < r in triangle mode)
__device__ __forceinline__ uint32_t cell_lcs(const DistParams& P, uint32_t r, uint32_t c)
{
    if (P.square) {
        const int s = side_row<true>(P.lcs, r);
        if (c == r && s < 0) return P.diag[r];
        if (c > r || s >= 0) return lcs_seq0(P.lcs, s, r, c);
    }
    return lcs_load(P.lcs.tri, P.lcs.eb, tri_index(r, c));      // lcs_seq0's cell for c < r without a side row
}

__device__ __forceinline__ float cell_value(const DistParams& P, uint32_t r, uint32_t c)
{
    const uint32_t lcs = cell_lcs(P, r, c);
    if (P.pid) return transform_f32(2, lcs, P.lens[r], P.lens[c], nullptr);
    return __double2float_rn(transform_f64(P.kind, lcs, P.lens[r], P.lens[c], P.pow075));
}

// ------------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------------

// residues that can match (codes 0..19) per sequence, caller order: the LCS of an unflagged sequence with itself
__global__ void k_dist_diag(const int8_t* __restrict__ raw, const uint64_t* __restrict__ raw_off,
                            const uint32_t* __restrict__ raw_len, uint32_t n, uint32_t* __restrict__ diag)
{
    const uint32_t s = blockIdx.x * (blockDim.x / 32) + threadIdx.x / 32, lane = threadIdx.x % 32;
    if (s >= n) return;
    const int8_t* src = raw + raw_off[s];
    uint32_t cnt = 0;
    for (uint32_t i = lane; i < raw_len[s]; i += 32) cnt += (src[i] >= 0 && src[i] < 20);
    for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if (lane == 0) diag[s] = cnt;
}

// pass 1: bytes of every row (id, ',', each value and its ',' -- the last ',' becomes '\n')
__global__ void __launch_bounds__(kFmtThreads) k_dist_row_bytes(const DistParams P, unsigned long long* __restrict__ row_bytes)
{
    using Reduce = cub::BlockReduce<unsigned long long, kFmtThreads>;
    __shared__ typename Reduce::TempStorage tmp;
    const uint32_t r = blockIdx.x;
    const uint32_t ncol = P.square ? P.lcs.n : r;
    unsigned long long sum = 0;
    for (uint32_t c = threadIdx.x; c < ncol; c += kFmtThreads) {
        unsigned long long a, b;
        split_value(cell_value(P, r, c), a, b);
        sum += value_chars(a, b) + 1;
    }
    sum = Reduce(tmp).Sum(sum);
    if (threadIdx.x == 0) row_bytes[r] = sum + (P.id_off[r + 1] - P.id_off[r]) + 1;
}

// pass 2: rows [r0, r0 + gridDim.x) into `out`, row r at row_start[r] - row_start[r0].  Five blocks per SM: what the
// stage's shared memory allows, and 48 registers hold a thread's four cells without spilling.
__global__ void __launch_bounds__(kFmtThreads, 5) k_dist_format(const DistParams P, uint32_t r0,
                                                             const unsigned long long* __restrict__ row_start,
                                                             char* __restrict__ out)
{
    using Scan = cub::BlockScan<uint32_t, kFmtThreads>;
    __shared__ typename Scan::TempStorage tmp;
    __shared__ __align__(16) char stage[kFmtTile * kMaxValueChars + 32];
    __shared__ uint32_t tile_total;
    const uint32_t r = r0 + blockIdx.x;
    const uint32_t ncol = P.square ? P.lcs.n : r;
    char* row = out + (row_start[r] - row_start[r0]);

    const uint64_t id0 = P.id_off[r], idlen = P.id_off[r + 1] - id0;
    for (uint64_t i = threadIdx.x; i < idlen; i += kFmtThreads) row[i] = P.ids[id0 + i];
    if (threadIdx.x == 0) row[idlen] = ncol ? ',' : '\n';
    char* dst = row + idlen + 1;

    for (uint32_t t0 = 0; t0 < ncol; t0 += kFmtTile) {
        unsigned long long a[kFmtPerThread], b[kFmtPerThread];
        uint32_t len[kFmtPerThread], mine = 0;
        const uint32_t c0 = t0 + threadIdx.x * kFmtPerThread;
#pragma unroll
        for (int k = 0; k < kFmtPerThread; ++k) {
            len[k] = 0;
            if (c0 + k < ncol) {
                split_value(cell_value(P, r, c0 + k), a[k], b[k]);
                len[k] = value_chars(a[k], b[k]) + 1;
            }
            mine += len[k];
        }
        uint32_t at, total;
        Scan(tmp).ExclusiveSum(mine, at, total);
        // characters at the destination's 16-byte phase, so that whole 16-byte units copy as they are
        const uint32_t phase = (uint32_t)((uintptr_t)dst & 15);
        at += phase;
#pragma unroll
        for (int k = 0; k < kFmtPerThread; ++k) {
            if (!len[k]) continue;
            put_value(stage + at, a[k], b[k]);
            stage[at + len[k] - 1] = c0 + k + 1 == ncol ? '\n' : ',';
            at += len[k];
        }
        if (threadIdx.x == 0) tile_total = total;
        __syncthreads();
        const uint32_t end = phase + tile_total;                 // stage [phase, end) -> dst [0, tile_total)
        char* base = dst - phase;                                 // 16-byte aligned
        const uint32_t units = (end + 15) / 16;
        for (uint32_t u = threadIdx.x; u < units; u += kFmtThreads) {
            const uint32_t lo = u * 16, hi = lo + 16;
            if (lo >= phase && hi <= end) {
                *reinterpret_cast<uint4*>(base + lo) = *reinterpret_cast<const uint4*>(stage + lo);
            } else {
                for (uint32_t i = lo < phase ? phase : lo; i < (hi < end ? hi : end); ++i) base[i] = stage[i];
            }
        }
        dst += tile_total;
        __syncthreads();                                          // the stage and tile_total are reused
    }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------

static int nomem(famsa_ctx* ctx, const char* what, uint64_t bytes)
{
    size_t free_b = 0, total_b = 0;
    cudaMemGetInfo(&free_b, &total_b);
    cudaGetLastError();
    set_error(std::string("famsa_dist_export: ") + what + " of " + std::to_string(ctx->lcs.n) + " sequences needs " +
              std::to_string(bytes) + " bytes of device memory; " + std::to_string(free_b) + " of " + std::to_string(total_b) +
              " bytes are free (the whole LCS triangle stays resident in HBM for the export)");
    return FAMSA_E_NOMEM;
}

void dist_export_release(famsa_ctx* ctx)
{
    LcsState& S = ctx->lcs;
    for (char*& h : S.h_dx_chunk)
        if (h) { cudaFreeHost(h); h = nullptr; }
    S.h_dx_chunk_cap = 0;
    for (cudaEvent_t& e : S.ev_dx)
        if (e) { cudaEventDestroy(e); e = nullptr; }
}

int dist_export(famsa_ctx* ctx, int kind, int square, int pid, const char* ids, const uint64_t* id_offsets,
                uint64_t chunk_bytes, famsa_write_fn write, void* user, uint64_t* bytes_written)
{
    LcsState& S = ctx->lcs;
    cudaStream_t st = ctx->stream;
    const uint32_t n = S.n;
    const int eb = S.elem_bytes();
    const uint64_t pairs = tri_index(n, 0);
    uint64_t written = 0;
    if (bytes_written) *bytes_written = 0;
    if (!S.ev_dx[0])
        for (int e = 0; e < 6; ++e) FB_CUDA(cudaEventCreateWithFlags(&S.ev_dx[e], e % 3 == 2 ? cudaEventDisableTiming : cudaEventDefault));

    // 1. the LCS triangle in caller order, resident for the whole call: row = seq0 (triangle), the true LCS (square)
    if (S.d_lcs_tri.reserve(std::max<uint64_t>(pairs, 1) * eb)) return nomem(ctx, "the LCS triangle", pairs * eb);
    S.tiles_marked = false;
    FB_CUDA(cudaEventRecord(ctx->ev[0], st));
    FB_TRY(lcs_triangle(ctx, 0, n, S.d_lcs_tri.p, eb, st, nullptr, 1, nullptr, /*quirk_fixups=*/!square));
    FB_CUDA(cudaEventRecord(ctx->ev[3], st));
    FB_CUDA(cudaStreamSynchronize(st));
    float lcs_total = 0.f, lcs_main = 0.f;
    FB_CUDA(cudaEventElapsedTime(&lcs_total, ctx->ev[0], ctx->ev[3]));
    FB_CUDA(cudaEventElapsedTime(&lcs_main, ctx->ev[1], ctx->ev[2]));

    // 2. per-sequence tables: diagonal, row byte counts and starts, id offsets
    const size_t meta_bytes = sizeof(uint32_t) * n + sizeof(unsigned long long) * (3 * (size_t)n + 2);
    if (S.d_dx_meta.reserve(meta_bytes + 64)) return nomem(ctx, "the per-sequence tables", meta_bytes);
    uint32_t* d_diag = S.d_dx_meta.as<uint32_t>();
    unsigned long long* d_row_bytes = reinterpret_cast<unsigned long long*>(S.d_dx_meta.as<char>() + (((size_t)4 * n + 15) & ~(size_t)15));
    unsigned long long* d_row_start = d_row_bytes + n;
    unsigned long long* d_id_off = d_row_start + n + 1;
    const uint64_t id_bytes = id_offsets[n] - id_offsets[0];
    std::vector<unsigned long long> id_off(n + 1);
    for (uint32_t i = 0; i <= n; ++i) id_off[i] = id_offsets[i] - id_offsets[0];
    if (S.d_dx_ids.reserve(std::max<uint64_t>(id_bytes, 1))) return nomem(ctx, "the ids", id_bytes);
    if (id_bytes) FB_CUDA(cudaMemcpyAsync(S.d_dx_ids.p, ids + id_offsets[0], id_bytes, cudaMemcpyHostToDevice, st));
    FB_CUDA(cudaMemcpyAsync(d_id_off, id_off.data(), sizeof(unsigned long long) * (n + 1), cudaMemcpyHostToDevice, st));

    // square: the diagonal and the side rows
    FB_CUDA(cudaEventRecord(ctx->ev_host[0], st));
    if (square) {
        k_dist_diag<<<(n + 7) / 8, 256, 0, st>>>(S.d_raw_codes.as<int8_t>(), S.d_raw_off.as<uint64_t>(), S.d_raw_len.as<uint32_t>(), n, d_diag);
        FB_CUDA(cudaGetLastError());
        ctx->launches++;
        FB_TRY(lcs_side_rows(ctx, st));
    }
    if (!pid) FB_TRY(lcs_pow075_f64(ctx, st));

    DistParams P{};
    P.lcs = Seq0View{S.d_lcs_tri.p, eb, n, S.d_side_idx.as<int>(), S.d_side_rows.as<uint32_t>()};
    P.lens = S.d_raw_len.as<uint32_t>();
    P.pow075 = S.d_pow075_f64.as<double>();
    P.kind = kind; P.pid = pid; P.square = square;
    P.diag = d_diag;
    P.ids = S.d_dx_ids.as<char>(); P.id_off = d_id_off;

    // 3. pass 1 and the row layout
    k_dist_row_bytes<<<n, kFmtThreads, 0, st>>>(P, d_row_bytes);
    FB_CUDA(cudaGetLastError());
    ctx->launches++;
    FB_CUDA(cudaEventRecord(ctx->ev_host[1], st));
    std::vector<unsigned long long> row_bytes(n), row_start(n + 1);
    FB_CUDA(cudaMemcpyAsync(row_bytes.data(), d_row_bytes, sizeof(unsigned long long) * n, cudaMemcpyDeviceToHost, st));
    FB_CUDA(cudaStreamSynchronize(st));
    float prep_ms = 0.f;
    FB_CUDA(cudaEventElapsedTime(&prep_ms, ctx->ev_host[0], ctx->ev_host[1]));
    if (!chunk_bytes) chunk_bytes = kDefaultChunk;
    uint64_t cap = chunk_bytes;
    std::vector<uint32_t> bounds{0};
    unsigned long long acc = 0;
    row_start[0] = 0;
    for (uint32_t r = 0; r < n; ++r) {
        cap = std::max<uint64_t>(cap, row_bytes[r]);
        if (acc && acc + row_bytes[r] > chunk_bytes) { bounds.push_back(r); acc = 0; }
        acc += row_bytes[r];
        row_start[r + 1] = row_start[r] + row_bytes[r];
    }
    bounds.push_back(n);
    FB_CUDA(cudaMemcpyAsync(d_row_start, row_start.data(), sizeof(unsigned long long) * (n + 1), cudaMemcpyHostToDevice, st));
    for (int b = 0; b < 2; ++b)
        if (S.d_dx_chunk[b].reserve(cap + 16)) return nomem(ctx, "two text chunk buffers next to the LCS triangle", 2 * (cap + 16));
    if (S.h_dx_chunk_cap < cap) {
        for (char*& h : S.h_dx_chunk)
            if (h) { cudaFreeHost(h); h = nullptr; }
        S.h_dx_chunk_cap = 0;
        for (char*& h : S.h_dx_chunk) {
            if (cudaHostAlloc(reinterpret_cast<void**>(&h), cap, cudaHostAllocDefault) != cudaSuccess) {
                cudaGetLastError();
                h = nullptr;
                set_error("famsa_dist_export: cudaHostAlloc(" + std::to_string(cap) + ") failed for a pinned chunk buffer");
                return FAMSA_E_NOMEM;
            }
        }
        S.h_dx_chunk_cap = cap;
    }

    auto refused = [&](int rc, uint64_t n_bytes) {
        set_error("famsa_dist_export: the write callback returned " + std::to_string(rc) + " for " + std::to_string(n_bytes) +
                  " bytes at byte offset " + std::to_string(written) + "; nothing after that offset was written");
        return FAMSA_E_SINK;
    };

    // 4. the header (square), then the chunks: format + copy of chunk k+1 run while `write` consumes chunk k
    if (square) {
        std::string head;
        head.reserve(id_bytes + n + 1);
        for (uint32_t i = 0; i < n; ++i) { head += ','; head.append(ids + id_offsets[i], id_offsets[i + 1] - id_offsets[i]); }
        head += '\n';
        const int rc = write(user, head.data(), head.size());
        if (rc) return refused(rc, head.size());
        written += head.size();
    }
    const int n_chunks = (int)bounds.size() - 1;
    auto enqueue = [&](int k) -> int {
        const int b = k & 1;
        const uint32_t r0 = bounds[k], r1 = bounds[k + 1];
        FB_CUDA(cudaStreamWaitEvent(st, S.ev_dx[3 * b + 2], 0));         // the copy of chunk k-2 has left this buffer
        FB_CUDA(cudaEventRecord(S.ev_dx[3 * b], st));
        k_dist_format<<<r1 - r0, kFmtThreads, 0, st>>>(P, r0, d_row_start, S.d_dx_chunk[b].as<char>());
        FB_CUDA(cudaGetLastError());
        ctx->launches++;
        FB_CUDA(cudaEventRecord(S.ev_dx[3 * b + 1], st));
        FB_CUDA(cudaStreamWaitEvent(ctx->copy_stream, S.ev_dx[3 * b + 1], 0));
        FB_CUDA(cudaMemcpyAsync(S.h_dx_chunk[b], S.d_dx_chunk[b].p, row_start[r1] - row_start[r0], cudaMemcpyDeviceToHost, ctx->copy_stream));
        FB_CUDA(cudaEventRecord(S.ev_dx[3 * b + 2], ctx->copy_stream));
        return FAMSA_OK;
    };
    for (int b = 0; b < 2; ++b) FB_CUDA(cudaEventRecord(S.ev_dx[3 * b + 2], ctx->copy_stream));
    float fmt_ms = 0.f;
    for (int k = 0; k < std::min(n_chunks, 2); ++k) FB_TRY(enqueue(k));
    for (int k = 0; k < n_chunks; ++k) {
        const int b = k & 1;
        FB_CUDA(cudaEventSynchronize(S.ev_dx[3 * b + 2]));
        float ms = 0.f;
        FB_CUDA(cudaEventElapsedTime(&ms, S.ev_dx[3 * b], S.ev_dx[3 * b + 1]));
        fmt_ms += ms;
        const uint64_t bytes = row_start[bounds[k + 1]] - row_start[bounds[k]];
        const int rc = bytes ? write(user, S.h_dx_chunk[b], bytes) : 0;
        if (rc) {
            FB_CUDA(cudaStreamSynchronize(st));                          // chunk k+1 may still be in flight
            FB_CUDA(cudaStreamSynchronize(ctx->copy_stream));
            if (bytes_written) *bytes_written = written;
            return refused(rc, bytes);
        }
        written += bytes;
        if (k + 2 < n_chunks) FB_TRY(enqueue(k + 2));
    }
    FB_CUDA(cudaStreamSynchronize(ctx->copy_stream));
    if (bytes_written) *bytes_written = written;
    ctx->lcs_timing.total_ms = lcs_total + prep_ms + fmt_ms;
    ctx->lcs_timing.main_ms = lcs_main;
    S.last_pairs = square ? (uint64_t)n * n : pairs;
    return FAMSA_OK;
}

} // namespace fb

// Formatter alone, for tests (exported, not declared in the header): n device-side floats -> the text num2str writes
// for them, each value followed by ','.  HOST pointers; *out_len = bytes written (out must hold 40 * n bytes).
namespace {
__global__ void k_debug_format(const float* __restrict__ v, uint64_t n, char* __restrict__ out)
{
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    unsigned long long a, b;
    fb::split_value(v[i], a, b);
    char* dst = out + i * fb::kMaxValueChars;
    fb::put_value(dst, a, b);
    const int len = fb::value_chars(a, b);
    dst[len] = ',';
    for (int k = len + 1; k < fb::kMaxValueChars; ++k) dst[k] = 0;
}
} // namespace

extern "C" int famsa_debug_format_f32(const float* values, uint64_t n, char* out, uint64_t* out_len)
{
    if (n && (!values || !out || !out_len)) { fb::set_error("NULL argument"); return FAMSA_E_INVALID; }
    if (out_len) *out_len = 0;
    if (!n) return FAMSA_OK;
    float* d_v = nullptr;
    char* d_out = nullptr;
    const size_t slot = fb::kMaxValueChars;
    FB_CUDA(cudaMalloc(&d_v, sizeof(float) * n));
    if (cudaMalloc(&d_out, slot * n) != cudaSuccess) { cudaGetLastError(); cudaFree(d_v); fb::set_error("out of device memory"); return FAMSA_E_NOMEM; }
    std::vector<char> slots(slot * n);
    int rc = [&]() -> int {
        FB_CUDA(cudaMemcpy(d_v, values, sizeof(float) * n, cudaMemcpyHostToDevice));
        k_debug_format<<<(unsigned)((n + 255) / 256), 256>>>(d_v, n, d_out);
        FB_CUDA(cudaGetLastError());
        FB_CUDA(cudaMemcpy(slots.data(), d_out, slot * n, cudaMemcpyDeviceToHost));
        return FAMSA_OK;
    }();
    cudaFree(d_v);
    cudaFree(d_out);
    if (rc) return rc;
    uint64_t at = 0;
    for (uint64_t i = 0; i < n; ++i) {
        const char* s = slots.data() + i * slot;
        const size_t len = strnlen(s, slot);
        memcpy(out + at, s, len);
        at += len;
    }
    *out_len = at;
    return FAMSA_OK;
}
