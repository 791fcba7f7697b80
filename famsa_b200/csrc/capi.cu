// C ABI of libfamsa_b200.so -- see include/famsa_b200.h for the contract of every entry point.
#include <cfloat>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <new>
#include <numeric>
#include <algorithm>
#include <vector>

#include "ctx.h"
#include "triangle_dev.cuh"

namespace fb {
int DevBuf::reserve(size_t bytes)
{
    if (bytes <= cap) return FAMSA_OK;
    release();
    size_t want = bytes + bytes / 8 + 256;
    cudaError_t e = cudaMalloc(&p, want);
    if (e != cudaSuccess) {
        p = nullptr;
        cudaGetLastError();          // callers may recover (famsa_lcs_prim falls back): do not leave the error for a later check
        set_error(std::string("cudaMalloc(") + std::to_string(want) + ") failed: " + cudaGetErrorString(e));
        return FAMSA_E_NOMEM;
    }
    cap = want;
    return FAMSA_OK;
}
void DevBuf::release()
{
    if (p) cudaFree(p);
    p = nullptr;
    cap = 0;
}

static thread_local std::string g_error;
void set_error(const std::string& msg) { g_error = msg; }
const char* get_error() { return g_error.c_str(); }

int scratch_acquire(famsa_ctx* ctx, cudaStream_t st)
{
    if (ctx->busy) FB_CUDA(cudaStreamWaitEvent(st, ctx->ev_busy, 0));
    return FAMSA_OK;
}
int scratch_release(famsa_ctx* ctx, cudaStream_t st, bool synced)
{
    if (synced) { ctx->busy = false; return FAMSA_OK; }
    FB_CUDA(cudaEventRecord(ctx->ev_busy, st));
    ctx->busy = true;
    return FAMSA_OK;
}
} // namespace fb

using fb::set_error;
using fb::tri_index;

#define FB_CHECK_CTX(ctx)                          \
    if (!(ctx)) {                                  \
        set_error("famsa_ctx is NULL");            \
        return FAMSA_E_INVALID;                    \
    }

// ------------------------------------------------------------------ the frame of an entry point

// Reads the call's timing once its stream is synchronised: total = ev[0]..ev[3], main = ev[1]..ev[2]
static int finish_timing(famsa_ctx* ctx, fb::CallTiming* t)
{
    FB_CUDA(cudaEventSynchronize(ctx->ev[3]));
    FB_CUDA(cudaEventElapsedTime(&t->total_ms, ctx->ev[0], ctx->ev[3]));
    FB_CUDA(cudaEventElapsedTime(&t->main_ms, ctx->ev[1], ctx->ev[2]));
    return FAMSA_OK;
}

// Every entry point that queues work on the context's scratch: the NULL context, the lock, the argument checks (`check`,
// before anything is queued), the device, the stream (the caller's, or the context's for NULL), the scratch order, then
// `run`.  On a caller's stream the call returns with its work queued and the scratch held until that work is done; on the
// context's stream it synchronises and, given `t`, reads the call's timing.
using Timing = fb::CallTiming famsa_ctx::*;

template <class Check, class Run>
static int entry(famsa_ctx* ctx, void* stream, Timing t, Check check, Run run)
{
    FB_CHECK_CTX(ctx);
    std::lock_guard<std::mutex> lk(ctx->mu);
    FB_TRY(check());
    FB_CUDA(cudaSetDevice(ctx->device));
    const cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : ctx->stream;
    FB_TRY(fb::scratch_acquire(ctx, st));
    FB_TRY(run(st));
    if (stream) return fb::scratch_release(ctx, st, false);
    FB_CUDA(cudaStreamSynchronize(st));
    fb::scratch_release(ctx, st, true);
    return t ? finish_timing(ctx, &(ctx->*t)) : FAMSA_OK;
}

// An LCS call's events: ev[0] and ev[3] around all it queues; lcs_triangle and lcs_rows mark their tile kernels in ev[1]
// and ev[2], and a call without any gets an empty span.
template <class Run>
static int lcs_timed(famsa_ctx* ctx, cudaStream_t st, Run run)
{
    ctx->lcs.tiles_marked = false;
    FB_CUDA(cudaEventRecord(ctx->ev[0], st));
    FB_TRY(run());
    if (!ctx->lcs.tiles_marked) { FB_CUDA(cudaEventRecord(ctx->ev[1], st)); FB_CUDA(cudaEventRecord(ctx->ev[2], st)); }
    FB_CUDA(cudaEventRecord(ctx->ev[3], st));
    return FAMSA_OK;
}

static int check_set(const famsa_ctx* ctx, uint32_t min_n)
{
    if (ctx->lcs.n >= min_n) return FAMSA_OK;
    set_error(ctx->lcs.n ? "the call needs at least " + std::to_string(min_n) + " uploaded sequences"
                         : std::string("famsa_lcs_upload has not been called"));
    return FAMSA_E_STATE;
}

// elem_bytes is 2 or 4 and at least `need` (LcsState::elem_bytes() for the LCS the library computes)
static int check_elem(int elem_bytes, int need)
{
    if (elem_bytes != 2 && elem_bytes != 4) { set_error("elem_bytes must be 2 or 4"); return FAMSA_E_INVALID; }
    if (elem_bytes < need) { set_error("elem_bytes == 2 needs every sequence shorter than 65536"); return FAMSA_E_INVALID; }
    return FAMSA_OK;
}

static int check_rows(const famsa_ctx* ctx, uint32_t row_begin, uint32_t row_end)
{
    if (row_begin <= row_end && row_end <= ctx->lcs.n) return FAMSA_OK;
    set_error("row range out of bounds");
    return FAMSA_E_INVALID;
}

static int check_ids(const famsa_ctx* ctx, const uint32_t* ids, uint32_t count, const char* what)
{
    for (uint32_t k = 0; k < count; ++k)
        if (ids[k] >= ctx->lcs.n) { set_error(std::string(what) + " id out of range"); return FAMSA_E_INVALID; }
    return FAMSA_OK;
}

extern "C" {

int famsa_abi_version(void) { return FAMSA_B200_ABI_VERSION; }

const char* famsa_last_error(void) { return fb::get_error(); }

int famsa_create(int device, famsa_ctx** out_ctx)
{
    if (!out_ctx) { set_error("out_ctx is NULL"); return FAMSA_E_INVALID; }
    *out_ctx = nullptr;
    int count = 0;
    cudaError_t e = cudaGetDeviceCount(&count);
    if (e != cudaSuccess || count == 0) {
        set_error(std::string("no CUDA device available (") + cudaGetErrorString(e) +
                  "); libfamsa_b200 has no CPU fallback");
        return FAMSA_E_NO_DEVICE;
    }
    if (device < 0) FB_CUDA(cudaGetDevice(&device));
    if (device >= count) { set_error("device ordinal out of range"); return FAMSA_E_INVALID; }
    FB_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop{};
    FB_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {
        set_error(std::string("device '") + prop.name + "' is sm_" + std::to_string(prop.major) +
                  std::to_string(prop.minor) + "; this library is built for sm_90a only");
        return FAMSA_E_NO_DEVICE;
    }
    famsa_ctx* ctx = new (std::nothrow) famsa_ctx();
    if (!ctx) { set_error("out of host memory"); return FAMSA_E_NOMEM; }
    ctx->device = device;
    ctx->sm_count = prop.multiProcessorCount;
    const int rc = [&]() -> int {
        FB_CUDA(cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking));
        for (auto& ev : ctx->ev) FB_CUDA(cudaEventCreate(&ev));
        FB_CUDA(cudaEventCreateWithFlags(&ctx->ev_busy, cudaEventDisableTiming));
        FB_CUDA(cudaEventCreateWithFlags(&ctx->ev_fork, cudaEventDisableTiming));
        for (auto& e : ctx->ev_copy) FB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        for (auto& e : ctx->ev_join) FB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        for (auto& a : ctx->aux_stream) FB_CUDA(cudaStreamCreateWithFlags(&a, cudaStreamNonBlocking));
        FB_CUDA(cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
        for (auto& e : ctx->ev_block) FB_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        for (auto& e : ctx->ev_host) FB_CUDA(cudaEventCreate(&e));
        // per-call scratch and resident profiles are stream-ordered allocations: the pool keeps what it has
        cudaMemPool_t pool;
        FB_CUDA(cudaDeviceGetDefaultMemPool(&pool, device));
        unsigned long long keep = ~0ull;
        FB_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep));
        return FAMSA_OK;
    }();
    if (rc) { famsa_destroy(ctx); return rc; }
    *out_ctx = ctx;
    return FAMSA_OK;
}

void famsa_destroy(famsa_ctx* ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    fb::dist_export_release(ctx);
    fb::refine_release(ctx);
    fb::prof_release_all(ctx);
    if (ctx->dp.h_pinned) cudaFreeHost(ctx->dp.h_pinned);
    for (auto& ev : ctx->ev)
        if (ev) cudaEventDestroy(ev);
    for (auto& ev : ctx->ev_block)
        if (ev) cudaEventDestroy(ev);
    for (auto& ev : ctx->ev_host)
        if (ev) cudaEventDestroy(ev);
    if (ctx->ev_busy) cudaEventDestroy(ctx->ev_busy);
    if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
    for (auto& e : ctx->ev_copy)
        if (e) cudaEventDestroy(e);
    for (auto& st : ctx->peer_stream)
        if (st) cudaStreamDestroy(st);
    for (auto& e : ctx->ev_join)
        if (e) cudaEventDestroy(e);
    for (auto& a : ctx->aux_stream)
        if (a) cudaStreamDestroy(a);
    if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;                                                    // the device buffers free themselves
}

uint64_t famsa_kernel_launches(const famsa_ctx* ctx) { return ctx ? ctx->launches : 0; }

// ------------------------------------------------------------------ HP-1

int famsa_lcs_upload(famsa_ctx* ctx, const int8_t* codes, const uint64_t* offsets, const uint32_t* lens,
                     uint32_t n_seqs)
{
    return entry(ctx, nullptr, nullptr, [&]() -> int {
        if (n_seqs && (!codes || !offsets || !lens)) { set_error("NULL sequence arrays"); return FAMSA_E_INVALID; }
        return FAMSA_OK;
    }, [&](cudaStream_t st) -> int {
        FB_CUDA(cudaStreamSynchronize(st));                             // earlier *_device calls may still read the old set
        fb::scratch_release(ctx, st, true);
        ctx->lcs.h_order.clear();
        fb::tree_state_invalidate(ctx);                                 // the leaves of the kept tree change
        return fb::lcs_upload(ctx, codes, offsets, lens, n_seqs);
    });
}

int famsa_lcs_upload_sorted(famsa_ctx* ctx, const int8_t* codes, const uint64_t* offsets, const uint32_t* lens, uint32_t n_seqs)
{
    FB_CHECK_CTX(ctx);
    if (n_seqs && (!codes || !offsets || !lens)) { set_error("NULL sequence arrays"); return FAMSA_E_INVALID; }
    // the permutation the library would apply internally (length descending, ties in caller order), applied up front: every
    // index of the calls that follow is then a position in that order
    std::vector<uint32_t> order(n_seqs);
    std::iota(order.begin(), order.end(), 0u);
    std::stable_sort(order.begin(), order.end(), [&](uint32_t x, uint32_t y) { return lens[x] > lens[y]; });
    std::vector<uint64_t> off(n_seqs);
    std::vector<uint32_t> len(n_seqs);
    uint64_t total = 0;
    for (uint32_t p = 0; p < n_seqs; ++p) { off[p] = total; len[p] = lens[order[p]]; total += len[p]; }
    std::vector<int8_t> packed(std::max<uint64_t>(total, 1));
    for (uint32_t p = 0; p < n_seqs; ++p) memcpy(packed.data() + off[p], codes + offsets[order[p]], len[p]);
    const int rc = famsa_lcs_upload(ctx, packed.data(), off.data(), len.data(), n_seqs);
    if (rc) return rc;
    std::lock_guard<std::mutex> lk(ctx->mu);
    ctx->lcs.h_order = std::move(order);
    return FAMSA_OK;
}

int famsa_lcs_sorted_order(famsa_ctx* ctx, uint32_t* sorted_to_caller)
{
    FB_CHECK_CTX(ctx);
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (!sorted_to_caller && ctx->lcs.n) { set_error("sorted_to_caller is NULL"); return FAMSA_E_INVALID; }
    if (ctx->lcs.h_order.size() == ctx->lcs.n) std::copy(ctx->lcs.h_order.begin(), ctx->lcs.h_order.end(), sorted_to_caller);
    else std::iota(sorted_to_caller, sorted_to_caller + ctx->lcs.n, 0u);          // plain famsa_lcs_upload: indices are the caller's
    return FAMSA_OK;
}

uint64_t famsa_lcs_last_tiles(const famsa_ctx* ctx) { return ctx ? ctx->lcs.last_tiles : 0; }

uint32_t famsa_lcs_n_seqs(const famsa_ctx* ctx) { return ctx ? ctx->lcs.n : 0; }

int famsa_lcs_triangle_device(famsa_ctx* ctx, uint32_t row_begin, uint32_t row_end, void* d_out, int elem_bytes,
                              void* stream)
{
    return entry(ctx, stream, &famsa_ctx::lcs_timing, [&]() -> int {
        FB_TRY(check_set(ctx, row_end > 0 ? 1 : 0));
        FB_TRY(check_rows(ctx, row_begin, row_end));
        FB_TRY(check_elem(elem_bytes, ctx->lcs.elem_bytes()));
        if (!d_out && row_end > row_begin && row_end > 1) { set_error("d_out is NULL"); return FAMSA_E_INVALID; }
        return FAMSA_OK;
    }, [&](cudaStream_t st) -> int {
        ctx->lcs.last_pairs = tri_index(row_end, 0) - tri_index(row_begin, 0);
        return lcs_timed(ctx, st, [&] { return fb::lcs_triangle(ctx, row_begin, row_end, d_out, elem_bytes, st); });
    });
}

int famsa_lcs_triangle(famsa_ctx* ctx, uint32_t row_begin, uint32_t row_end, void* out, int elem_bytes)
{
    const uint64_t pairs = tri_index(row_end, 0) - tri_index(row_begin, 0);
    return entry(ctx, nullptr, nullptr, [&]() -> int {
        FB_TRY(check_rows(ctx, row_begin, row_end));
        FB_TRY(check_elem(elem_bytes, ctx->lcs.elem_bytes()));
        if (pairs && !out) { set_error("out is NULL"); return FAMSA_E_INVALID; }
        return FAMSA_OK;
    }, [&](cudaStream_t st) -> int {
        fb::LcsState& S = ctx->lcs;
        FB_TRY(S.d_out_stage.reserve(std::max<uint64_t>(pairs, 1) * elem_bytes));
        char* d_out = static_cast<char*>(S.d_out_stage.p);
        // Row blocks with equal numbers of pairs: all kernels are queued first, then every block is copied back as
        // soon as its event fires, so the D2H of block k overlaps the kernels of blocks k+1...
        constexpr int kBlocks = 8;
        // (worth it only when the copy is long compared with the tail of a kernel: hundreds of millions of pairs)
        unsigned long long block_min = 400000000ull;
        if (const char* e = getenv("FAMSA_LCS_BLOCK_MIN_PAIRS")) block_min = strtoull(e, nullptr, 10);   // test knob
        const int n_blocks = (S.identity_perm && pairs > block_min) ? kBlocks : 1;
        uint32_t bounds[kBlocks + 1];
        fb::lcs_row_pieces(row_begin, row_end, n_blocks, nullptr, bounds);
        FB_CUDA(cudaEventRecord(ctx->ev_host[0], st));
        FB_TRY(fb::lcs_triangle(ctx, row_begin, row_end, d_out, elem_bytes, st, bounds, n_blocks, ctx->ev_block, true, true));
        if (!S.identity_perm && n_blocks == 1) FB_CUDA(cudaEventRecord(ctx->ev_block[0], st));
        FB_CUDA(cudaEventRecord(ctx->ev_host[1], st));
        for (int b = 0; b < n_blocks; ++b) {
            const uint64_t off = (tri_index(bounds[b], 0) - tri_index(row_begin, 0)) * elem_bytes;
            const uint64_t bytes = (tri_index(bounds[b + 1], 0) - tri_index(bounds[b], 0)) * elem_bytes;
            if (!bytes) continue;
            FB_CUDA(cudaStreamWaitEvent(ctx->copy_stream, ctx->ev_block[b], 0));
            FB_CUDA(cudaMemcpyAsync(static_cast<char*>(out) + off, d_out + off, bytes, cudaMemcpyDeviceToHost, ctx->copy_stream));
        }
        FB_CUDA(cudaStreamSynchronize(st));
        FB_CUDA(cudaStreamSynchronize(ctx->copy_stream));
        // its own timing: the kernels of all blocks, their copies overlapped
        FB_CUDA(cudaEventElapsedTime(&ctx->lcs_timing.main_ms, ctx->ev_host[0], ctx->ev_host[1]));
        ctx->lcs_timing.total_ms = ctx->lcs_timing.main_ms;
        S.last_pairs = pairs;
        return FAMSA_OK;
    });
}

// ------------------------------------------------------------------ multi-GPU exchange over peer memory

int famsa_device_alloc(famsa_ctx* ctx, uint64_t bytes, void** d_ptr)
{
    FB_CHECK_CTX(ctx);
    if (!d_ptr) { set_error("d_ptr is NULL"); return FAMSA_E_INVALID; }
    FB_CUDA(cudaSetDevice(ctx->device));
    *d_ptr = nullptr;
    const cudaError_t e = cudaMalloc(d_ptr, std::max<uint64_t>(bytes, 1));   // a whole allocation: exportable as it is
    if (e == cudaErrorMemoryAllocation) { cudaGetLastError(); set_error("out of device memory (" + std::to_string(bytes) + " bytes)"); return FAMSA_E_NOMEM; }
    FB_CUDA(e);
    return FAMSA_OK;
}

int famsa_device_free(famsa_ctx* ctx, void* d_ptr)
{
    FB_CHECK_CTX(ctx);
    FB_CUDA(cudaSetDevice(ctx->device));
    FB_CUDA(cudaDeviceSynchronize());
    FB_CUDA(cudaFree(d_ptr));
    return FAMSA_OK;
}

int famsa_ipc_export(famsa_ctx* ctx, void* d_ptr, uint8_t handle[64])
{
    FB_CHECK_CTX(ctx);
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size is part of the ABI");
    if (!d_ptr || !handle) { set_error("NULL argument"); return FAMSA_E_INVALID; }
    FB_CUDA(cudaSetDevice(ctx->device));
    cudaIpcMemHandle_t h;
    FB_CUDA(cudaIpcGetMemHandle(&h, d_ptr));
    memcpy(handle, &h, 64);
    return FAMSA_OK;
}

int famsa_ipc_open(famsa_ctx* ctx, const uint8_t handle[64], void** d_ptr)
{
    FB_CHECK_CTX(ctx);
    if (!d_ptr || !handle) { set_error("NULL argument"); return FAMSA_E_INVALID; }
    FB_CUDA(cudaSetDevice(ctx->device));
    cudaIpcMemHandle_t h;
    memcpy(&h, handle, 64);
    FB_CUDA(cudaIpcOpenMemHandle(d_ptr, h, cudaIpcMemLazyEnablePeerAccess));
    return FAMSA_OK;
}

int famsa_ipc_close(famsa_ctx* ctx, void* d_ptr)
{
    FB_CHECK_CTX(ctx);
    FB_CUDA(cudaSetDevice(ctx->device));
    FB_CUDA(cudaDeviceSynchronize());
    FB_CUDA(cudaIpcCloseMemHandle(d_ptr));
    return FAMSA_OK;
}

int famsa_lcs_triangle_exchange(famsa_ctx* ctx, uint32_t row_begin, uint32_t row_end, void* d_full, void* const* d_peer_full,
                                uint32_t n_peers, int elem_bytes, uint32_t n_pieces, void* stream)
{
    constexpr uint32_t kPieces = sizeof(ctx->ev_block) / sizeof(ctx->ev_block[0]);
    return entry(ctx, stream, &famsa_ctx::lcs_timing, [&]() -> int {
        FB_TRY(check_set(ctx, 1));
        FB_TRY(check_rows(ctx, row_begin, row_end));
        if (!d_full || (n_peers && !d_peer_full)) { set_error("NULL triangle buffer"); return FAMSA_E_INVALID; }
        for (uint32_t k = 0; k < n_peers; ++k)
            if (!d_peer_full[k]) { set_error("NULL peer buffer"); return FAMSA_E_INVALID; }
        return check_elem(elem_bytes, ctx->lcs.elem_bytes());
    }, [&](cudaStream_t st) -> int {
        // Pieces (a non-identity order cannot be cut by rows: one piece).  The copy of the LAST piece is the only exposed part
        // of the exchange, so the pieces shrink towards the end: 14 % of the pairs each at first, 8 % at last.
        const uint32_t np = ctx->lcs.identity_perm ? std::min(std::max(n_pieces, 1u), kPieces) : 1u;
        static const double kCut8[9] = {0.0, 0.14, 0.28, 0.42, 0.56, 0.70, 0.82, 0.92, 1.0};
        double frac[kPieces + 1];
        for (uint32_t b = 0; b <= np; ++b) frac[b] = np == 8 ? kCut8[b] : (double)b / np;
        uint32_t bounds[kPieces + 1];
        fb::lcs_row_pieces(row_begin, row_end, (int)np, frac, bounds);
        ctx->lcs.last_pairs = tri_index(row_end, 0) - tri_index(row_begin, 0);
        char* own = static_cast<char*>(d_full) + tri_index(row_begin, 0) * elem_bytes;    // lcs_triangle indexes from its first row
        FB_TRY(lcs_timed(ctx, st, [&] {
            return fb::lcs_triangle(ctx, row_begin, row_end, own, elem_bytes, st, bounds, (int)np, ctx->ev_block, true, true);
        }));
        // every finished piece goes to the same place of every peer's triangle while the next pieces are being computed:
        // copy engines over NVLink, no SM and no collective kernel involved
        if (!n_peers) return FAMSA_OK;
        constexpr int kLanes = 1 + sizeof(ctx->peer_stream) / sizeof(ctx->peer_stream[0]);
        cudaStream_t lanes[kLanes];
        lanes[0] = ctx->copy_stream;
        for (int a = 1; a < kLanes; ++a) {
            if (!ctx->peer_stream[a - 1]) FB_CUDA(cudaStreamCreateWithFlags(&ctx->peer_stream[a - 1], cudaStreamNonBlocking));
            lanes[a] = ctx->peer_stream[a - 1];
        }
        const int n_lanes = (int)std::min<uint32_t>(n_peers, kLanes);
        for (uint32_t b = 0; b < np; ++b) {
            const uint64_t off = tri_index(bounds[b], 0) * elem_bytes, bytes = (tri_index(bounds[b + 1], 0) - tri_index(bounds[b], 0)) * elem_bytes;
            if (!bytes) continue;
            for (int a = 0; a < n_lanes; ++a) FB_CUDA(cudaStreamWaitEvent(lanes[a], ctx->ev_block[b], 0));
            for (uint32_t k = 0; k < n_peers; ++k)
                FB_CUDA(cudaMemcpyAsync(static_cast<char*>(d_peer_full[k]) + off, static_cast<char*>(d_full) + off, bytes,
                                        cudaMemcpyDeviceToDevice, lanes[k % n_lanes]));
        }
        for (int a = 0; a < n_lanes; ++a) {                           // the caller's stream continues after the last copy
            FB_CUDA(cudaEventRecord(ctx->ev_copy[a], lanes[a]));
            FB_CUDA(cudaStreamWaitEvent(st, ctx->ev_copy[a], 0));
        }
        return FAMSA_OK;
    });
}

int famsa_lcs_rows_device(famsa_ctx* ctx, const uint32_t* d_ref_ids, uint32_t n_ref, const uint32_t* d_col_ids,
                          uint32_t n_col, void* d_out, int elem_bytes, void* stream)
{
    std::vector<uint32_t> h_ref(n_ref);
    return entry(ctx, stream, &famsa_ctx::lcs_timing, [&]() -> int {
        FB_TRY(check_set(ctx, 1));
        FB_TRY(check_elem(elem_bytes, ctx->lcs.elem_bytes()));
        if (!d_col_ids && n_col > ctx->lcs.n) { set_error("n_col exceeds the number of sequences"); return FAMSA_E_INVALID; }
        if (n_ref && !d_ref_ids) { set_error("d_ref_ids is NULL"); return FAMSA_E_INVALID; }
        if (n_ref) {      // ordered on the caller's stream (a blocking copy on the legacy stream would not be)
            FB_CUDA(cudaSetDevice(ctx->device));
            cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : ctx->stream;
            FB_CUDA(cudaMemcpyAsync(h_ref.data(), d_ref_ids, sizeof(uint32_t) * n_ref, cudaMemcpyDeviceToHost, st));
            FB_CUDA(cudaStreamSynchronize(st));
        }
        return check_ids(ctx, h_ref.data(), n_ref, "ref");
    }, [&](cudaStream_t st) -> int {
        ctx->lcs.last_pairs = (uint64_t)n_ref * n_col;
        return lcs_timed(ctx, st, [&] { return fb::lcs_rows(ctx, h_ref.data(), n_ref, d_col_ids, n_col, d_out, elem_bytes, st); });
    });
}

int famsa_lcs_rows(famsa_ctx* ctx, const uint32_t* ref_ids, uint32_t n_ref, const uint32_t* col_ids, uint32_t n_col,
                   void* out, int elem_bytes)
{
    return entry(ctx, nullptr, &famsa_ctx::lcs_timing, [&]() -> int {
        FB_TRY(check_set(ctx, 1));
        FB_TRY(check_elem(elem_bytes, ctx->lcs.elem_bytes()));
        if (!col_ids && n_col > ctx->lcs.n) { set_error("n_col exceeds the number of sequences"); return FAMSA_E_INVALID; }
        if ((n_ref && !ref_ids) || (n_ref && n_col && !out)) { set_error("NULL argument"); return FAMSA_E_INVALID; }
        if (col_ids) FB_TRY(check_ids(ctx, col_ids, n_col, "col"));
        return check_ids(ctx, ref_ids, n_ref, "ref");
    }, [&](cudaStream_t st) -> int {
        fb::LcsState& S = ctx->lcs;
        const uint64_t cells = (uint64_t)n_ref * n_col;
        FB_TRY(S.d_out_stage.reserve(std::max<uint64_t>(cells, 1) * elem_bytes));
        const uint32_t* d_cols = nullptr;
        if (col_ids) {
            FB_TRY(S.d_ids_b.reserve(sizeof(uint32_t) * std::max(1u, n_col)));
            FB_CUDA(cudaMemcpyAsync(S.d_ids_b.p, col_ids, sizeof(uint32_t) * n_col, cudaMemcpyHostToDevice, st));
            d_cols = S.d_ids_b.as<uint32_t>();
        }
        S.last_pairs = cells;
        FB_TRY(lcs_timed(ctx, st, [&] { return fb::lcs_rows(ctx, ref_ids, n_ref, d_cols, n_col, S.d_out_stage.p, elem_bytes, st); }));
        if (cells) FB_CUDA(cudaMemcpyAsync(out, S.d_out_stage.p, cells * elem_bytes, cudaMemcpyDeviceToHost, st));
        return FAMSA_OK;
    });
}

int famsa_lcs_prim(famsa_ctx* ctx, int distance_kind, int32_t* edge_from, int32_t* edge_to, double* edge_dist,
                   int32_t* prim_order)
{
    std::vector<fb::MstEdge> tree;
    const int rc = entry(ctx, nullptr, &famsa_ctx::lcs_timing, [&]() -> int {
        FB_TRY(check_set(ctx, 1));
        if (!prim_order || (ctx->lcs.n > 1 && (!edge_from || !edge_to || !edge_dist))) { set_error("NULL argument"); return FAMSA_E_INVALID; }
        if (distance_kind != 0 && distance_kind != 1) { set_error("MSTPrim is instantiated for distance_kind 0 and 1 only"); return FAMSA_E_INVALID; }
        return FAMSA_OK;
    }, [&](cudaStream_t st) -> int {
        ctx->lcs.last_pairs = tri_index(ctx->lcs.n, 0);
        return lcs_timed(ctx, st, [&] { return fb::lcs_prim(ctx, distance_kind, edge_from, edge_to, edge_dist, prim_order, tree); });
    });
    if (rc || tree.empty()) return rc;
    return fb::prim_replay(tree, edge_from, edge_to, edge_dist, prim_order);     // host only: outside the call's timing
}

int famsa_lcs_slink(famsa_ctx* ctx, int distance_kind, int32_t* tree)
{
    std::vector<fb::MstEdge> edges;
    const int rc = entry(ctx, nullptr, &famsa_ctx::lcs_timing, [&]() -> int {
        FB_TRY(check_set(ctx, 1));
        if (!tree && ctx->lcs.n > 1) { set_error("NULL argument"); return FAMSA_E_INVALID; }
        if (distance_kind != 0 && distance_kind != 1) { set_error("SingleLinkage is instantiated for distance_kind 0 and 1 only"); return FAMSA_E_INVALID; }
        return FAMSA_OK;
    }, [&](cudaStream_t st) -> int {
        ctx->lcs.last_pairs = tri_index(ctx->lcs.n, 0);
        return lcs_timed(ctx, st, [&] { return fb::lcs_slink(ctx, distance_kind, edges); });
    });
    if (rc || edges.empty()) return rc;
    const uint32_t n = (uint32_t)edges.size() + 1;
    fb::slink_labels(std::move(edges), n, tree);                                // host only: outside the call's timing
    return FAMSA_OK;
}

int famsa_lcs_assign(famsa_ctx* ctx, const uint32_t* seed_ids, uint32_t n_seeds, int distance_kind, uint32_t* assignments,
                     float* min_dist)
{
    return entry(ctx, nullptr, &famsa_ctx::lcs_timing, [&]() -> int {
        FB_TRY(check_set(ctx, 1));
        if (!seed_ids || !n_seeds || !assignments || !min_dist) { set_error("NULL argument / no seeds"); return FAMSA_E_INVALID; }
        if (distance_kind < 0 || distance_kind > 2) { set_error("distance_kind must be 0, 1 or 2"); return FAMSA_E_INVALID; }
        return check_ids(ctx, seed_ids, n_seeds, "seed");
    }, [&](cudaStream_t st) -> int {
        ctx->lcs.last_pairs = (uint64_t)n_seeds * ctx->lcs.n;
        return lcs_timed(ctx, st, [&] { return fb::lcs_assign(ctx, seed_ids, n_seeds, distance_kind, assignments, min_dist); });
    });
}

int famsa_lcs_upgma(famsa_ctx* ctx, int distance_kind, int modified, int32_t* tree)
{
    return entry(ctx, nullptr, &famsa_ctx::lcs_timing, [&]() -> int {
        FB_TRY(check_set(ctx, 2));
        if (!tree) { set_error("NULL argument"); return FAMSA_E_INVALID; }
        if (distance_kind != 0 && distance_kind != 1) { set_error("UPGMA is instantiated for distance_kind 0 and 1 only"); return FAMSA_E_INVALID; }
        return FAMSA_OK;
    }, [&](cudaStream_t st) -> int {
        ctx->lcs.last_pairs = tri_index(ctx->lcs.n, 0);
        return lcs_timed(ctx, st, [&] { return fb::lcs_upgma(ctx, distance_kind, modified, tree); });
    });
}

int famsa_lcs_nj(famsa_ctx* ctx, int distance_kind, int32_t* tree)
{
    return entry(ctx, nullptr, &famsa_ctx::lcs_timing, [&]() -> int {
        FB_TRY(check_set(ctx, 2));
        if (!tree) { set_error("NULL argument"); return FAMSA_E_INVALID; }
        if (distance_kind != 0 && distance_kind != 1) { set_error("NeighborJoining is instantiated for distance_kind 0 and 1 only"); return FAMSA_E_INVALID; }
        return FAMSA_OK;
    }, [&](cudaStream_t st) -> int {
        ctx->lcs.last_pairs = tri_index(ctx->lcs.n, 0);
        return lcs_timed(ctx, st, [&] { return fb::lcs_nj(ctx, distance_kind, tree); });
    });
}

int famsa_lcs_upgma_from_triangle(famsa_ctx* ctx, int distance_kind, int modified, const void* d_triangle, int elem_bytes, int32_t* tree)
{
    return entry(ctx, nullptr, &famsa_ctx::lcs_timing, [&]() -> int {
        FB_TRY(check_set(ctx, 2));
        if (!tree || !d_triangle) { set_error("NULL argument"); return FAMSA_E_INVALID; }
        if (distance_kind != 0 && distance_kind != 1) { set_error("UPGMA is instantiated for distance_kind 0 and 1 only"); return FAMSA_E_INVALID; }
        return check_elem(elem_bytes, 2);                               // the caller's triangle: any width the caller chose
    }, [&](cudaStream_t st) -> int {
        ctx->lcs.last_pairs = 0;
        return lcs_timed(ctx, st, [&] { return fb::lcs_upgma(ctx, distance_kind, modified, tree, d_triangle, elem_bytes); });
    });
}

int famsa_lcs_assign_shard(famsa_ctx* ctx, const uint32_t* seed_ids, uint32_t n_seeds, int distance_kind, uint32_t shard,
                           uint32_t n_shards, int64_t* d_packed, void* stream)
{
    // (the seed ids are handed to an async copy from pageable memory: staged by the driver before the call returns)
    return entry(ctx, stream, &famsa_ctx::lcs_timing, [&]() -> int {
        FB_TRY(check_set(ctx, 1));
        if (!seed_ids || !n_seeds || !d_packed) { set_error("NULL argument / no seeds"); return FAMSA_E_INVALID; }
        if (distance_kind < 0 || distance_kind > 2) { set_error("distance_kind must be 0, 1 or 2"); return FAMSA_E_INVALID; }
        if (!n_shards || shard >= n_shards) { set_error("shard out of range"); return FAMSA_E_INVALID; }
        return check_ids(ctx, seed_ids, n_seeds, "seed");
    }, [&](cudaStream_t st) -> int {
        return lcs_timed(ctx, st, [&] {
            return fb::lcs_assign_shard(ctx, seed_ids, n_seeds, distance_kind, shard, n_shards, reinterpret_cast<long long*>(d_packed), st);
        });
    });
}

// Not through entry(): the export keeps its own timing and gives the scratch back even when it fails.
int famsa_dist_export(famsa_ctx* ctx, int distance_kind, int square, int pid, const char* ids, const uint64_t* id_offsets,
                      uint64_t chunk_bytes, famsa_write_fn write, void* user, uint64_t* bytes_written)
{
    FB_CHECK_CTX(ctx);
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (bytes_written) *bytes_written = 0;
    FB_TRY(check_set(ctx, 1));
    if (!ctx->lcs.h_order.empty()) {
        set_error("famsa_dist_export: the set was uploaded with famsa_lcs_upload_sorted; the export works in the caller's order "
                  "(upload it with famsa_lcs_upload)");
        return FAMSA_E_STATE;
    }
    if (!pid && distance_kind != 0 && distance_kind != 1) { set_error("famsa_dist_export: distance_kind must be 0 or 1"); return FAMSA_E_INVALID; }
    if (!ids || !id_offsets || !write) { set_error("famsa_dist_export: NULL ids, id_offsets or write"); return FAMSA_E_INVALID; }
    for (uint32_t i = 0; i < ctx->lcs.n; ++i)
        if (id_offsets[i + 1] < id_offsets[i]) { set_error("famsa_dist_export: id_offsets must not decrease"); return FAMSA_E_INVALID; }
    FB_CUDA(cudaSetDevice(ctx->device));
    FB_TRY(fb::scratch_acquire(ctx, ctx->stream));
    const int rc = fb::dist_export(ctx, distance_kind, square, pid, ids, id_offsets, chunk_bytes, write, user, bytes_written);
    cudaStreamSynchronize(ctx->stream);
    fb::scratch_release(ctx, ctx->stream, true);
    return rc;
}

int famsa_lcs_last_timing(const famsa_ctx* ctx, float* total_ms, float* main_kernel_ms, uint64_t* n_pairs)
{
    FB_CHECK_CTX(ctx);
    if (total_ms) *total_ms = ctx->lcs_timing.total_ms;
    if (main_kernel_ms) *main_kernel_ms = ctx->lcs_timing.main_ms;
    if (n_pairs) *n_pairs = ctx->lcs.last_pairs;
    return FAMSA_OK;
}

// ------------------------------------------------------------------ HP-2

int famsa_dp_align_batch(famsa_ctx* ctx, const famsa_dp_job* jobs, uint32_t n_jobs, const int64_t gaps[4],
                         famsa_dp_result* results, uint8_t* path_buf, uint8_t* dirs_buf)
{
    return entry(ctx, nullptr, &famsa_ctx::dp_timing, [&]() -> int {
        if (n_jobs && (!jobs || !gaps || !results || !path_buf)) { set_error("NULL argument"); return FAMSA_E_INVALID; }
        return FAMSA_OK;
    }, [&](cudaStream_t) { return fb::dp_run_host(ctx, jobs, n_jobs, gaps, results, path_buf, dirs_buf); });
}

int famsa_dp_align_batch_device(famsa_ctx* ctx, const famsa_dp_job* jobs, uint32_t n_jobs, const int64_t gaps[4],
                                famsa_dp_result* d_results, uint8_t* d_path_buf, uint8_t* d_dirs_buf, void* stream)
{
    return entry(ctx, stream, &famsa_ctx::dp_timing, [&]() -> int {
        if (n_jobs && (!jobs || !gaps || !d_results || !d_path_buf)) { set_error("NULL argument"); return FAMSA_E_INVALID; }
        return FAMSA_OK;
    }, [&](cudaStream_t st) {
        return fb::dp_run_device(ctx, jobs, nullptr, n_jobs, gaps, d_results, d_path_buf, d_dirs_buf, nullptr, nullptr, st);
    });
}

int famsa_dp_last_timing(const famsa_ctx* ctx, float* total_ms, float* kernel_ms, uint64_t* n_cells)
{
    FB_CHECK_CTX(ctx);
    if (total_ms) *total_ms = ctx->dp_timing.total_ms;
    if (kernel_ms) *kernel_ms = ctx->dp_timing.main_ms;
    if (n_cells) *n_cells = ctx->dp.last_cells;
    return FAMSA_OK;
}

// ------------------------------------------------------------------ resident profiles (SURVEY 8f-2)

int famsa_prof_set_scoring(famsa_ctx* ctx, const int64_t score_matrix[24 * 24])
{
    FB_CHECK_CTX(ctx);
    if (!score_matrix) { set_error("NULL argument"); return FAMSA_E_INVALID; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    FB_CUDA(cudaSetDevice(ctx->device));
    return fb::prof_set_scoring(ctx, score_matrix);
}

int famsa_prof_put(famsa_ctx* ctx, const famsa_dp_profile* profiles, uint32_t n, uint32_t* ids_out)
{
    FB_CHECK_CTX(ctx);
    if (n && (!profiles || !ids_out)) { set_error("NULL argument"); return FAMSA_E_INVALID; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    FB_CUDA(cudaSetDevice(ctx->device));
    return fb::prof_put(ctx, profiles, n, ids_out);
}

int famsa_prof_put_rows(famsa_ctx* ctx, const uint8_t* rows, uint32_t n_rows, uint32_t width, const int64_t gaps[4], int flags,
                        uint32_t* id_out)
{
    return entry(ctx, nullptr, nullptr, [&]() -> int {
        if (!rows || !gaps || !id_out) { set_error("NULL argument"); return FAMSA_E_INVALID; }
        if (flags & ~FAMSA_PUT_ROWS_FROM_TEXT) { set_error("famsa_prof_put_rows: unknown flags"); return FAMSA_E_INVALID; }
        return FAMSA_OK;
    }, [&](cudaStream_t) { return fb::prof_put_rows(ctx, rows, n_rows, width, gaps, flags, id_out); });
}

int famsa_prof_merge_batch(famsa_ctx* ctx, const famsa_prof_merge* merges, uint32_t n, const int64_t gaps[4],
                           uint32_t* merged_ids_out, famsa_dp_result* results, uint8_t* path_buf, uint64_t path_cap)
{
    // an empty batch leaves the timing of the last one
    return entry(ctx, nullptr, n ? &famsa_ctx::dp_timing : nullptr, [&]() -> int {
        if (n && (!merges || !gaps || !merged_ids_out || !results || !path_buf)) { set_error("NULL argument"); return FAMSA_E_INVALID; }
        return FAMSA_OK;
    }, [&](cudaStream_t) { return fb::prof_merge_batch(ctx, merges, n, gaps, merged_ids_out, results, path_buf, path_cap); });
}

int famsa_prof_align_tree(famsa_ctx* ctx, const int32_t* tree, uint32_t n_leaves, const int64_t gaps[4],
                          famsa_dp_result* results, uint32_t* root_id_out, uint64_t* path_bytes_out, famsa_tree_stats* stats)
{
    return entry(ctx, nullptr, nullptr, [&]() -> int {
        ctx->prof.tree_valid = false;                                   // a failed call leaves no tree for famsa_prof_tree_rows
        if (!tree || !gaps || !results) { set_error("NULL argument"); return FAMSA_E_INVALID; }
        return FAMSA_OK;
    }, [&](cudaStream_t) { return fb::prof_align_tree(ctx, tree, n_leaves, gaps, results, root_id_out, path_bytes_out, stats); });
}

int famsa_prof_tree_rows(famsa_ctx* ctx, const uint32_t* order, uint32_t n_rows, uint8_t* rows, uint64_t cap, uint32_t* width_out)
{
    return entry(ctx, nullptr, nullptr, [&]() -> int { return FAMSA_OK; },
                 [&](cudaStream_t) { return fb::prof_tree_rows(ctx, order, n_rows, rows, cap, width_out); });
}

int famsa_prof_tree_paths(famsa_ctx* ctx, uint8_t* path_buf, uint64_t path_cap)
{
    FB_CHECK_CTX(ctx);
    if (!path_buf) { set_error("NULL argument"); return FAMSA_E_INVALID; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    return fb::prof_tree_paths(ctx, path_buf, path_cap);
}

int famsa_prof_refine(famsa_ctx* ctx, uint32_t root_id, const uint8_t* rows, uint32_t n_rows, uint32_t width,
                      const int64_t gaps[4], uint32_t n_refinements, int flags, uint32_t* refined_id_out, uint32_t* width_out,
                      int64_t* total_score_out, famsa_refine_stats* stats)
{
    return entry(ctx, nullptr, nullptr, [&]() -> int {
        if (flags & FAMSA_REFINE_TREE_ROWS) {
            if (rows) { set_error("famsa_prof_refine: FAMSA_REFINE_TREE_ROWS takes the kept rows; rows must be NULL"); return FAMSA_E_INVALID; }
        } else if (!rows) { set_error("NULL argument"); return FAMSA_E_INVALID; }
        if (!gaps || !refined_id_out || !width_out || !total_score_out) { set_error("NULL argument"); return FAMSA_E_INVALID; }
        if (flags & ~(FAMSA_REFINE_NO_GAP_OPT | FAMSA_REFINE_NO_TOTAL_SCORE | FAMSA_REFINE_TREE_ROWS)) { set_error("famsa_prof_refine: unknown flags"); return FAMSA_E_INVALID; }
        return FAMSA_OK;
    }, [&](cudaStream_t) {
        return fb::prof_refine(ctx, root_id, rows, n_rows, width, gaps, n_refinements, flags, refined_id_out, width_out, total_score_out, stats);
    });
}

int famsa_prof_refined_rows(famsa_ctx* ctx, uint8_t* rows, uint64_t cap)
{
    FB_CHECK_CTX(ctx);
    if (!rows) { set_error("NULL argument"); return FAMSA_E_INVALID; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    FB_CUDA(cudaSetDevice(ctx->device));
    return fb::prof_refined_rows(ctx, rows, cap);
}

int famsa_prof_get(famsa_ctx* ctx, uint32_t id, uint32_t* width, uint32_t* card, int64_t* scores, int32_t* counters)
{
    FB_CHECK_CTX(ctx);
    std::lock_guard<std::mutex> lk(ctx->mu);
    FB_CUDA(cudaSetDevice(ctx->device));
    return fb::prof_get(ctx, id, width, card, scores, counters);
}

int famsa_prof_drop(famsa_ctx* ctx, const uint32_t* ids, uint32_t n)
{
    FB_CHECK_CTX(ctx);
    if (n && !ids) { set_error("NULL argument"); return FAMSA_E_INVALID; }
    std::lock_guard<std::mutex> lk(ctx->mu);
    FB_CUDA(cudaSetDevice(ctx->device));
    return fb::prof_drop(ctx, ids, n);
}

int famsa_prof_last_timing(famsa_ctx* ctx, float* total_ms, float* construct_ms)
{
    FB_CHECK_CTX(ctx);
    std::lock_guard<std::mutex> lk(ctx->mu);
    FB_CUDA(cudaSetDevice(ctx->device));
    return fb::prof_last_timing(ctx, total_ms, construct_ms);
}

int famsa_prof_stats(famsa_ctx* ctx, uint64_t* n_live, uint64_t* resident_bytes)
{
    FB_CHECK_CTX(ctx);
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (n_live) *n_live = ctx->prof.n_live;
    if (resident_bytes) *resident_bytes = ctx->prof.resident_bytes;
    return FAMSA_OK;
}

// ------------------------------------------------------------------ Transform<T, Distance>
// reference src/tree/AbstractTreeGenerator.hpp:28-82; kept on the host so that distances are
// bit-identical to the reference's (same libm pow, same float/double narrowing points).

double famsa_transform_f64(int kind, uint32_t lcs, uint32_t len1, uint32_t len2)
{
    if (kind == 2) return (double)lcs / std::min(len1, len2);
    const double indel = (double)(len1 + len2 - 2 * lcs);
    if (!lcs) return std::nextafter(DBL_MAX, 0.0);
    if (kind == 0) return (double)std::pow((double)(uint32_t)indel, 0.75) / (double)lcs;
    return indel / lcs;
}

float famsa_transform_f32(int kind, uint32_t lcs, uint32_t len1, uint32_t len2)
{
    if (kind == 2) return (float)lcs / std::min(len1, len2);
    const float indel = (float)(len1 + len2 - 2 * lcs);
    if (!lcs) return (float)std::nextafter((double)FLT_MAX, 0.0);
    if (kind == 0) return (float)std::pow((double)(uint32_t)indel, 0.75) / (float)lcs;
    return indel / lcs;
}

} // extern "C"
