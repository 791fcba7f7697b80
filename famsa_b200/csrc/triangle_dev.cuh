// The packed LCS triangle and the distances read from it: element (hi, lo), hi > lo, of a triangle of u16 or u32 LCS
// values, the LCS with a given sequence as seq0, and Transform<T, Distance> (reference src/tree/AbstractTreeGenerator.hpp:28-82).  Shared by lcs.cu, tree.cu,
// dist_export.cu and capi.cu.
#pragma once
#include <cstddef>
#include <cstdint>

namespace fb {

// Offset of element (hi, lo), lo < hi, in rows 1.. of the packed triangle; tri_index(r, 0) = pairs in the rows before r.
__host__ __device__ __forceinline__ size_t tri_index(uint32_t hi, uint32_t lo) { return (size_t)hi * (hi - 1) / 2 + lo; }

// LCS element `at` of an array of width eb (2 or 4 bytes)
__host__ __device__ __forceinline__ uint32_t lcs_load(const void* p, int eb, size_t at)
{
    return eb == 2 ? static_cast<const uint16_t*>(p)[at] : static_cast<const uint32_t*>(p)[at];
}
__host__ __device__ __forceinline__ void lcs_store(void* p, int eb, size_t at, uint32_t v)
{
    if (eb == 2) static_cast<uint16_t*>(p)[at] = (uint16_t)v;
    else static_cast<uint32_t*>(p)[at] = v;
}

// The LCS values as the reference computes them, with the row sequence as seq0: the true-LCS triangle (lcs_triangle
// without quirk fix-ups) and the own rows of the sequences whose value depends on being seq0 (lcs_side_rows).
struct Seq0View {
    const void* tri;               // true-LCS triangle, caller order
    int eb;                        // its element bytes
    uint32_t n;
    const int* side_idx;           // caller id -> its row in `side`, or -1
    const uint32_t* side;          // those rows, n wide, u32
};

// r's row in `side`, or -1 (always, with kSide = false: no side rows, every lookup reads the triangle).  Read once per
// row sequence: k_prim issues it at the top of a step, where its latency hides behind the step's other loads.
template <bool kSide>
__device__ __forceinline__ int side_row(const Seq0View& L, uint32_t r)
{
    return kSide ? L.side_idx[r] : -1;
}

// LCS with r as seq0 against c, s = side_row(L, r) (r != c, or r has a side row)
__device__ __forceinline__ uint32_t lcs_seq0(const Seq0View& L, int s, uint32_t r, uint32_t c)
{
    if (s >= 0) return L.side[(size_t)s * L.n + c];
    return lcs_load(L.tri, L.eb, tri_index(r > c ? r : c, r > c ? c : r));
}

// Transform's distance for "no common residue": (float) nextafter((double) FLT_MAX, 0) == FLT_MAX, and
// nextafter(DBL_MAX, 0)
constexpr float kNeverF32 = 0x1.fffffep+127f;
constexpr double kNeverF64 = 0x1.ffffffffffffep+1023;

// Transform<float, Distance> with the host-computed (float) pow(i, 0.75) table; IEEE division, so the result is the
// host's bit for bit.
__device__ __forceinline__ float transform_f32(int kind, uint32_t lcs, uint32_t len1, uint32_t len2,
                                               const float* __restrict__ pow075)
{
    if (kind == 2) return __fdiv_rn((float)lcs, (float)(len1 < len2 ? len1 : len2));
    const uint32_t indel_i = len1 + len2 - 2 * lcs;
    if (!lcs) return kNeverF32;
    if (kind == 0) return __fdiv_rn(pow075[indel_i], (float)lcs);
    return __fdiv_rn((float)indel_i, (float)lcs);
}

// Transform<double, Distance> with the host-libm (double) pow(i, 0.75) table.
__device__ __forceinline__ double transform_f64(int kind, uint32_t lcs, uint32_t len1, uint32_t len2,
                                                const double* __restrict__ pow075)
{
    const uint32_t indel_i = len1 + len2 - 2 * lcs;
    if (!lcs) return kNeverF64;
    if (kind == 0) return __ddiv_rn(pow075[indel_i], (double)lcs);
    return __ddiv_rn((double)indel_i, (double)lcs);
}

} // namespace fb
