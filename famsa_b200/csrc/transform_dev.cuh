// Device Transform<T, Distance> (reference src/tree/AbstractTreeGenerator.hpp:28-82), shared by lcs.cu and dist_export.cu.
#pragma once
#include <cstdint>

namespace fb {

// Transform<float, Distance> (AbstractTreeGenerator.hpp:28-82) with the host-computed (float) pow(i, 0.75) table;
// IEEE division, so the result is the host's bit for bit.
__device__ __forceinline__ float transform_f32(int kind, uint32_t lcs, uint32_t len1, uint32_t len2,
                                               const float* __restrict__ pow075, float never)
{
    if (kind == 2) return __fdiv_rn((float)lcs, (float)(len1 < len2 ? len1 : len2));
    const uint32_t indel_i = len1 + len2 - 2 * lcs;
    if (!lcs) return never;                                  // (float) nextafter((double) FLT_MAX, 0) == FLT_MAX
    if (kind == 0) return __fdiv_rn(pow075[indel_i], (float)lcs);
    return __fdiv_rn((float)indel_i, (float)lcs);
}

// Transform<double, Distance> with the host-libm (double) pow(i, 0.75) table.
__device__ __forceinline__ double transform_f64(int kind, uint32_t lcs, uint32_t len1, uint32_t len2,
                                                const double* __restrict__ pow075, double never)
{
    const uint32_t indel_i = len1 + len2 - 2 * lcs;
    if (!lcs) return never;                                  // nextafter(DBL_MAX, 0)
    if (kind == 0) return __ddiv_rn(pow075[indel_i], (double)lcs);
    return __ddiv_rn((double)indel_i, (double)lcs);
}

} // namespace fb
