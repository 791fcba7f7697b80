// Device-side records shared by the DP kernels (dp.cu) and the resident-profile kernels (prof.cu).
#pragma once
#include <cstdint>

namespace fb {

constexpr int kGapGO = 25, kGapGE = 26, kGapTE = 27, kGapTO = 28;   // GAP_OPEN, GAP_EXT, GAP_TERM_EXT, GAP_TERM_OPEN (defs.h:62-66)
constexpr long long kNegInf = -(1ll << 62);                        // infty (defs.h:57), takes part in additions unsaturated
constexpr uint32_t kWidthBad = 0xffffffffu;                        // published instead of a width when a merge failed

__host__ __device__ inline unsigned long long align_up(unsigned long long v, unsigned long long a) { return (v + a - 1) / a * a; }

// Skewed (wavefront-major) storage of the direction bytes: stripe k (rows 32k+1 .. 32k+32), wavefront step s, lane l hold
// cell (32k+1+l, s-l).  One warp step of k_dp_fill then writes 32 consecutive bytes instead of 32 different rows.
__host__ __device__ inline unsigned long long skew_elems_oriented(uint32_t wr, uint32_t wc)
{
    return (unsigned long long)((wr + 31) / 32) * 32ull * ((unsigned long long)wc + 32);
}
// the orientation is chosen on the device (k_dp_prep): reserve for the larger of the two
__host__ __device__ inline unsigned long long skew_elems(uint32_t w1, uint32_t w2)
{
    const unsigned long long a = skew_elems_oriented(w1, w2), b = skew_elems_oriented(w2, w1);
    return a > b ? a : b;
}

// One merge as the kernels see it.  w1 / w2 size every buffer of the job; when a child is itself a merge that is still
// queued on the stream they are upper bounds and the child's real width is read from *w1_src / *w2_src on the device.
struct DpJobDev {
    const long long* s1; const int* c1;
    const long long* s2; const int* c2;
    uint32_t w1, card1, w2, card2;
    const uint32_t* w1_src; const uint32_t* w2_src;
    uint32_t* w_dst;                                               // receives the merged width (path length), or kWidthBad
    unsigned long long path_off, dirs_off, scratch_off, t_off;     // t_off: offset of the job's skewed direction bytes
    uint32_t x1, x2;                                               // counter columns past the width that ProfProf's orientation counts
};

// host-side companion of famsa_dp_job for dp_run_device
struct DpJobExt {
    const uint32_t* w1_src; const uint32_t* w2_src;
    uint32_t* w_dst;
    // 1 for a profile built from rows read as text (FAMSA_PUT_ROWS_FROM_TEXT): its counters keep the set-aside last
    // column, which the reference's get_num_of_non_zeros counts (CalculateCountersScores sizes them gapped_size + 1)
    uint32_t x1 = 0, x2 = 0;
};

struct DpFusedPlan { unsigned long long scratch_bytes, skew_bytes, path_bytes, cells; };

struct DpMeta {            // written by k_dp_prep
    const long long* SR; const int* CR;        // row profile of the DP matrix (after the orientation swap)
    const long long* SC; const int* CC;        // column profile
    uint32_t WR, WC;                            // real widths
    int nR, nC, var, sw;
    int bad;               // 1: a count of the ProfProf tables is negative or exceeds the member count (not a profile CProfile can build); 2: a child merge failed
    int tmode;             // column-pair scores T: 0 IMMA with one counter digit, 1 IMMA with two, 2 scalar / look-up
    int t32;               // every T fits in int32: the fill's T ring holds 4-byte entries
};

} // namespace fb
