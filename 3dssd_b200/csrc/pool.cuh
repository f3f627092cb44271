// pool.cuh -- max-pool over the rows of a warp-held tile: "reduce and transpose" butterfly.
#pragma once

namespace ssd3d {

// One step over v[0 .. 2*half): lanes that differ in bit o exchange halves and each keeps the maximum of the half its
// bit selects, so the number of live values per lane halves.  Callers hold a wgmma fragment and pass literals, which fold
// under forced inlining.
template <int N>
__device__ __forceinline__ void colmax_step(float (&v)[N], int lane, int o, int half)
{
    const bool up = (lane & o) != 0;
#pragma unroll
    for (int i = 0; i < half; i++) {
        const float send = up ? v[i] : v[i + half];
        const float keep = up ? v[i + half] : v[i];
        v[i] = fmaxf(keep, __shfl_xor_sync(0xffffffffu, send, o));
    }
}

// The same over the 8 lanes of a column quad of a wgmma fragment (lane bits 2-4, i.e. the 8 rows t/4 of a fragment
// half): on return lane t owns, in v[i], the maximum of value slot i + (N/8)(t/4) over those 8 lanes.  N - N/8 shuffles.
// (The steps are written out: an index the compiler cannot resolve would move the accumulator fragment to local memory
// for the whole kernel.)
template <int N>
__device__ __forceinline__ void quad_rowmax_transpose(float (&v)[N], int lane)
{
    colmax_step(v, lane, 16, N / 2);
    colmax_step(v, lane, 8, N / 4);
    colmax_step(v, lane, 4, N / 8);
}

// The same over the 4 lanes of a column quad that share lane bit 4 (rows 0-3 or 4-7 of a fragment half, the 4-row units of
// a unit list): on return lane t owns, in v[i], i < N/4, the maximum of value slot i + (N/4)((t/4) % 4) over rows
// 4(t/16) .. 4(t/16)+3.  N/2 + N/4 shuffles, one step fewer than the 8-row pool.
template <int N>
__device__ __forceinline__ void quad_rowmax4_transpose(float (&v)[N], int lane)
{
    colmax_step(v, lane, 8, N / 2);
    colmax_step(v, lane, 4, N / 4);
}

}  // namespace ssd3d
