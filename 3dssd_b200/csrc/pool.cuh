// pool.cuh -- max-pool over the rows of a warp-held tile: "reduce and transpose" butterfly.
#pragma once

namespace ssd3d {

// One step over v[0 .. 2*half): lanes that differ in bit o exchange halves and each keeps the maximum of the half its
// bit selects, so the number of live values per lane halves.  o and half are arguments, not template parameters, so that
// warp_colmax_transpose can stay a loop: unrolling it fully costs the sa_fused layer-2 kernels ~10 registers.  Callers
// that hold a wgmma fragment pass literals, which fold under forced inlining.
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

// Each lane holds one ROW of a [32 rows x 32 columns] block in v[0..31].  Computes, for every run of GP consecutive
// lanes (rows), the column-wise maximum; on return lane L owns columns (L % GP) * (32/GP) + k, k < 32/GP, of its
// group's result in v[k].  31 shuffles for GP = 32 (instead of 32 full-warp reductions).
template <int GP>
__device__ __forceinline__ void warp_colmax_transpose(float (&v)[32], int lane)
{
#pragma unroll
    for (int o = GP / 2, cnt = 32; o >= 1; o >>= 1, cnt >>= 1) colmax_step(v, lane, o, cnt / 2);
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

}  // namespace ssd3d
