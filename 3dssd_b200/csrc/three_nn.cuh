// three_nn.cuh -- the device code of three_nn and three_interpolate, shared by three_nn.cu, gather_group.cu and the fused
// FP-layer operand kernel (fp_interp.cu), so that every route finds the same neighbours and interpolates the same bits.
#pragma once
#include "common.cuh"

namespace ssd3d {

constexpr int TNN_TILE = 1024;

// Running best three of one unknown point (ux, uy, uz) over the m known points of a scene, staged through the block's
// shared tile[TNN_TILE * 3] (every thread of the block must call this, valid or not: it synchronises the block).
//
// Bit-exactness with the reference (tf_interpolate_g.cu:24-84): squared distance with its contraction (dy*dy,
// fma(dx,dx,.), fma(dz,dz,.)), strict '<' so the earliest index wins ties.  The reference widens to double only to
// compare against its 1e40 initial value; an fp32 compare against +inf takes exactly the same decisions (inf < inf is
// false, as inf < 1e40 is), and (float)1e40 == +inf is what the reference stores when fewer than 3 points exist.
__device__ __forceinline__ void three_nn_scan(int m, const float *__restrict__ known, float *tile, float ux, float uy, float uz,
                                              float (&best)[3], int (&bidx)[3])
{
    float b1 = INFINITY, b2 = INFINITY, b3 = INFINITY;
    int i1 = 0, i2 = 0, i3 = 0;
    for (int base = 0; base < m; base += TNN_TILE) {
        const int npts = min(TNN_TILE, m - base);
        __syncthreads();
        for (int e = threadIdx.x; e < npts * 3; e += blockDim.x) tile[e] = known[(size_t)base * 3 + e];
        __syncthreads();
#pragma unroll 4
        for (int j = 0; j < npts; j++) {
            const float dx = tile[j * 3] - ux, dy = tile[j * 3 + 1] - uy, dz = tile[j * 3 + 2] - uz;
            float d = __fmul_rn(dy, dy);
            d = __fmaf_rn(dx, dx, d);
            d = __fmaf_rn(dz, dz, d);
            const int k = base + j;
            if (d < b1) { b3 = b2; i3 = i2; b2 = b1; i2 = i1; b1 = d; i1 = k; }
            else if (d < b2) { b3 = b2; i3 = i2; b2 = d; i2 = k; }
            else if (d < b3) { b3 = d; i3 = k; }
        }
    }
    best[0] = b1; best[1] = b2; best[2] = b3;
    bidx[0] = i1; bidx[1] = i2; bidx[2] = i3;
}

// fma(w3,c3, fma(w1,c1, w2*c2)) -- the reference's contraction (PTX of tf_interpolate_g.cu:110)
__device__ __forceinline__ float three_interp_value(float w1, float w2, float w3, float c1, float c2, float c3)
{
    float t = __fmul_rn(w2, c2);
    t = __fmaf_rn(w1, c1, t);
    return __fmaf_rn(w3, c3, t);
}

}  // namespace ssd3d
