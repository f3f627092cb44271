// operand.cuh -- the split-bf16 operand format of the tensor-core kernels (mlp_tc.cu, sa_fused.cu, train_grad.cu).
//
// Every fp32 operand of a wgmma GEMM is stored as two bf16 terms, x = hi + lo with hi = bf16(x), lo = bf16(x - hi)
// (wgmma.cuh, wg_mma3).  The routes that build an operand in shared memory or in HBM -- TMA-fed, gathered by producer
// warps, materialised by an elementwise pass, or fused into a whole SA scale -- all build it with the helpers below, so
// the route that runs changes the speed, never the bits.
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

namespace ssd3d {

// Split of a value pair, packed {x1 : x0} like two adjacent bf16 (x0 at the lower column)
__device__ __forceinline__ void split_pair(float x0, float x1, uint32_t &hw, uint32_t &lw)
{
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(hw) : "f"(x1), "f"(x0));
    const float h0 = __uint_as_float(hw << 16), h1 = __uint_as_float(hw & 0xffff0000u);
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(lw) : "f"(x1 - h1), "f"(x0 - h0));
}

// Split of one value
__device__ __forceinline__ void split_one(float x, __nv_bfloat16 &h, __nv_bfloat16 &l)
{
    h = __float2bfloat16_rn(x);
    l = __float2bfloat16_rn(x - __bfloat162float(h));
}
__device__ __forceinline__ void split_store(float x, __nv_bfloat16 *hi, __nv_bfloat16 *lo) { split_one(x, *hi, *lo); }

// 8 consecutive columns f[i0 .. i0+7] -> split -> the 16-byte hi chunk h and lo chunk l
template <int N>
__device__ __forceinline__ void split8(const float (&f)[N], int i0, uint4 &h, uint4 &l)
{
    uint32_t hw[4], lw[4];
#pragma unroll
    for (int t = 0; t < 4; t++) split_pair(f[i0 + 2 * t], f[i0 + 2 * t + 1], hw[t], lw[t]);
    h = make_uint4(hw[0], hw[1], hw[2], hw[3]);
    l = make_uint4(lw[0], lw[1], lw[2], lw[3]);
}
// ... stored at hi and lo (16-byte aligned)
__device__ __forceinline__ void split_store8(void *hi, void *lo, const float (&f)[8])
{
    uint4 h, l;
    split8(f, 0, h, l);
    *reinterpret_cast<uint4 *>(hi) = h;
    *reinterpret_cast<uint4 *>(lo) = l;
}

// Byte offset of 16-byte chunk c16 (columns 8 c16 .. 8 c16 + 7) of `row` in a K-major SWIZZLE_128B tile of 128-byte
// rows, the layout the wgmma descriptors (wg_desc(.., 128)) and the 128B-swizzled TMA boxes use
__device__ __forceinline__ uint32_t sw128_chunk(uint32_t row, uint32_t c16) { return row * 128u + ((c16 ^ (row & 7u)) << 4); }

// Unit lists (include/ssd3d.h, ssd3d_query_ball_point_multi_ws_ex): desc = (group << 4) | j names rows U j .. U j + U-1
// of neighbour list `group`, U = 1 << lgu rows per unit (8 or 4, fixed per list).  Row e (< U) of the unit is entry
// unit_slot(desc, ns, lgu, e) of idx[] (grouped rows < 2^31).  Templated kernels pass lgu as a literal.
__device__ __forceinline__ uint32_t unit_group(uint32_t desc) { return desc >> 4; }
__device__ __forceinline__ uint32_t unit_slot(uint32_t desc, uint32_t ns, uint32_t lgu, uint32_t e) { return (desc >> 4) * ns + ((desc & 15u) << lgu) + e; }

// Columns k0 .. k0+7 of a grouped operand row concat(src_f[0:c], src_x - ctr) cut at column kend (c + 3, or c when only
// the features are wanted), zero beyond kend and for a row that does not exist (!ok).  vec: src_f is 16-byte aligned.
__device__ __forceinline__ void load_concat8(float (&f)[8], const float *src_f, const float *src_x, const float *ctr, int c,
                                             int kend, int k0, bool vec, bool ok)
{
    if (vec && ok && k0 + 8 <= c) {
        const float4 u0 = __ldg(reinterpret_cast<const float4 *>(src_f + k0));
        const float4 u1 = __ldg(reinterpret_cast<const float4 *>(src_f + k0 + 4));
        f[0] = u0.x; f[1] = u0.y; f[2] = u0.z; f[3] = u0.w;
        f[4] = u1.x; f[5] = u1.y; f[6] = u1.z; f[7] = u1.w;
        return;
    }
#pragma unroll
    for (int e = 0; e < 8; e++) {
        const int k = k0 + e;
        float val = 0.0f;
        if (ok) {
            if (k < c) val = __ldg(src_f + k);
            else if (k < kend) val = __ldg(src_x + (k - c)) - __ldg(ctr + (k - c));
        }
        f[e] = val;
    }
}

// The operand of the conv after a hoisted first conv (DESIGN.md 3.4): 8 columns of relu(z + d . Wx'), z in f on entry.
// w: column k0 of the [3][kp] table Wx' (16-byte aligned, zero beyond the first conv's width, where z is zero too, so
// the padding columns come out +0: fmaf(d, +0, +0) is +0 for finite d).
__device__ __forceinline__ void hoisted_row8(float (&f)[8], const float *w, int kp, float dx, float dy, float dz)
{
#pragma unroll
    for (int e4 = 0; e4 < 8; e4 += 4) {
        const float4 w0 = *reinterpret_cast<const float4 *>(w + e4);
        const float4 w1 = *reinterpret_cast<const float4 *>(w + kp + e4);
        const float4 w2 = *reinterpret_cast<const float4 *>(w + 2 * kp + e4);
        f[e4 + 0] = fmaxf(fmaf(dz, w2.x, fmaf(dy, w1.x, fmaf(dx, w0.x, f[e4 + 0]))), 0.0f);
        f[e4 + 1] = fmaxf(fmaf(dz, w2.y, fmaf(dy, w1.y, fmaf(dx, w0.y, f[e4 + 1]))), 0.0f);
        f[e4 + 2] = fmaxf(fmaf(dz, w2.z, fmaf(dy, w1.z, fmaf(dx, w0.z, f[e4 + 2]))), 0.0f);
        f[e4 + 3] = fmaxf(fmaf(dz, w2.w, fmaf(dy, w1.w, fmaf(dx, w0.w, f[e4 + 3]))), 0.0f);
    }
}

// Pooled output value (row, col): 0 for a masked group (the cnt == 0 mask of layers_util.py:180), then the fp32 and / or
// the split-bf16 output (a null pointer: not wanted).  Each address is formed only where its store is made.
__device__ __forceinline__ void store_pooled_value(float v, bool masked, size_t row, int col, float *out_f32, int ld_f32,
                                                   __nv_bfloat16 *out_hi, __nv_bfloat16 *out_lo, int ld_split)
{
    v = masked ? 0.0f : v;
    if (out_f32) asm volatile("st.global.f32 [%0], %1;" ::"l"(out_f32 + row * ld_f32 + col), "f"(v) : "memory");
    if (out_hi) {
        __nv_bfloat16 h, l;
        split_one(v, h, l);
        asm volatile("st.global.b16 [%0], %1;" ::"l"(out_hi + row * ld_split + col), "h"(__bfloat16_as_ushort(h)) : "memory");
        asm volatile("st.global.b16 [%0], %1;" ::"l"(out_lo + row * ld_split + col), "h"(__bfloat16_as_ushort(l)) : "memory");
    }
}

// Unit-list pooling: a post-ReLU value (>= 0) combined into the caller's zero-filled fp32 output by atomicMax on its bit
// pattern -- for non-negative floats the unsigned order of the bits is the float order (a -0.0 is folded to +0.0)
__device__ __forceinline__ void atomic_max_nonneg(float *dst, float v)
{
    atomicMax(reinterpret_cast<unsigned int *>(dst), __float_as_uint(v) & 0x7fffffffu);
}

}  // namespace ssd3d
