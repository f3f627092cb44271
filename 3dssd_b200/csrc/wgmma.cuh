// wgmma.cuh -- Hopper warpgroup MMA (wgmma) helpers shared by mlp_tc.cu and sa_fused.cu.
//
// One wgmma.mma_async computes a 64-row slab D[64 x N] += A[64 x 16] . B[N x 16]^T for the four warps of a warpgroup,
// both operands read from shared memory through matrix descriptors, the fp32 accumulator held in registers: thread t of
// warp w holds rows 16w + t/4 (d[4j], d[4j+1]) and 16w + t/4 + 8 (d[4j+2], d[4j+3]) of columns 8j + 2(t%4) + {0, 1}.
// N is part of the instruction, hence one specialisation per width.
#pragma once
#include <stdint.h>

namespace ssd3d {

// K-major operand descriptor: rows of rb bytes (= the swizzle span: 128 -> SWIZZLE_128B, 64 -> _64B, 32 -> _32B),
// 8-row groups 8*rb bytes apart.  Advancing K by 16 bf16 elements adds 2 (32 bytes >> 4) to the descriptor.
__device__ __forceinline__ uint64_t wg_desc(uint32_t smem_addr, int rb)
{
    const uint64_t layout = rb == 128 ? 1ull : (rb == 64 ? 2ull : 3ull);
    return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | (1ull << 16) | ((uint64_t)((8 * rb) >> 4) << 32) | (layout << 62);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int PENDING>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(PENDING) : "memory"); }

template <int N> struct Wgmma;
template <> struct Wgmma<16> {
    static __device__ __forceinline__ void mma(float (&d)[8], uint64_t a, uint64_t b, uint32_t accumulate)
    {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "l"(a), "l"(b), "r"(accumulate));
    }
};
template <> struct Wgmma<32> {
    static __device__ __forceinline__ void mma(float (&d)[16], uint64_t a, uint64_t b, uint32_t accumulate)
    {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "l"(a), "l"(b), "r"(accumulate));
    }
};
template <> struct Wgmma<48> {
    static __device__ __forceinline__ void mma(float (&d)[24], uint64_t a, uint64_t b, uint32_t accumulate)
    {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
            : "l"(a), "l"(b), "r"(accumulate));
    }
};
template <> struct Wgmma<64> {
    static __device__ __forceinline__ void mma(float (&d)[32], uint64_t a, uint64_t b, uint32_t accumulate)
    {
        asm volatile(
            "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
            "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "l"(a), "l"(b), "r"(accumulate));
    }
};

// fp32 x ~= hi + lo (two bf16 terms) product through three bf16 MMAs: a_hi.b_hi + a_lo.b_hi + a_hi.b_lo
template <int N>
__device__ __forceinline__ void wg_mma3(float (&d)[N / 2], uint64_t a_hi, uint64_t a_lo, uint64_t b_hi, uint64_t b_lo,
                                        uint32_t accumulate)
{
    Wgmma<N>::mma(d, a_hi, b_hi, accumulate);
    Wgmma<N>::mma(d, a_lo, b_hi, 1u);
    Wgmma<N>::mma(d, a_hi, b_lo, 1u);
}

}  // namespace ssd3d
