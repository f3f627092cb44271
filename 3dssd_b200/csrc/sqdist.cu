// sqdist.cu -- pairwise squared feature distance, the F-FPS input of the reference:
//   model_util.calc_square_dist(a, a, norm=False)  (/root/reference/lib/utils/model_util.py:144-160)
//   out[b,i,j] = (|a_i|^2 + |a_j|^2) - 2 <a_i, a_j>
// The reference gets <a_i,a_j> from a TF-1.4 cuBLAS SGEMM whose summation order is unspecified, so this
// kernel PINS the order (sequential fp32 fma chain over the channel index, starting from 0) to make the
// result reproducible bit-for-bit by the CPU oracle -- which is why it runs on the fp32 FMA pipe and not
// on tensor cores.  64x64 output tile per block, both operand slabs ([c][64], channel-major) resident in
// shared memory for the whole tile, 4x4 outputs per thread fed by two 16-byte broadcast loads per channel.
#include "common.cuh"

namespace ssd3d {

constexpr int SQ_TILE = 64;
constexpr int SQ_THREADS = 256;
constexpr int SQ_PITCH = 68;  // 64 + 4: keeps 16-byte alignment of the float4 reads, 4-way (not 32-way) staging conflicts

__global__ void __launch_bounds__(SQ_THREADS)
sqdist_kernel(int n, int c, const float *__restrict__ a, float *__restrict__ out)
{
    extern __shared__ float4 dyn_smem[];
    float *As = reinterpret_cast<float *>(dyn_smem);  // [c][64] rows of the i-tile
    float *Bs = As + (size_t)c * SQ_PITCH;             // [c][64] rows of the j-tile
    float *sqA = Bs + (size_t)c * SQ_PITCH;            // [64]
    float *sqB = sqA + SQ_TILE;                        // [64]

    // The pinned arithmetic is exactly symmetric (fma(a,b,.) == fma(b,a,.), fp add commutes), so only tile pairs on
    // or above the diagonal are computed and each result is stored twice: out[i,j] and out[j,i].
    if (blockIdx.x < blockIdx.y) return;
    const bool mirror = blockIdx.x != blockIdx.y;
    const int scene = blockIdx.z;
    const int i0 = blockIdx.y * SQ_TILE, j0 = blockIdx.x * SQ_TILE;
    const float *A = a + (size_t)scene * n * c;
    const int tid = threadIdx.x;

    // stage both slabs transposed; consecutive threads read consecutive channels of one point (coalesced)
    for (int e = tid; e < SQ_TILE * c; e += SQ_THREADS) {
        const int r = e / c, l = e - r * c;
        As[l * SQ_PITCH + r] = (i0 + r < n) ? A[(size_t)(i0 + r) * c + l] : 0.0f;
        Bs[l * SQ_PITCH + r] = (j0 + r < n) ? A[(size_t)(j0 + r) * c + l] : 0.0f;
    }
    __syncthreads();
    if (tid < 2 * SQ_TILE) {
        const float *S = tid < SQ_TILE ? As : Bs;
        const int r = tid & (SQ_TILE - 1);
        float s = 0.0f;
        for (int l = 0; l < c; l++) s = __fmaf_rn(S[l * SQ_PITCH + r], S[l * SQ_PITCH + r], s);
        (tid < SQ_TILE ? sqA : sqB)[r] = s;
    }
    __syncthreads();

    const int ty = tid / 16, tx = tid % 16;
    float acc[4][4];
#pragma unroll
    for (int y = 0; y < 4; y++)
#pragma unroll
        for (int x = 0; x < 4; x++) acc[y][x] = 0.0f;
    for (int l = 0; l < c; l++) {
        const float4 av = *reinterpret_cast<const float4 *>(As + l * SQ_PITCH + ty * 4);
        const float4 bv = *reinterpret_cast<const float4 *>(Bs + l * SQ_PITCH + tx * 4);
        const float ar[4] = {av.x, av.y, av.z, av.w};
        const float br[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
        for (int y = 0; y < 4; y++)
#pragma unroll
            for (int x = 0; x < 4; x++) acc[y][x] = __fmaf_rn(ar[y], br[x], acc[y][x]);
    }
    float *O = out + (size_t)scene * n * n;
#pragma unroll
    for (int y = 0; y < 4; y++) {
        const float si = sqA[ty * 4 + y];
#pragma unroll
        for (int x = 0; x < 4; x++)
            acc[y][x] = __fsub_rn(__fadd_rn(si, sqB[tx * 4 + x]), __fmul_rn(2.0f, acc[y][x]));
    }
#pragma unroll
    for (int y = 0; y < 4; y++) {
        const int i = i0 + ty * 4 + y;
        if (i >= n) continue;
        const int j = j0 + tx * 4;
        float *dst = O + (size_t)i * n + j;
        if (j + 3 < n && ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0))
            *reinterpret_cast<float4 *>(dst) = make_float4(acc[y][0], acc[y][1], acc[y][2], acc[y][3]);
        else
            for (int x = 0; x < 4; x++)
                if (j + x < n) dst[x] = acc[y][x];
    }
    if (mirror) {
#pragma unroll
        for (int x = 0; x < 4; x++) {
            const int j = j0 + tx * 4 + x;
            if (j >= n) continue;
            const int i = i0 + ty * 4;
            float *dst = O + (size_t)j * n + i;
            if (i + 3 < n && ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0))
                *reinterpret_cast<float4 *>(dst) = make_float4(acc[0][x], acc[1][x], acc[2][x], acc[3][x]);
            else
                for (int y = 0; y < 4; y++)
                    if (i + y < n) dst[y] = acc[y][x];
        }
    }
}

// 128x128 tile, 8x8 outputs per thread: 64 FFMA per 4 shared-memory loads, so the fp32 FMA pipe (not the LSU) is
// the limiter.  Same pinned arithmetic, same symmetric double store.
constexpr int SQ2_TILE = 128;
constexpr int SQ2_PITCH = 132;

__global__ void __launch_bounds__(SQ_THREADS)
sqdist128_kernel(int n, int c, const float *__restrict__ a, float *__restrict__ out)
{
    if (blockIdx.x < blockIdx.y) return;
    const bool mirror = blockIdx.x != blockIdx.y;
    extern __shared__ float4 dyn_smem[];
    float *As = reinterpret_cast<float *>(dyn_smem);
    float *Bs = As + (size_t)c * SQ2_PITCH;
    float *sqA = Bs + (size_t)c * SQ2_PITCH;
    float *sqB = sqA + SQ2_TILE;
    const int scene = blockIdx.z;
    const int i0 = blockIdx.y * SQ2_TILE, j0 = blockIdx.x * SQ2_TILE;
    const float *A = a + (size_t)scene * n * c;
    const int tid = threadIdx.x;
    for (int e = tid; e < SQ2_TILE * c; e += SQ_THREADS) {
        const int r = e / c, l = e - r * c;
        As[l * SQ2_PITCH + r] = (i0 + r < n) ? A[(size_t)(i0 + r) * c + l] : 0.0f;
        Bs[l * SQ2_PITCH + r] = (j0 + r < n) ? A[(size_t)(j0 + r) * c + l] : 0.0f;
    }
    __syncthreads();
    {
        const float *S = tid < SQ2_TILE ? As : Bs;
        const int r = tid & (SQ2_TILE - 1);
        float sacc = 0.0f;
        for (int l = 0; l < c; l++) sacc = __fmaf_rn(S[l * SQ2_PITCH + r], S[l * SQ2_PITCH + r], sacc);
        (tid < SQ2_TILE ? sqA : sqB)[r] = sacc;
    }
    __syncthreads();
    const int ty = tid / 16, tx = tid % 16;
    // fp32 pairs: two independent IEEE fmas each -- bit-identical to the scalar chain.
    float2 acc2[8][4];
#pragma unroll
    for (int y = 0; y < 8; y++)
#pragma unroll
        for (int x = 0; x < 4; x++) acc2[y][x] = make_float2(0.0f, 0.0f);
    for (int l = 0; l < c; l++) {
        const float4 a0 = *reinterpret_cast<const float4 *>(As + l * SQ2_PITCH + ty * 8);
        const float4 a1 = *reinterpret_cast<const float4 *>(As + l * SQ2_PITCH + ty * 8 + 4);
        const float4 b0 = *reinterpret_cast<const float4 *>(Bs + l * SQ2_PITCH + tx * 8);
        const float4 b1 = *reinterpret_cast<const float4 *>(Bs + l * SQ2_PITCH + tx * 8 + 4);
        const float ar[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
        const float2 bp[4] = {make_float2(b0.x, b0.y), make_float2(b0.z, b0.w), make_float2(b1.x, b1.y), make_float2(b1.z, b1.w)};
#pragma unroll
        for (int y = 0; y < 8; y++) {
            const float2 ap = make_float2(ar[y], ar[y]);
#pragma unroll
            for (int x = 0; x < 4; x++) acc2[y][x] = fma2_rn(ap, bp[x], acc2[y][x]);
        }
    }
    float acc[8][8];
#pragma unroll
    for (int y = 0; y < 8; y++)
#pragma unroll
        for (int x = 0; x < 4; x++) { acc[y][2 * x] = acc2[y][x].x; acc[y][2 * x + 1] = acc2[y][x].y; }
    float *O = out + (size_t)scene * n * n;
#pragma unroll
    for (int y = 0; y < 8; y++) {
        const float si = sqA[ty * 8 + y];
#pragma unroll
        for (int x = 0; x < 8; x++) acc[y][x] = __fsub_rn(__fadd_rn(si, sqB[tx * 8 + x]), __fmul_rn(2.0f, acc[y][x]));
    }
    // Stage the finished tile in shared memory (the operand slabs are dead by now) so that both the tile and its
    // mirror image leave as whole 512-byte rows instead of 16-byte fragments scattered over 32 rows.
    constexpr int SP = SQ2_TILE + 1;
    float *stage = reinterpret_cast<float *>(dyn_smem);
    __syncthreads();
#pragma unroll
    for (int y = 0; y < 8; y++)
#pragma unroll
        for (int x = 0; x < 8; x++) stage[(ty * 8 + y) * SP + tx * 8 + x] = acc[y][x];
    __syncthreads();
    const bool vec = (n % 4) == 0 && ((reinterpret_cast<uintptr_t>(out) & 15u) == 0);
    const int lane = tid & 31, wid = tid >> 5;
    for (int r = wid; r < SQ2_TILE; r += SQ_THREADS / 32) {
        const int i = i0 + r, j = j0 + lane * 4;
        if (i < n) {
            const float v0 = stage[r * SP + lane * 4], v1 = stage[r * SP + lane * 4 + 1];
            const float v2 = stage[r * SP + lane * 4 + 2], v3 = stage[r * SP + lane * 4 + 3];
            float *dst = O + (size_t)i * n + j;
            if (vec && j + 3 < n) *reinterpret_cast<float4 *>(dst) = make_float4(v0, v1, v2, v3);
            else {
                if (j < n) dst[0] = v0;
                if (j + 1 < n) dst[1] = v1;
                if (j + 2 < n) dst[2] = v2;
                if (j + 3 < n) dst[3] = v3;
            }
        }
        if (mirror) {                                     // out[j0 + r'][i0 + ...] = tile[...][r']  with r' = r
            const int jj = j0 + r, ii = i0 + lane * 4;
            if (jj < n) {
                const float v0 = stage[(lane * 4) * SP + r], v1 = stage[(lane * 4 + 1) * SP + r];
                const float v2 = stage[(lane * 4 + 2) * SP + r], v3 = stage[(lane * 4 + 3) * SP + r];
                float *dst = O + (size_t)jj * n + ii;
                if (vec && ii + 3 < n) *reinterpret_cast<float4 *>(dst) = make_float4(v0, v1, v2, v3);
                else {
                    if (ii < n) dst[0] = v0;
                    if (ii + 1 < n) dst[1] = v1;
                    if (ii + 2 < n) dst[2] = v2;
                    if (ii + 3 < n) dst[3] = v3;
                }
            }
        }
    }
}

}  // namespace ssd3d

using namespace ssd3d;

extern "C" int ssd3d_calc_square_dist(int b, int n, int c, const float *a, float *out, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && n > 0 && c > 0, "calc_square_dist: bad shape b=%d n=%d c=%d", b, n, c);
    SSD3D_REQUIRE(a && out, "calc_square_dist: null pointer");
    if (b == 0) return 0;
    size_t smem128 = ((size_t)2 * c * SQ2_PITCH + 2 * SQ2_TILE) * sizeof(float);
    const size_t stage128 = (size_t)SQ2_TILE * (SQ2_TILE + 1) * sizeof(float);   // output staging reuses the slabs
    if (smem128 < stage128) smem128 = stage128;
    if (n >= 256 && smem128 <= 200 * 1024) {
        cudaError_t e2 = cudaFuncSetAttribute((const void *)sqdist128_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem128);
        if (e2 != cudaSuccess) return cuda_status(e2, "calc_square_dist attr");
        dim3 grid2((unsigned)ceil_div(n, SQ2_TILE), (unsigned)ceil_div(n, SQ2_TILE), (unsigned)b);
        sqdist128_kernel<<<grid2, SQ_THREADS, smem128, (cudaStream_t)stream>>>(n, c, a, out);
        SSD3D_LAUNCH_CHECK("sqdist128_kernel");
    }
    const size_t smem = ((size_t)2 * c * SQ_PITCH + 2 * SQ_TILE) * sizeof(float);
    SSD3D_REQUIRE(smem <= 220 * 1024, "calc_square_dist: c=%d too large for the shared-memory slabs", c);
    cudaError_t e = cudaFuncSetAttribute((const void *)sqdist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return cuda_status(e, "calc_square_dist attr");
    dim3 grid((unsigned)ceil_div(n, SQ_TILE), (unsigned)ceil_div(n, SQ_TILE), (unsigned)b);
    sqdist_kernel<<<grid, SQ_THREADS, smem, (cudaStream_t)stream>>>(n, c, a, out);
    SSD3D_LAUNCH_CHECK("sqdist_kernel");
}
