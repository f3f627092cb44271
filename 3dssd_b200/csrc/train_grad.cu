// train_grad.cu -- backward operators of the training-mode SA / vote / head layers (DESIGN.md "Backward").
//
//   linear_wgrad       grad_w[cin, cout] = x^T . dz (+ grad_b = column sums of dz): the weight gradient of a 1x1 conv,
//                      on the tensor cores with the three-term bf16 split of the forward (csrc/wgmma.cuh, wg_mma3)
//   rowgroup_max_grad  backward of tf.reduce_max(axis=2) * mask (lib/utils/layers_util.py:178-180), ties split evenly
//   group_concat_grad  backward of the gather + centre-subtract + concat of layers_util.py:160-165
//   vote_translate_grad  backward of the clamp of vote_layer (layers_util.py:20-23)
// (the backward of the training BatchNorm lives next to its forward, in bn.cu)
//
// linear_wgrad.  The contraction runs over the ROWS of two row-major operands, i.e. both are MN-major for this product.
// One CTA = one warpgroup owns a 64 (cin) x BN (cout) tile of grad_w and one contiguous row range (split-K).  Per 64-row
// chunk its 128 threads load x[rows, ci] and dz[rows, co] column-wise (lanes = consecutive channels: coalesced), split
// each value into bf16 hi + lo, and store the pairs TRANSPOSED into the K-major SWIZZLE_128B layout the wgmma
// descriptors of wgmma.cuh read, so the operands are never rewritten in HBM.  Two smem stages: the loads of chunk i+1 are
// in flight while the wgmma group of chunk i runs.  Every split writes its fp32 tile to the caller's workspace and a
// second kernel adds the splits in a fixed order (in double): the result is the same bits from run to run, no atomics.
#include <cuda_bf16.h>

#include "common.cuh"
#include "wgmma.cuh"

namespace ssd3d {

constexpr int WG_BM = 64;          // grad_w rows (input channels) per CTA: the wgmma M
constexpr int WG_BK = 64;          // conv rows per chunk: one 128-byte swizzle row of bf16
constexpr int WG_THREADS = 128;
constexpr int WG_CTAS_PER_SM = 3;

static int wgrad_bn(int cout) { return cout <= 16 ? 16 : (cout <= 32 ? 32 : 64); }

// rows per split (a multiple of WG_BK) and the number of splits: about WG_CTAS_PER_SM CTAs per SM over all tiles
static void wgrad_plan(long rows, int cin, int cout, long &rps, int &splits)
{
    const long tiles = (long)ceil_div(cin, WG_BM) * ceil_div(cout, wgrad_bn(cout));
    const long chunks = (rows + WG_BK - 1) / WG_BK;
    long s = ((long)kNumSMs * WG_CTAS_PER_SM + tiles - 1) / tiles;
    s = s < chunks ? s : chunks;
    s = s < 1 ? 1 : s;
    rps = ((chunks + s - 1) / s) * WG_BK;
    splits = (int)((rows + rps - 1) / rps);
    if (splits < 1) splits = 1;
}

__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void split_pair_bf16(float x0, float x1, uint32_t &hw, uint32_t &lw)
{
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(hw) : "f"(x1), "f"(x0));       // {x1 : x0}: x0 at the lower k index
    const float h0 = __uint_as_float(hw << 16), h1 = __uint_as_float(hw & 0xffff0000u);
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(lw) : "f"(x1 - h1), "f"(x0 - h0));
}

// 8 consecutive rows of one channel -> one 16-byte chunk (k = 8 c16 .. 8 c16 + 7) of smem row `ch`, hi and lo images
__device__ __forceinline__ void store_chunk(uint8_t *img_hi, uint32_t lo_off, int ch, int c16, const float (&f)[8])
{
    uint32_t hw[4], lw[4];
#pragma unroll
    for (int t = 0; t < 4; t++) split_pair_bf16(f[2 * t], f[2 * t + 1], hw[t], lw[t]);
    const uint32_t off = (uint32_t)ch * 128u + (uint32_t)((c16 ^ (ch & 7)) << 4);
    *reinterpret_cast<uint4 *>(img_hi + off) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
    *reinterpret_cast<uint4 *>(img_hi + lo_off + off) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
}

template <int BN>
__global__ void __launch_bounds__(WG_THREADS, WG_CTAS_PER_SM)
linear_wgrad_kernel(long rows, int cin, int cout, const float *__restrict__ x, int ldx, const float *__restrict__ dz,
                    int lddz, long rps, float *__restrict__ part_w, double *__restrict__ part_b)
{
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    __shared__ double s_red[WG_THREADS];
    constexpr uint32_t A_BYTES = WG_BM * 128, B_BYTES = BN * 128, STAGE = 2 * A_BYTES + 2 * B_BYTES;
    constexpr int BJ = BN / 16;                              // B chunks per thread and 64-row chunk
    uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int ci0 = blockIdx.x * WG_BM, co0 = blockIdx.y * BN, split = blockIdx.z;
    const long r_begin = (long)split * rps;
    const long r_end = r_begin + rps < rows ? r_begin + rps : rows;
    const int nch = (int)((r_end - r_begin + WG_BK - 1) / WG_BK);
    // fixed channel per thread: A row ci (chunks c16 = tid/64 + 2j), B row co (chunks c16 = tid/BN + j*128/BN)
    const int a_ch = tid & (WG_BM - 1), a_c0 = tid >> 6;
    const int b_ch = tid % BN, b_c0 = tid / BN;
    const bool a_ok = ci0 + a_ch < cin, b_ok = co0 + b_ch < cout;
    const float *xa = x + ci0 + a_ch;
    const float *db = dz + co0 + b_ch;
    const bool want_b = part_b != nullptr && blockIdx.x == 0;
    float fa[4][8], fb[BJ][8];
    double sb = 0.0;

    auto load = [&](long r0) {
#pragma unroll
        for (int j = 0; j < 4; j++)
#pragma unroll
            for (int e = 0; e < 8; e++) {
                const long r = r0 + (a_c0 + 2 * j) * 8 + e;
                fa[j][e] = (a_ok && r < r_end) ? __ldg(xa + (size_t)r * ldx) : 0.0f;
            }
#pragma unroll
        for (int j = 0; j < BJ; j++)
#pragma unroll
            for (int e = 0; e < 8; e++) {
                const long r = r0 + (b_c0 + j * (WG_THREADS / BN)) * 8 + e;
                fb[j][e] = (b_ok && r < r_end) ? __ldg(db + (size_t)r * lddz) : 0.0f;
            }
    };

    float d[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; i++) d[i] = 0.0f;
    if (nch > 0) load(r_begin);
    for (int i = 0; i < nch; i++) {
        uint8_t *st = smem + (size_t)(i & 1) * STAGE;
        __syncthreads();                                     // every warp retired the wgmma group that read this stage
#pragma unroll
        for (int j = 0; j < 4; j++) store_chunk(st, A_BYTES, a_ch, a_c0 + 2 * j, fa[j]);
#pragma unroll
        for (int j = 0; j < BJ; j++) {
            store_chunk(st + 2 * A_BYTES, B_BYTES, b_ch, b_c0 + j * (WG_THREADS / BN), fb[j]);
            if (want_b) {
#pragma unroll
                for (int e = 0; e < 8; e++) sb += (double)fb[j][e];
            }
        }
        fence_proxy_async();
        __syncthreads();
        const uint32_t base = smem_u32(st);
        const uint64_t a_hi = wg_desc(base, 128), a_lo = wg_desc(base + A_BYTES, 128);
        const uint64_t b_hi = wg_desc(base + 2 * A_BYTES, 128), b_lo = wg_desc(base + 2 * A_BYTES + B_BYTES, 128);
        wg_fence();
#pragma unroll
        for (int ks = 0; ks < WG_BK / 16; ks++)
            wg_mma3<BN>(d, a_hi + 2 * ks, a_lo + 2 * ks, b_hi + 2 * ks, b_lo + 2 * ks, 1u);
        wg_commit();
        if (i + 1 < nch) load(r_begin + (long)(i + 1) * WG_BK);   // global loads overlap the MMAs
        wg_wait<1>();
    }
    wg_wait<0>();
    // fragment: rows 16w + lane/4 (+8), columns 8j + 2(lane%4) + {0,1}
    float *pw = part_w + (size_t)split * cin * cout;
    const int r0 = ci0 + warp * 16 + (lane >> 2), c = co0 + 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < BN / 8; j++) {
        const int col = c + 8 * j;
        if (r0 < cin) {
            if (col < cout) pw[(size_t)r0 * cout + col] = d[4 * j];
            if (col + 1 < cout) pw[(size_t)r0 * cout + col + 1] = d[4 * j + 1];
        }
        if (r0 + 8 < cin) {
            if (col < cout) pw[(size_t)(r0 + 8) * cout + col] = d[4 * j + 2];
            if (col + 1 < cout) pw[(size_t)(r0 + 8) * cout + col + 1] = d[4 * j + 3];
        }
    }
    if (want_b) {                                            // fixed-order combine of the threads sharing a column
        s_red[tid] = sb;
        __syncthreads();
        if (tid < BN && co0 + tid < cout) {
            double s = 0.0;
            for (int k = 0; k < WG_THREADS / BN; k++) s += s_red[tid + k * BN];
            part_b[(size_t)split * cout + co0 + tid] = s;
        }
    }
}

__global__ void wgrad_reduce_kernel(int splits, int cin, int cout, const float *__restrict__ part_w,
                                    const double *__restrict__ part_b, float *__restrict__ grad_w, float *__restrict__ grad_b)
{
    const long nw = (long)cin * cout;
    for (long e = blockIdx.x * (long)blockDim.x + threadIdx.x; e < nw + (grad_b ? cout : 0); e += (long)gridDim.x * blockDim.x) {
        double s = 0.0;
        if (e < nw) {
            for (int k = 0; k < splits; k++) s += (double)part_w[(size_t)k * nw + e];
            grad_w[e] = (float)s;
        } else {
            const long co = e - nw;
            for (int k = 0; k < splits; k++) s += part_b[(size_t)k * cout + co];
            grad_b[co] = (float)s;
        }
    }
}

// grad_y[g*pool + r, o] = (ind / num) * (grad_out[g, o] * mask[g]),  ind = (y == max), num = #ties: TF's _MinOrMaxGrad
// (indicators / num_selected) * grad after the Mul gradient of the mask, in the same float32 operation order
__global__ void rowgroup_max_grad_kernel(long groups, int pool, int c, const float *__restrict__ y, int ldy,
                                         const int *__restrict__ rowmask, const float *__restrict__ grad_out,
                                         float *__restrict__ grad_y, int ldgy)
{
    const long total = groups * c;
    for (long e = blockIdx.x * (long)blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x) {
        const long g = e / c;
        const int o = (int)(e - g * c);
        const float *yg = y + (size_t)g * pool * ldy + o;
        float mx = -INFINITY;
        for (int r = 0; r < pool; r++) mx = fmaxf(mx, yg[(size_t)r * ldy]);
        int num = 0;
        for (int r = 0; r < pool; r++) num += yg[(size_t)r * ldy] == mx;
        float gm = __ldg(grad_out + e);
        if (rowmask) gm = __fmul_rn(gm, rowmask[g] != 0 ? 1.0f : 0.0f);
        float *out = grad_y + (size_t)g * pool * ldgy + o;
        for (int r = 0; r < pool; r++)
            out[(size_t)r * ldgy] = __fmul_rn(__fdiv_rn(yg[(size_t)r * ldy] == mx ? 1.0f : 0.0f, (float)num), gm);
    }
}

// grad_x[row, 0:c] -> grad_points[scene, idx[row], :], grad_x[row, c:c+3] -> grad_xyz[scene, idx[row], :] (fp32 atomics)
__global__ void group_concat_scatter_kernel(long rows, int n, int c, int m, int ns, const int *__restrict__ idx,
                                            const float *__restrict__ gx, int ldx, float *__restrict__ grad_points,
                                            float *__restrict__ grad_xyz)
{
    const int w = (grad_points ? c : 0) + 3;
    const long total = rows * w;
    const long rows_per_scene = (long)m * ns;
    for (long e = blockIdx.x * (long)blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x) {
        const long row = e / w;
        int col = (int)(e - row * w);
        if (!grad_points) col += c;
        const int a = __ldg(idx + row);
        if (a < 0) continue;
        const long scene = row / rows_per_scene;
        const float v = __ldg(gx + (size_t)row * ldx + col);
        if (col < c) atomicAdd(grad_points + ((size_t)scene * n + a) * c + col, v);
        else if (grad_xyz) atomicAdd(grad_xyz + ((size_t)scene * n + a) * 3 + (col - c), v);
    }
}

// grad_new_xyz[q, k] = -sum_s grad_x[q*ns + s, c + k]   (sequential over s: deterministic)
__global__ void group_concat_centre_kernel(long queries, int c, int ns, const float *__restrict__ gx, int ldx,
                                           float *__restrict__ grad_new_xyz)
{
    const long total = queries * 3;
    for (long e = blockIdx.x * (long)blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x) {
        const long q = e / 3;
        const int k = (int)(e - q * 3);
        float s = 0.0f;
        for (int j = 0; j < ns; j++) s += __ldg(gx + ((size_t)q * ns + j) * ldx + c + k);
        grad_new_xyz[e] = -s;
    }
}

// grad_offsets = grad_out where lo <= off <= -lo, else 0 (tf.maximum / tf.minimum route ties to their first input)
__global__ void vote_translate_grad_kernel(long rows, const float *__restrict__ off, int ldoff, const float *__restrict__ gout,
                                           float lx, float ly, float lz, float *__restrict__ goff)
{
    const long total = rows * 3;
    for (long e = blockIdx.x * (long)blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x) {
        const long r = e / 3;
        const int l = (int)(e - r * 3);
        const float lo = l == 0 ? lx : (l == 1 ? ly : lz);
        const float v = off[r * ldoff + l];
        goff[e] = (v >= lo && v <= -lo) ? gout[e] : 0.0f;
    }
}

static int grid_1d(long total)
{
    const long want = (total + 255) / 256;
    return (int)(want < 1 ? 1 : (want < (long)kNumSMs * 16 ? want : (long)kNumSMs * 16));
}

template <int BN>
static int launch_wgrad(long rows, int cin, int cout, const float *x, int ldx, const float *dz, int lddz, long rps, int splits,
                        float *part_w, double *part_b, cudaStream_t st)
{
    const size_t smem = 2 * (size_t)(2 * WG_BM * 128 + 2 * BN * 128) + 1024;
    cudaError_t e = cudaFuncSetAttribute(linear_wgrad_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return cuda_status(e, "linear_wgrad_kernel attribute");
    dim3 grid((unsigned)ceil_div(cin, WG_BM), (unsigned)ceil_div(cout, BN), (unsigned)splits);
    linear_wgrad_kernel<BN><<<grid, WG_THREADS, smem, st>>>(rows, cin, cout, x, ldx, dz, lddz, rps, part_w, part_b);
    return cuda_status(cudaGetLastError(), "linear_wgrad_kernel");
}

}  // namespace ssd3d

using namespace ssd3d;

extern "C" size_t ssd3d_linear_wgrad_workspace(long rows, int cin, int cout)
{
    if (rows <= 0 || cin <= 0 || cout <= 0) return 0;
    long rps;
    int splits;
    wgrad_plan(rows, cin, cout, rps, splits);
    return (size_t)splits * cout * sizeof(double) + (size_t)splits * cin * cout * sizeof(float);
}

extern "C" int ssd3d_linear_wgrad(long rows, int cin, int cout, const float *x, int ldx, const float *dz, int lddz,
                                  void *workspace, size_t workspace_bytes, float *grad_w, float *grad_b, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(rows > 0 && cin > 0 && cout > 0 && ldx >= cin && lddz >= cout,
                  "linear_wgrad: bad shape rows=%ld cin=%d cout=%d ldx=%d lddz=%d", rows, cin, cout, ldx, lddz);
    SSD3D_REQUIRE(x && dz && workspace && grad_w, "linear_wgrad: null pointer");
    SSD3D_REQUIRE(workspace_bytes >= ssd3d_linear_wgrad_workspace(rows, cin, cout),
                  "linear_wgrad: workspace of %zu bytes, %zu needed", workspace_bytes, ssd3d_linear_wgrad_workspace(rows, cin, cout));
    SSD3D_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 7u) == 0, "linear_wgrad: workspace must be 8-byte aligned");
    long rps;
    int splits;
    wgrad_plan(rows, cin, cout, rps, splits);
    double *part_b = grad_b ? (double *)workspace : nullptr;
    float *part_w = (float *)((double *)workspace + (size_t)splits * cout);
    cudaStream_t st = (cudaStream_t)stream;
    const int bn = wgrad_bn(cout);
    int rc = bn == 16 ? launch_wgrad<16>(rows, cin, cout, x, ldx, dz, lddz, rps, splits, part_w, part_b, st)
           : bn == 32 ? launch_wgrad<32>(rows, cin, cout, x, ldx, dz, lddz, rps, splits, part_w, part_b, st)
                      : launch_wgrad<64>(rows, cin, cout, x, ldx, dz, lddz, rps, splits, part_w, part_b, st);
    if (rc) return rc;
    wgrad_reduce_kernel<<<grid_1d((long)cin * cout + cout), 256, 0, st>>>(splits, cin, cout, part_w, part_b, grad_w, grad_b);
    SSD3D_LAUNCH_CHECK("wgrad_reduce_kernel");
}

extern "C" int ssd3d_rowgroup_max_grad(long groups, int pool, int c, const float *y, int ldy, const int *rowmask,
                                       const float *grad_out, float *grad_y, int ldgy, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(groups >= 0 && pool >= 1 && c > 0 && ldy >= c && ldgy >= c, "rowgroup_max_grad: bad shape");
    if (groups == 0) return 0;
    SSD3D_REQUIRE(y && grad_out && grad_y, "rowgroup_max_grad: null pointer");
    rowgroup_max_grad_kernel<<<grid_1d(groups * c), 256, 0, (cudaStream_t)stream>>>(groups, pool, c, y, ldy, rowmask, grad_out,
                                                                                   grad_y, ldgy);
    SSD3D_LAUNCH_CHECK("rowgroup_max_grad_kernel");
}

extern "C" int ssd3d_group_concat_grad(int b, int n, int c, int m, int nsample, const int *idx, const float *grad_x, int ldx,
                                       float *grad_points, float *grad_xyz, float *grad_new_xyz, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && n > 0 && m >= 0 && c >= 0 && nsample > 0 && ldx >= c + 3, "group_concat_grad: bad shape");
    SSD3D_REQUIRE(idx && grad_x, "group_concat_grad: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaSuccess;
    if (grad_points && c > 0) e = cudaMemsetAsync(grad_points, 0, sizeof(float) * (size_t)b * n * c, st);
    if (e == cudaSuccess && grad_xyz) e = cudaMemsetAsync(grad_xyz, 0, sizeof(float) * (size_t)b * n * 3, st);
    if (e != cudaSuccess) return cuda_status(e, "group_concat_grad memset");
    const long rows = (long)b * m * nsample;
    if (rows == 0) return 0;
    if (grad_points && c == 0) grad_points = nullptr;
    if (grad_points || grad_xyz) {
        group_concat_scatter_kernel<<<grid_1d(rows * ((grad_points ? c : 0) + 3)), 256, 0, st>>>(rows, n, c, m, nsample, idx,
                                                                                                grad_x, ldx, grad_points, grad_xyz);
        int rc = cuda_status(cudaGetLastError(), "group_concat_scatter_kernel");
        if (rc) return rc;
    }
    if (!grad_new_xyz) return 0;
    group_concat_centre_kernel<<<grid_1d((long)b * m * 3), 256, 0, st>>>((long)b * m, c, nsample, grad_x, ldx, grad_new_xyz);
    SSD3D_LAUNCH_CHECK("group_concat_centre_kernel");
}

extern "C" int ssd3d_vote_translate_grad(long rows, const float *offsets, int ld_offsets, const float *grad_out, float min_x,
                                         float min_y, float min_z, float *grad_offsets, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(rows >= 0 && ld_offsets >= 3, "vote_translate_grad: bad shape rows=%ld ld=%d", rows, ld_offsets);
    if (rows == 0) return 0;
    SSD3D_REQUIRE(offsets && grad_out && grad_offsets, "vote_translate_grad: null pointer");
    vote_translate_grad_kernel<<<grid_1d(rows * 3), 256, 0, (cudaStream_t)stream>>>(rows, offsets, ld_offsets, grad_out, min_x,
                                                                                     min_y, min_z, grad_offsets);
    SSD3D_LAUNCH_CHECK("vote_translate_grad_kernel");
}
