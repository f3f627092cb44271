// linear.cu -- 1x1 convolution + folded BatchNorm + ReLU (+ max-pool over the neighbour axis), fp32 FMA path.
//
// Replaces, for inference, the TF op chain of tf_util.conv2d / conv1d
// (/root/reference/lib/utils/tf_util.py:127-201, :51-124: conv, bias_add, unfused batch_norm :424-444, relu)
// and the tf.reduce_max + mask that closes each SA scale (/root/reference/lib/utils/layers_util.py:178-180):
// one kernel per layer instead of ~5 TF kernels that each stream [B,M,K,C] through HBM.
//
// This is the exact-fp32 path (CUDA-core FFMA, sequential-k accumulation per output): it serves the layers
// tensor cores cannot fill (Cin=4 first layer) and is the numerical cross-check of the wgmma path
// (mlp_tc.cu).  128x64 output tile per block, 8x4 outputs per thread, k-step 16.
#include "common.cuh"

namespace ssd3d {

int launch_rowgroup_max(long groups, int pool, int c, const float *y, int ldy, const int *rowmask, float *out,
                        cudaStream_t st);

constexpr int LN_BM = 128, LN_BN = 64, LN_BK = 16, LN_THREADS = 256;
constexpr int LN_XP = LN_BM + 4;

template <bool POOL>
__global__ void __launch_bounds__(LN_THREADS)
linear_kernel(long rows, int cin, int cout, const float *__restrict__ x, int ldx, const float *__restrict__ w,
              const float *__restrict__ scale, const float *__restrict__ shift, int relu, int pool,
              const int *__restrict__ rowmask, float *__restrict__ y, int ldy)
{
    __shared__ __align__(16) float Xs[LN_BK][LN_XP];
    __shared__ __align__(16) float Ws[LN_BK][LN_BN];
    __shared__ float stage[POOL ? LN_BM : 1][POOL ? LN_BN + 1 : 1];

    const int tid = threadIdx.x;
    const long row0 = (long)blockIdx.x * LN_BM;
    const int n0 = blockIdx.y * LN_BN;
    const int ty = tid / 16, tx = tid % 16;

    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; i++)
#pragma unroll
        for (int j = 0; j < 4; j++) acc[i][j] = 0.0f;

    for (int k0 = 0; k0 < cin; k0 += LN_BK) {
#pragma unroll
        for (int i = 0; i < 8; i++) {
            const int e = tid + i * LN_THREADS;
            const int r = e / LN_BK, kk = e % LN_BK;
            const long gr = row0 + r;
            Xs[kk][r] = (gr < rows && k0 + kk < cin) ? __ldg(x + (size_t)gr * ldx + k0 + kk) : 0.0f;
        }
#pragma unroll
        for (int i = 0; i < 4; i++) {
            const int e = tid + i * LN_THREADS;
            const int kk = e / LN_BN, nn = e % LN_BN;
            Ws[kk][nn] = (k0 + kk < cin && n0 + nn < cout) ? __ldg(w + (size_t)(k0 + kk) * cout + n0 + nn) : 0.0f;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < LN_BK; kk++) {
            const float4 a0 = *reinterpret_cast<const float4 *>(&Xs[kk][ty * 8]);
            const float4 a1 = *reinterpret_cast<const float4 *>(&Xs[kk][ty * 8 + 4]);
            const float4 bv = *reinterpret_cast<const float4 *>(&Ws[kk][tx * 4]);
            const float ar[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float br[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
            for (int i = 0; i < 8; i++)
#pragma unroll
                for (int j = 0; j < 4; j++) acc[i][j] = fmaf(ar[i], br[j], acc[i][j]);
        }
        __syncthreads();
    }

    float sc[4], sh[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
        const int o = n0 + tx * 4 + j;
        sc[j] = o < cout ? (scale ? __ldg(scale + o) : 1.0f) : 0.0f;
        sh[j] = o < cout ? (shift ? __ldg(shift + o) : 0.0f) : 0.0f;
    }
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const long gr = row0 + ty * 8 + i;
#pragma unroll
        for (int j = 0; j < 4; j++) {
            float v = fmaf(acc[i][j], sc[j], sh[j]);
            if (relu) v = fmaxf(v, 0.0f);
            if (POOL) stage[ty * 8 + i][tx * 4 + j] = gr < rows ? v : -INFINITY;
            else if (gr < rows && n0 + tx * 4 + j < cout) y[(size_t)gr * ldy + n0 + tx * 4 + j] = v;
        }
    }
    if (POOL) {
        __syncthreads();
        const int groups = LN_BM / pool;
        for (int e = tid; e < groups * LN_BN; e += LN_THREADS) {
            const int g = e / LN_BN, nn = e % LN_BN;
            const long gg = row0 / pool + g;
            if (gg * pool >= rows || n0 + nn >= cout) continue;
            float mx = -INFINITY;
            for (int r = 0; r < pool; r++) mx = fmaxf(mx, stage[g * pool + r][nn]);
            if (rowmask && rowmask[gg] == 0) mx = 0.0f;
            y[(size_t)gg * ldy + n0 + nn] = mx;
        }
    }
}

}  // namespace ssd3d

using namespace ssd3d;

extern "C" int ssd3d_linear_bn_relu(long rows, int cin, int cout, const float *x, int ldx, const float *w,
                                    const float *scale, const float *shift, int relu, int pool, const int *rowmask,
                                    float *y, int ldy, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(rows >= 0 && cin > 0 && cout > 0, "linear_bn_relu: bad shape rows=%ld cin=%d cout=%d", rows, cin, cout);
    SSD3D_REQUIRE(ldx >= cin && ldy >= cout, "linear_bn_relu: ldx=%d < cin=%d or ldy=%d < cout=%d", ldx, cin, ldy, cout);
    SSD3D_REQUIRE(x && w && y, "linear_bn_relu: null pointer");
    SSD3D_REQUIRE(pool >= 1 && rows % pool == 0, "linear_bn_relu: rows=%ld not a multiple of pool=%d", rows, pool);
    if (rows == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    dim3 grid((unsigned)ceil_div(rows, LN_BM), (unsigned)ceil_div(cout, LN_BN));
    if (pool > 1) {
        SSD3D_REQUIRE(LN_BM % pool == 0, "linear_bn_relu: fused pooling needs pool | %d (got %d)", LN_BM, pool);
        linear_kernel<true><<<grid, LN_THREADS, 0, st>>>(rows, cin, cout, x, ldx, w, scale, shift, relu, pool, rowmask, y, ldy);
    } else {
        linear_kernel<false><<<grid, LN_THREADS, 0, st>>>(rows, cin, cout, x, ldx, w, scale, shift, relu, 1, nullptr, y, ldy);
    }
    SSD3D_LAUNCH_CHECK("linear_kernel");
}

// max over runs of `pool` rows (any pool), for nsample values the fused epilogue does not cover
extern "C" int ssd3d_rowgroup_max(long groups, int pool, int c, const float *y, int ldy, const int *rowmask, float *out,
                                  ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(groups >= 0 && pool >= 1 && c > 0 && ldy >= c, "rowgroup_max: bad shape");
    SSD3D_REQUIRE(y && out, "rowgroup_max: null pointer");
    return launch_rowgroup_max(groups, pool, c, y, ldy, rowmask, out, (cudaStream_t)stream);
}
