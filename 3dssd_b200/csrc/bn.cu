// bn.cu -- training-mode BatchNorm of the SA-path convolutions (SURVEY.md section 8f, row f3).
//
// Replaces batch_norm_template with is_training=True (/root/reference/lib/utils/tf_util.py:424-444):
// tf.contrib.layers.batch_norm(center, scale, decay=bn_decay, updates_collections=None, fused=False), i.e.
//   mean, var = tf.nn.moments(x, all axes but the channel)              (population variance)
//   y = x * inv + (beta - mean * inv),  inv = gamma * rsqrt(var + 0.001)  (tf.nn.batch_normalization)
//   moving_mean -= (moving_mean - mean) * (1 - decay), same for moving_variance   (in place, during the forward)
// followed by the ReLU of the conv wrapper (tf_util.py:127-201).
//
// HBM-bound: two reads of x[rows, c] (statistics, then apply) and one write.  Statistics accumulate in double per
// thread (2M rows x fp32 would lose the variance of well-centred channels), partial sums per row-block go through a
// caller-owned workspace, a one-CTA finalize folds them, updates the moving statistics and emits the per-channel
// (scale, shift) pair that the apply pass -- and later the folded inference conv -- uses.
#include "common.cuh"

namespace ssd3d {

constexpr int BN_TX = 32, BN_TY = 8;
constexpr int BN_MAX_RB = 256;                // row blocks (partials per channel)

__global__ void __launch_bounds__(BN_TX * BN_TY)
bn_partial_kernel(long rows, int c, const float *__restrict__ x, int ldx, double *__restrict__ partial)
{
    __shared__ double s_sum[BN_TY][BN_TX], s_sq[BN_TY][BN_TX];
    const int tx = threadIdx.x, ty = threadIdx.y;
    const int col = blockIdx.x * BN_TX + tx;
    double sum = 0.0, sq = 0.0;
    if (col < c)
        for (long r = (long)blockIdx.y * BN_TY + ty; r < rows; r += (long)gridDim.y * BN_TY) {
            const double v = (double)__ldg(x + (size_t)r * ldx + col);
            sum += v; sq += v * v;
        }
    s_sum[ty][tx] = sum; s_sq[ty][tx] = sq;
    __syncthreads();
    if (ty == 0 && col < c) {
#pragma unroll
        for (int i = 1; i < BN_TY; i++) { sum += s_sum[i][tx]; sq += s_sq[i][tx]; }
        partial[((size_t)blockIdx.y * 2 + 0) * c + col] = sum;
        partial[((size_t)blockIdx.y * 2 + 1) * c + col] = sq;
    }
}

__global__ void bn_finalize_kernel(int nrb, long rows, int c, const double *__restrict__ partial, const float *__restrict__ gamma,
                                   const float *__restrict__ beta, float *__restrict__ moving_mean,
                                   float *__restrict__ moving_var, float decay, float eps, float *__restrict__ scale,
                                   float *__restrict__ shift, float *__restrict__ batch_mean, float *__restrict__ batch_var)
{
    const int col = blockIdx.x * blockDim.x + threadIdx.x;
    if (col >= c) return;
    double sum = 0.0, sq = 0.0;
    for (int rb = 0; rb < nrb; rb++) { sum += partial[((size_t)rb * 2) * c + col]; sq += partial[((size_t)rb * 2 + 1) * c + col]; }
    const double mean_d = sum / (double)rows;
    double var_d = sq / (double)rows - mean_d * mean_d;
    var_d = var_d > 0.0 ? var_d : 0.0;
    const float mean = (float)mean_d, var = (float)var_d;
    const float inv = __fmul_rn(gamma[col], __frsqrt_rn(__fadd_rn(var, eps)));
    scale[col] = inv;
    shift[col] = __fsub_rn(beta[col], __fmul_rn(mean, inv));
    if (batch_mean) batch_mean[col] = mean;
    if (batch_var) batch_var[col] = var;
    if (moving_mean) {   // assign_moving_average: variable -= (variable - value) * (1 - decay)
        const float om = 1.0f - decay;
        moving_mean[col] = __fsub_rn(moving_mean[col], __fmul_rn(__fsub_rn(moving_mean[col], mean), om));
        moving_var[col] = __fsub_rn(moving_var[col], __fmul_rn(__fsub_rn(moving_var[col], var), om));
    }
}

__global__ void scale_shift_act_kernel(long rows, int c, const float *__restrict__ x, int ldx, const float *__restrict__ scale,
                                       const float *__restrict__ shift, int relu, float *__restrict__ out, int ldo)
{
    const long total = rows * c;
    for (long e = blockIdx.x * (long)blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x) {
        const long r = e / c;
        const int col = (int)(e - r * c);
        float v = __fmaf_rn(x[(size_t)r * ldx + col], scale[col], shift[col]);
        if (relu) v = fmaxf(v, 0.0f);
        out[(size_t)r * ldo + col] = v;
    }
}

// ---- backward (DESIGN.md "Backward"): with x^ = (x - mean) * r, r = rsqrt(var + eps), g = upstream gradient times the
// forward's own ReLU decision fma(x, scale, shift) > 0, the batch-statistics gradient is
//   grad_beta = sum g,  grad_gamma = sum g x^,  grad_x = gamma r / N * (N g - sum g - x^ sum g x^)
// sums per channel in double (partials per row block, fixed-order finalize), the apply pass in double per element.
__device__ __forceinline__ float relu_masked(float g, float x, float scale, float shift, int relu)
{
    return (relu && !(__fmaf_rn(x, scale, shift) > 0.0f)) ? 0.0f : g;
}

__global__ void __launch_bounds__(BN_TX * BN_TY)
bn_grad_partial_kernel(long rows, int c, const float *__restrict__ x, int ldx, const float *__restrict__ gout, int ldg,
                       const float *__restrict__ scale, const float *__restrict__ shift, const float *__restrict__ mean,
                       const float *__restrict__ var, float eps, int relu, double *__restrict__ partial)
{
    __shared__ double s_g[BN_TY][BN_TX], s_gx[BN_TY][BN_TX];
    const int tx = threadIdx.x, ty = threadIdx.y;
    const int col = blockIdx.x * BN_TX + tx;
    double sg = 0.0, sgx = 0.0;
    if (col < c) {
        const float sc = scale[col], sh = shift[col];
        const double mu = (double)mean[col], r = 1.0 / sqrt((double)var[col] + (double)eps);
        for (long i = (long)blockIdx.y * BN_TY + ty; i < rows; i += (long)gridDim.y * BN_TY) {
            const float xv = __ldg(x + (size_t)i * ldx + col);
            const double g = (double)relu_masked(__ldg(gout + (size_t)i * ldg + col), xv, sc, sh, relu);
            sg += g; sgx += g * (((double)xv - mu) * r);
        }
    }
    s_g[ty][tx] = sg; s_gx[ty][tx] = sgx;
    __syncthreads();
    if (ty == 0 && col < c) {
#pragma unroll
        for (int i = 1; i < BN_TY; i++) { sg += s_g[i][tx]; sgx += s_gx[i][tx]; }
        partial[((size_t)blockIdx.y * 2 + 0) * c + col] = sg;
        partial[((size_t)blockIdx.y * 2 + 1) * c + col] = sgx;
    }
}

// coef[0..3][c] = (gamma r, sum g / N, sum g x^ / N, r)
__global__ void bn_grad_finalize_kernel(int nrb, long rows, int c, const double *__restrict__ partial, const float *__restrict__ gamma,
                                        const float *__restrict__ var, float eps, double *__restrict__ coef,
                                        float *__restrict__ grad_gamma, float *__restrict__ grad_beta)
{
    const int col = blockIdx.x * blockDim.x + threadIdx.x;
    if (col >= c) return;
    double sg = 0.0, sgx = 0.0;
    for (int rb = 0; rb < nrb; rb++) { sg += partial[((size_t)rb * 2) * c + col]; sgx += partial[((size_t)rb * 2 + 1) * c + col]; }
    const double r = 1.0 / sqrt((double)var[col] + (double)eps);
    coef[col] = (double)gamma[col] * r;
    coef[c + col] = sg / (double)rows;
    coef[2 * c + col] = sgx / (double)rows;
    coef[3 * c + col] = r;
    if (grad_beta) grad_beta[col] = (float)sg;
    if (grad_gamma) grad_gamma[col] = (float)sgx;
}

__global__ void bn_grad_apply_kernel(long rows, int c, const float *__restrict__ x, int ldx, const float *__restrict__ gout, int ldg,
                                     const float *__restrict__ scale, const float *__restrict__ shift, const float *__restrict__ mean,
                                     int relu, const double *__restrict__ coef, float *__restrict__ gx, int ldgx)
{
    const long total = rows * c;
    for (long e = blockIdx.x * (long)blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x) {
        const long i = e / c;
        const int col = (int)(e - i * c);
        const float xv = x[(size_t)i * ldx + col];
        const double g = (double)relu_masked(gout[(size_t)i * ldg + col], xv, scale[col], shift[col], relu);
        const double xh = ((double)xv - (double)mean[col]) * coef[3 * c + col];
        gx[(size_t)i * ldgx + col] = (float)(coef[col] * (g - coef[c + col] - xh * coef[2 * c + col]));
    }
}

}  // namespace ssd3d

using namespace ssd3d;

extern "C" size_t ssd3d_bn_train_workspace(int c) { return c > 0 ? (size_t)BN_MAX_RB * 2 * (size_t)c * sizeof(double) : 0; }

extern "C" size_t ssd3d_bn_train_grad_workspace(int c) { return c > 0 ? (size_t)(BN_MAX_RB * 2 + 4) * (size_t)c * sizeof(double) : 0; }

extern "C" int ssd3d_bn_train_grad(long rows, int c, const float *x, int ldx, const float *grad_out, int ldg, const float *scale,
                                   const float *shift, const float *batch_mean, const float *batch_var, const float *gamma,
                                   float eps, int relu, void *workspace, float *grad_gamma, float *grad_beta, float *grad_x,
                                   int ldgx, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(rows > 0 && c > 0 && ldx >= c && ldg >= c && ldgx >= c,
                  "bn_train_grad: bad shape rows=%ld c=%d ldx=%d ldg=%d ldgx=%d", rows, c, ldx, ldg, ldgx);
    SSD3D_REQUIRE(x && grad_out && scale && shift && batch_mean && batch_var && gamma && workspace && grad_x,
                  "bn_train_grad: null pointer");
    SSD3D_REQUIRE(eps >= 0.0f, "bn_train_grad: eps=%g must be >= 0", eps);
    SSD3D_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 7u) == 0, "bn_train_grad: workspace must be 8-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    long want = (rows + BN_TY * 64 - 1) / (BN_TY * 64);
    const int nrb = (int)(want < 1 ? 1 : (want > BN_MAX_RB ? BN_MAX_RB : want));
    double *partial = (double *)workspace, *coef = partial + (size_t)BN_MAX_RB * 2 * c;
    dim3 grid((unsigned)((c + BN_TX - 1) / BN_TX), (unsigned)nrb), block(BN_TX, BN_TY);
    bn_grad_partial_kernel<<<grid, block, 0, st>>>(rows, c, x, ldx, grad_out, ldg, scale, shift, batch_mean, batch_var, eps, relu,
                                                   partial);
    int rc = cuda_status(cudaGetLastError(), "bn_grad_partial_kernel");
    if (rc) return rc;
    bn_grad_finalize_kernel<<<(c + 127) / 128, 128, 0, st>>>(nrb, rows, c, partial, gamma, batch_var, eps, coef, grad_gamma, grad_beta);
    rc = cuda_status(cudaGetLastError(), "bn_grad_finalize_kernel");
    if (rc) return rc;
    const long total = rows * c;
    const int blocks = (int)((total + 255) / 256 < (long)kNumSMs * 16 ? (total + 255) / 256 : (long)kNumSMs * 16);
    bn_grad_apply_kernel<<<blocks, 256, 0, st>>>(rows, c, x, ldx, grad_out, ldg, scale, shift, batch_mean, relu, coef, grad_x, ldgx);
    SSD3D_LAUNCH_CHECK("bn_grad_apply_kernel");
}

extern "C" int ssd3d_bn_train(long rows, int c, const float *x, int ldx, const float *gamma, const float *beta,
                              float *moving_mean, float *moving_var, float decay, float eps, void *workspace, float *scale,
                              float *shift, float *batch_mean, float *batch_var, int relu, float *out, int ldo,
                              ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(rows > 0 && c > 0 && ldx >= c && ldo >= c, "bn_train: bad shape rows=%ld c=%d ldx=%d ldo=%d", rows, c, ldx, ldo);
    SSD3D_REQUIRE(x && gamma && beta && workspace && scale && shift && out, "bn_train: null pointer");
    SSD3D_REQUIRE((moving_mean == nullptr) == (moving_var == nullptr), "bn_train: moving_mean and moving_var go together");
    SSD3D_REQUIRE(decay >= 0.0f && decay <= 1.0f && eps >= 0.0f, "bn_train: decay=%g must be in [0,1], eps=%g >= 0", decay, eps);
    SSD3D_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 7u) == 0, "bn_train: workspace must be 8-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    long want = (rows + BN_TY * 64 - 1) / (BN_TY * 64);                 // >= 64 rows per thread before another block pays
    const int nrb = (int)(want < 1 ? 1 : (want > BN_MAX_RB ? BN_MAX_RB : want));
    dim3 grid((unsigned)((c + BN_TX - 1) / BN_TX), (unsigned)nrb), block(BN_TX, BN_TY);
    bn_partial_kernel<<<grid, block, 0, st>>>(rows, c, x, ldx, (double *)workspace);
    int rc = cuda_status(cudaGetLastError(), "bn_partial_kernel");
    if (rc) return rc;
    bn_finalize_kernel<<<(c + 127) / 128, 128, 0, st>>>(nrb, rows, c, (const double *)workspace, gamma, beta, moving_mean,
                                                        moving_var, decay, eps, scale, shift, batch_mean, batch_var);
    rc = cuda_status(cudaGetLastError(), "bn_finalize_kernel");
    if (rc) return rc;
    const long total = rows * c;
    const int blocks = (int)((total + 255) / 256 < (long)kNumSMs * 16 ? (total + 255) / 256 : (long)kNumSMs * 16);
    scale_shift_act_kernel<<<blocks, 256, 0, st>>>(rows, c, x, ldx, scale, shift, relu, out, ldo);
    SSD3D_LAUNCH_CHECK("scale_shift_act_kernel");
}
