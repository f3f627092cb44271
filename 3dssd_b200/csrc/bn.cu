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
#include "peer_sync.cuh"

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

// Row-block partials of one channel, folded in block order (the same order with and without SyncBN).
__device__ __forceinline__ void bn_fold_partials(int nrb, int c, const double *__restrict__ partial, int col, double &a, double &b)
{
    a = 0.0; b = 0.0;
    for (int rb = 0; rb < nrb; rb++) { a += partial[((size_t)rb * 2) * c + col]; b += partial[((size_t)rb * 2 + 1) * c + col]; }
}

// The float32 finalize of one channel from its sums over `rows` rows: the one copy of the formula, used by the
// single-GPU finalize and by the synchronised one (so SyncBN over one rank gives the same bits).
__device__ __forceinline__ void bn_finalize_channel(int col, double sum, double sq, double rows, const float *__restrict__ gamma,
                                                    const float *__restrict__ beta, float *__restrict__ moving_mean,
                                                    float *__restrict__ moving_var, float decay, float eps, float *__restrict__ scale,
                                                    float *__restrict__ shift, float *__restrict__ batch_mean, float *__restrict__ batch_var)
{
    const double mean_d = sum / rows;
    double var_d = sq / rows - mean_d * mean_d;
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

__global__ void bn_finalize_kernel(int nrb, long rows, int c, const double *__restrict__ partial, const float *__restrict__ gamma,
                                   const float *__restrict__ beta, float *__restrict__ moving_mean,
                                   float *__restrict__ moving_var, float decay, float eps, float *__restrict__ scale,
                                   float *__restrict__ shift, float *__restrict__ batch_mean, float *__restrict__ batch_var)
{
    const int col = blockIdx.x * blockDim.x + threadIdx.x;
    if (col >= c) return;
    double sum, sq;
    bn_fold_partials(nrb, c, partial, col, sum, sq);
    bn_finalize_channel(col, sum, sq, (double)rows, gamma, beta, moving_mean, moving_var, decay, eps, scale, shift, batch_mean,
                        batch_var);
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

// coef[0..3][c] = (gamma r, sum g / N, sum g x^ / N, r) of one channel from its sums over `rows` rows (shared like
// bn_finalize_channel)
__device__ __forceinline__ void bn_grad_coef_channel(int col, int c, double sg, double sgx, double rows, const float *__restrict__ gamma,
                                                     const float *__restrict__ var, float eps, double *__restrict__ coef)
{
    const double r = 1.0 / sqrt((double)var[col] + (double)eps);
    coef[col] = (double)gamma[col] * r;
    coef[c + col] = sg / rows;
    coef[2 * c + col] = sgx / rows;
    coef[3 * c + col] = r;
}

__global__ void bn_grad_finalize_kernel(int nrb, long rows, int c, const double *__restrict__ partial, const float *__restrict__ gamma,
                                        const float *__restrict__ var, float eps, double *__restrict__ coef,
                                        float *__restrict__ grad_gamma, float *__restrict__ grad_beta)
{
    const int col = blockIdx.x * blockDim.x + threadIdx.x;
    if (col >= c) return;
    double sg, sgx;
    bn_fold_partials(nrb, c, partial, col, sg, sgx);
    bn_grad_coef_channel(col, c, sg, sgx, (double)rows, gamma, var, eps, coef);
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


// ---- SyncBN (DESIGN.md section 3.18): the finalize of a BatchNorm whose batch is sharded over `world` ranks.  One
// exchange-and-finalize launch of ceil(c / 128) CTAs replaces the finalize; CTA j owns channels [128 j, 128 j + 128).
// Per (scope, direction) every rank's symmetric buffer holds an area (ssd3d_bn_sync_area_bytes) of
//     data[par][src][3][c]  doubles: rank src's (rows, sum a, sum b) per channel      flags[par][src][ctas]  int32
// Replay s (counted on the device in state[0]) uses par = s & 1.  CTA j folds its channels' partials, stores the triples
// into every peer's data[par][me], fences, releases every peer's flags[par][me][j] = s, waits until its own
// flags[par][q][j] >= s for every q, then adds the triples in rank order 0..G-1 in double and finalizes.  Reuse: rank A
// writes parity par again in replay s+2 only after its replay s+1 waited for every peer's flag of s+1, which a peer
// publishes only after its launch of replay s -- every read included -- has finished (same stream).  A wait that gives
// up is counted in state[2] and the CTA finalizes from NaN sums, so a broken exchange poisons its channels.
constexpr int BN_SYNC_THREADS = 128;

struct BnSyncParams {
    uint8_t *const *peer_base;   // DEVICE array [world]: every rank's symmetric allocation as mapped here
    size_t area;                 // byte offset of this (scope, direction)'s area inside every rank's allocation
    int *state;                  // [0] replays done, [1] CTAs of the current replay that have finished, [2] time-outs
    int world, rank;
};

struct BnFwdOut {                // the forward finalize's operands (bn_finalize_channel)
    const float *gamma, *beta;
    float *moving_mean, *moving_var;
    float decay, eps;
    float *scale, *shift, *batch_mean, *batch_var;
};

struct BnGradOut {               // the backward finalize's operands (bn_grad_coef_channel); grad_gamma / grad_beta are local
    const float *gamma, *var;
    float eps;
    double *coef;
    float *grad_gamma, *grad_beta;
};

__device__ __forceinline__ void bn_sync_finish(const BnFwdOut &o, int col, int, double n, double a, double b, double, double)
{
    bn_finalize_channel(col, a, b, n, o.gamma, o.beta, o.moving_mean, o.moving_var, o.decay, o.eps, o.scale, o.shift,
                        o.batch_mean, o.batch_var);
}

__device__ __forceinline__ void bn_sync_finish(const BnGradOut &o, int col, int c, double n, double a, double b, double la, double lb)
{
    bn_grad_coef_channel(col, c, a, b, n, o.gamma, o.var, o.eps, o.coef);
    if (o.grad_beta) o.grad_beta[col] = (float)la;
    if (o.grad_gamma) o.grad_gamma[col] = (float)lb;
}

__host__ __device__ __forceinline__ size_t bn_sync_data_bytes(int world, int c) { return ((size_t)world * 3 * c * sizeof(double) + 15) / 16 * 16; }
__host__ __device__ __forceinline__ size_t bn_sync_flag_bytes(int world, int c)
{
    return ((size_t)world * ((c + BN_SYNC_THREADS - 1) / BN_SYNC_THREADS) * sizeof(int) + 15) / 16 * 16;
}

template <class Out>
__global__ void __launch_bounds__(BN_SYNC_THREADS)
bn_sync_finalize_kernel(int nrb, long rows, int c, const double *__restrict__ partial, const BnSyncParams p, const Out o)
{
    const int j = blockIdx.x, tid = threadIdx.x, col = j * BN_SYNC_THREADS + tid, G = p.world, me = p.rank;
    __shared__ int s_seq, s_ok;
    if (tid == 0) { s_seq = *reinterpret_cast<volatile int *>(p.state) + 1; s_ok = 1; }   // state[0] changes only after every CTA read it
    __syncthreads();
    const int seq = s_seq, par = seq & 1;
    const size_t dbytes = bn_sync_data_bytes(G, c), fbytes = bn_sync_flag_bytes(G, c);
    const size_t data_off = p.area + par * dbytes, flag_off = p.area + 2 * dbytes + par * fbytes;
    double a = 0.0, b = 0.0;
    if (col < c) bn_fold_partials(nrb, c, partial, col, a, b);
    const double n_me = (double)rows;
#pragma unroll 1
    for (int k = 0; k < G; k++) {
        const int q = (me + 1 + k) % G;                      // spread the first stores over the links
        double *dst = reinterpret_cast<double *>(p.peer_base[q] + data_off) + (size_t)me * 3 * c;
        if (col < c) { dst[col] = n_me; dst[c + col] = a; dst[2 * c + col] = b; }
    }
    __threadfence_system();
    __syncthreads();
    if (tid == 0) {
        for (int q = 0; q < G; q++) st_release_sys(reinterpret_cast<int *>(p.peer_base[q] + flag_off) + (size_t)me * gridDim.x + j, seq);
        uint8_t *mine = p.peer_base[me];
        for (int q = 0; q < G; q++) {
            const int *flag = reinterpret_cast<const int *>(mine + flag_off) + (size_t)q * gridDim.x + j;
            const long long t0 = clock64();
            while (ld_acquire_sys(flag) < seq) {
                if (clock64() - t0 > kPeerSpinLimit) { atomicAdd(p.state + 2, 1); s_ok = 0; break; }   // counted, not hung
            }
        }
    }
    __syncthreads();
    if (col < c) {
        const double *src = reinterpret_cast<const double *>(p.peer_base[me] + data_off);
        double n, sa, sb;
        if (s_ok) {
            n = __ldcg(src + col); sa = __ldcg(src + c + col); sb = __ldcg(src + 2 * c + col);   // rank 0 first, no +0.0
#pragma unroll 1
            for (int q = 1; q < G; q++) {
                const double *t = src + (size_t)q * 3 * c;
                n += __ldcg(t + col); sa += __ldcg(t + c + col); sb += __ldcg(t + 2 * c + col);
            }
        } else {
            n = sa = sb = __longlong_as_double(0x7ff8000000000000LL);
        }
        bn_sync_finish(o, col, c, n, sa, sb, a, b);
    }
    __syncthreads();
    if (tid == 0) {
        __threadfence();
        if (atomicAdd(p.state + 1, 1) == (int)gridDim.x - 1) {   // last CTA of this replay: publish the new count
            p.state[1] = 0;
            __threadfence();
            *reinterpret_cast<volatile int *>(p.state) = seq;
        }
    }
}

}  // namespace ssd3d

using namespace ssd3d;

extern "C" size_t ssd3d_bn_train_workspace(int c) { return c > 0 ? (size_t)BN_MAX_RB * 2 * (size_t)c * sizeof(double) : 0; }

extern "C" size_t ssd3d_bn_train_grad_workspace(int c) { return c > 0 ? (size_t)(BN_MAX_RB * 2 + 4) * (size_t)c * sizeof(double) : 0; }

static int bn_sync_check(void *const *peer_base, int world, int rank, size_t area_off, const int *state, const char *what)
{
    SSD3D_REQUIRE(world >= 1 && world <= 64 && rank >= 0 && rank < world, "%s: bad world=%d rank=%d", what, world, rank);
    SSD3D_REQUIRE(peer_base && state, "%s: null pointer", what);
    SSD3D_REQUIRE(area_off % 16 == 0, "%s: area offset %zu must be a 16-byte multiple", what, area_off);
    return 0;
}

static int bn_nrb(long rows)
{
    const long want = (rows + BN_TY * 64 - 1) / (BN_TY * 64);          // >= 64 rows per thread before another block pays
    return (int)(want < 1 ? 1 : (want > BN_MAX_RB ? BN_MAX_RB : want));
}

static int bn_apply_blocks(long rows, int c)
{
    const long total = rows * c;
    return (int)((total + 255) / 256 < (long)kNumSMs * 16 ? (total + 255) / 256 : (long)kNumSMs * 16);
}

// partial -> finalize (sync == nullptr) or exchange-and-finalize -> apply
static int bn_train_grad_launch(long rows, int c, const float *x, int ldx, const float *grad_out, int ldg, const float *scale,
                                const float *shift, const float *batch_mean, const float *batch_var, const float *gamma, float eps,
                                int relu, void *workspace, float *grad_gamma, float *grad_beta, float *grad_x, int ldgx,
                                const BnSyncParams *sync, cudaStream_t st)
{
    SSD3D_REQUIRE(rows > 0 && c > 0 && ldx >= c && ldg >= c && ldgx >= c,
                  "bn_train_grad: bad shape rows=%ld c=%d ldx=%d ldg=%d ldgx=%d", rows, c, ldx, ldg, ldgx);
    SSD3D_REQUIRE(x && grad_out && scale && shift && batch_mean && batch_var && gamma && workspace && grad_x,
                  "bn_train_grad: null pointer");
    SSD3D_REQUIRE(eps >= 0.0f, "bn_train_grad: eps=%g must be >= 0", eps);
    SSD3D_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 7u) == 0, "bn_train_grad: workspace must be 8-byte aligned");
    const int nrb = bn_nrb(rows);
    double *partial = (double *)workspace, *coef = partial + (size_t)BN_MAX_RB * 2 * c;
    dim3 grid((unsigned)((c + BN_TX - 1) / BN_TX), (unsigned)nrb), block(BN_TX, BN_TY);
    bn_grad_partial_kernel<<<grid, block, 0, st>>>(rows, c, x, ldx, grad_out, ldg, scale, shift, batch_mean, batch_var, eps, relu,
                                                   partial);
    int rc = cuda_status(cudaGetLastError(), "bn_grad_partial_kernel");
    if (rc) return rc;
    if (sync) {
        const BnGradOut o = {gamma, batch_var, eps, coef, grad_gamma, grad_beta};
        bn_sync_finalize_kernel<BnGradOut><<<(c + BN_SYNC_THREADS - 1) / BN_SYNC_THREADS, BN_SYNC_THREADS, 0, st>>>(nrb, rows, c, partial,
                                                                                                                 *sync, o);
        rc = cuda_status(cudaGetLastError(), "bn_sync_finalize_kernel<grad>");
    } else {
        bn_grad_finalize_kernel<<<(c + 127) / 128, 128, 0, st>>>(nrb, rows, c, partial, gamma, batch_var, eps, coef, grad_gamma, grad_beta);
        rc = cuda_status(cudaGetLastError(), "bn_grad_finalize_kernel");
    }
    if (rc) return rc;
    bn_grad_apply_kernel<<<bn_apply_blocks(rows, c), 256, 0, st>>>(rows, c, x, ldx, grad_out, ldg, scale, shift, batch_mean, relu, coef,
                                                                    grad_x, ldgx);
    SSD3D_LAUNCH_CHECK("bn_grad_apply_kernel");
}

static int bn_train_launch(long rows, int c, const float *x, int ldx, const float *gamma, const float *beta, float *moving_mean,
                           float *moving_var, float decay, float eps, void *workspace, float *scale, float *shift, float *batch_mean,
                           float *batch_var, int relu, float *out, int ldo, const BnSyncParams *sync, cudaStream_t st)
{
    SSD3D_REQUIRE(rows > 0 && c > 0 && ldx >= c && ldo >= c, "bn_train: bad shape rows=%ld c=%d ldx=%d ldo=%d", rows, c, ldx, ldo);
    SSD3D_REQUIRE(x && gamma && beta && workspace && scale && shift && out, "bn_train: null pointer");
    SSD3D_REQUIRE((moving_mean == nullptr) == (moving_var == nullptr), "bn_train: moving_mean and moving_var go together");
    SSD3D_REQUIRE(decay >= 0.0f && decay <= 1.0f && eps >= 0.0f, "bn_train: decay=%g must be in [0,1], eps=%g >= 0", decay, eps);
    SSD3D_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 7u) == 0, "bn_train: workspace must be 8-byte aligned");
    const int nrb = bn_nrb(rows);
    dim3 grid((unsigned)((c + BN_TX - 1) / BN_TX), (unsigned)nrb), block(BN_TX, BN_TY);
    bn_partial_kernel<<<grid, block, 0, st>>>(rows, c, x, ldx, (double *)workspace);
    int rc = cuda_status(cudaGetLastError(), "bn_partial_kernel");
    if (rc) return rc;
    if (sync) {
        const BnFwdOut o = {gamma, beta, moving_mean, moving_var, decay, eps, scale, shift, batch_mean, batch_var};
        bn_sync_finalize_kernel<BnFwdOut><<<(c + BN_SYNC_THREADS - 1) / BN_SYNC_THREADS, BN_SYNC_THREADS, 0, st>>>(
            nrb, rows, c, (const double *)workspace, *sync, o);
        rc = cuda_status(cudaGetLastError(), "bn_sync_finalize_kernel<fwd>");
    } else {
        bn_finalize_kernel<<<(c + 127) / 128, 128, 0, st>>>(nrb, rows, c, (const double *)workspace, gamma, beta, moving_mean,
                                                            moving_var, decay, eps, scale, shift, batch_mean, batch_var);
        rc = cuda_status(cudaGetLastError(), "bn_finalize_kernel");
    }
    if (rc) return rc;
    scale_shift_act_kernel<<<bn_apply_blocks(rows, c), 256, 0, st>>>(rows, c, x, ldx, scale, shift, relu, out, ldo);
    SSD3D_LAUNCH_CHECK("scale_shift_act_kernel");
}

extern "C" int ssd3d_bn_train_grad(long rows, int c, const float *x, int ldx, const float *grad_out, int ldg, const float *scale,
                                   const float *shift, const float *batch_mean, const float *batch_var, const float *gamma,
                                   float eps, int relu, void *workspace, float *grad_gamma, float *grad_beta, float *grad_x,
                                   int ldgx, ssd3d_stream_t stream)
{
    return bn_train_grad_launch(rows, c, x, ldx, grad_out, ldg, scale, shift, batch_mean, batch_var, gamma, eps, relu, workspace,
                                grad_gamma, grad_beta, grad_x, ldgx, nullptr, (cudaStream_t)stream);
}

extern "C" int ssd3d_bn_train(long rows, int c, const float *x, int ldx, const float *gamma, const float *beta,
                              float *moving_mean, float *moving_var, float decay, float eps, void *workspace, float *scale,
                              float *shift, float *batch_mean, float *batch_var, int relu, float *out, int ldo,
                              ssd3d_stream_t stream)
{
    return bn_train_launch(rows, c, x, ldx, gamma, beta, moving_mean, moving_var, decay, eps, workspace, scale, shift, batch_mean,
                           batch_var, relu, out, ldo, nullptr, (cudaStream_t)stream);
}

extern "C" size_t ssd3d_bn_sync_area_bytes(int world, int c)
{
    return (world >= 1 && c > 0) ? 2 * bn_sync_data_bytes(world, c) + 2 * bn_sync_flag_bytes(world, c) : 0;
}

extern "C" int ssd3d_bn_sync_resident_ctas(void)
{
    int dev = 0, sms = 0, fwd = 0, grad = 0;
    int rc = cuda_status(cudaGetDevice(&dev), "bn_sync_resident_ctas");
    if (rc) return rc;
    rc = cuda_status(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev), "bn_sync_resident_ctas");
    if (rc) return rc;
    rc = cuda_status(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&fwd, bn_sync_finalize_kernel<BnFwdOut>, BN_SYNC_THREADS, 0),
                     "bn_sync_resident_ctas");
    if (rc) return rc;
    rc = cuda_status(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&grad, bn_sync_finalize_kernel<BnGradOut>, BN_SYNC_THREADS, 0),
                     "bn_sync_resident_ctas");
    if (rc) return rc;
    return sms * (fwd < grad ? fwd : grad);
}

extern "C" int ssd3d_bn_train_sync(long rows, int c, const float *x, int ldx, const float *gamma, const float *beta,
                                   float *moving_mean, float *moving_var, float decay, float eps, void *workspace, float *scale,
                                   float *shift, float *batch_mean, float *batch_var, int relu, float *out, int ldo,
                                   void *const *peer_base, int world, int rank, size_t area_off, int *state, ssd3d_stream_t stream)
{
    const int rc = bn_sync_check(peer_base, world, rank, area_off, state, "bn_train_sync");
    if (rc) return rc;
    const BnSyncParams p = {(uint8_t *const *)peer_base, area_off, state, world, rank};
    return bn_train_launch(rows, c, x, ldx, gamma, beta, moving_mean, moving_var, decay, eps, workspace, scale, shift, batch_mean,
                           batch_var, relu, out, ldo, &p, (cudaStream_t)stream);
}

extern "C" int ssd3d_bn_train_grad_sync(long rows, int c, const float *x, int ldx, const float *grad_out, int ldg, const float *scale,
                                        const float *shift, const float *batch_mean, const float *batch_var, const float *gamma,
                                        float eps, int relu, void *workspace, float *grad_gamma, float *grad_beta, float *grad_x,
                                        int ldgx, void *const *peer_base, int world, int rank, size_t area_off, int *state,
                                        ssd3d_stream_t stream)
{
    const int rc = bn_sync_check(peer_base, world, rank, area_off, state, "bn_train_grad_sync");
    if (rc) return rc;
    const BnSyncParams p = {(uint8_t *const *)peer_base, area_off, state, world, rank};
    return bn_train_grad_launch(rows, c, x, ldx, grad_out, ldg, scale, shift, batch_mean, batch_var, gamma, eps, relu, workspace,
                                grad_gamma, grad_beta, grad_x, ldgx, &p, (cudaStream_t)stream);
}
