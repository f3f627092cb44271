// solver.cu -- the optimizer step of training (DESIGN.md section 3.11).
//
// The reference trains with tf.train.AdamOptimizer(learning_rate) (lib/core/trainer.py:74-75, :87) and drives the
// learning rate from global_step with tf.train.piecewise_constant (lib/core/trainer_utils.py:7-13).  Two kernels restate
// the update with every float32 operation rounded once, and rebuild what the next forward reads from the weights:
//
//   adam_step         ONE launch over the flat parameter buffer.  The state block (global_step, beta1_power, beta2_power,
//                     lr_used) lives on the device and belongs to the caller.  Per launch, with the OLD state:
//                       lr    = values[number of boundaries < global_step]            (piecewise_constant)
//                       alpha = rn(rn(lr * rn(sqrt(rn(1 - beta2_power)))) / rn(1 - beta1_power))
//                       m'    = rn(m + rn(rn(g - m) * rn(1 - beta1)))
//                       v'    = rn(v + rn(rn(rn(g * g) - v) * rn(1 - beta2)))
//                       p'    = rn(p - rn(rn(m' * alpha) / rn(rn(sqrt(v')) + epsilon)))     (epsilon outside the bias
//                                                                                            correction: TF's ApplyAdam)
//                     then beta1_power = rn(beta1_power * beta1), likewise beta2, global_step += 1, lr_used = lr.
//                     Every block reads the state before it touches an element and counts itself done afterwards; the
//                     block that counts last is the only writer of the new state, so no block can see it half updated.
//                     The library is built with -fmad=true: the arithmetic is spelled with __f*_rn so that contraction
//                     cannot change a bit.  Non-finite gradients propagate into m, v and p.
//   momentum_step     ONE launch of tf.train.MomentumOptimizer(lr, momentum) (use_nesterov=False, TF's ApplyMomentum) over
//                     the same flat buffer, with the same schedule and the same state block and "last block publishes"
//                     protocol; beta1_power and beta2_power are left as they are.  Per element, with the OLD state's lr:
//                       accum' = rn(rn(accum * momentum) + g)
//                       p'     = rn(p - rn(accum' * lr))
//                     TF states this as an Eigen expression (accum * momentum + grad; var -= accum * lr) and it is not
//                     known whether the reference's GPU build contracted either line into an fma.  The uncontracted form
//                     is the one chosen here: every product and sum rounded once, spelled with __f*_rn.  Non-finite
//                     gradients propagate into accum and p.
//   weight_operands   ONE launch that rebuilds the split-bf16 tensor-core operands (operand.cuh) of every conv weight
//                     from the flat parameter buffer: for W [cin, cout] the forward operand = split of W^T
//                     [cout, round16(cin)] and the grad-x operand = split of W [cin, round16(cout)], zero padded.  A
//                     32 x 32 tile goes through shared memory so the read of W and both writes are coalesced.
#include "common.cuh"
#include "operand.cuh"

namespace ssd3d {

constexpr int ADAM_THREADS = 256;
constexpr int ADAM_MAX_BOUNDARIES = 8;                 // ssd3d.h
constexpr int WOP_TILE = 32, WOP_ROWS = 8;             // a 32 x 32 tile of W per block of 32 x 8 threads
constexpr int WOP_COLS = 8;                            // int64 columns of a descriptor row (ssd3d.h)

struct AdamState {                                      // the caller's 32-byte device block (ssd3d.h)
    long long global_step;
    float beta1_power, beta2_power, lr_used;
    unsigned int done;                                  // blocks of the running launch that have finished; 0 between launches
    unsigned int reserved[2];
};
static_assert(sizeof(AdamState) == 32, "ssd3d.h documents a 32-byte state block");

struct AdamSchedule {
    long long boundaries[ADAM_MAX_BOUNDARIES];
    float values[ADAM_MAX_BOUNDARIES + 1];
    int nb;
};

struct AdamCoef {
    float alpha, omb1, omb2, eps;
};

// Thread 0 of every block: the old state and the learning rate it selects (piecewise_constant; boundaries increase, so the
// last boundary below global_step wins).  Nothing is written: the state changes only after every block counted itself done.
__device__ __forceinline__ float read_state(const AdamState *state, const AdamSchedule &sch, long long &step, float &b1p, float &b2p)
{
    const volatile AdamState *st = state;
    step = st->global_step;
    float lr = sch.values[0];
#pragma unroll                                          // constant indices: the schedule stays in the parameter bank
    for (int k = 0; k < ADAM_MAX_BOUNDARIES; k++)
        if (k < sch.nb && step > sch.boundaries[k]) lr = sch.values[k + 1];
    b1p = st->beta1_power; b2p = st->beta2_power;
    return lr;
}

// Thread 0 of every block, after the block's last element: the block that counts last writes the new state.
__device__ __forceinline__ bool last_block_done(AdamState *state)
{
    __threadfence();
    if (atomicAdd(&state->done, 1u) != gridDim.x - 1) return false;
    state->done = 0;
    return true;
}

__device__ __forceinline__ void adam_one(float &p, float g, float &m, float &v, const AdamCoef c)
{
    m = __fadd_rn(m, __fmul_rn(__fsub_rn(g, m), c.omb1));
    v = __fadd_rn(v, __fmul_rn(__fsub_rn(__fmul_rn(g, g), v), c.omb2));
    p = __fsub_rn(p, __fdiv_rn(__fmul_rn(m, c.alpha), __fadd_rn(__fsqrt_rn(v), c.eps)));
}

__global__ void __launch_bounds__(ADAM_THREADS)
adam_step_kernel(float *__restrict__ param, const float *__restrict__ grad, float *__restrict__ m, float *__restrict__ v, long n,
                 AdamState *state, float beta1, float beta2, float omb1, float omb2, float eps, const AdamSchedule sch)
{
    __shared__ long long s_step;
    __shared__ float s_b1p, s_b2p, s_lr;
    const int tid = threadIdx.x;
    if (tid == 0) s_lr = read_state(state, sch, s_step, s_b1p, s_b2p);
    __syncthreads();
    const float lr = s_lr, b1p = s_b1p, b2p = s_b2p;
    AdamCoef c;
    c.alpha = __fdiv_rn(__fmul_rn(lr, __fsqrt_rn(__fsub_rn(1.0f, b2p))), __fsub_rn(1.0f, b1p));
    c.omb1 = omb1; c.omb2 = omb2; c.eps = eps;

    const long n4 = n / 4, stride = (long)gridDim.x * ADAM_THREADS;
    float4 *p4 = reinterpret_cast<float4 *>(param), *m4 = reinterpret_cast<float4 *>(m), *v4 = reinterpret_cast<float4 *>(v);
    const float4 *g4 = reinterpret_cast<const float4 *>(grad);
    for (long i = (long)blockIdx.x * ADAM_THREADS + tid; i < n4; i += stride) {
        float4 p = p4[i], mm = m4[i], vv = v4[i];
        const float4 g = __ldg(g4 + i);
        adam_one(p.x, g.x, mm.x, vv.x, c); adam_one(p.y, g.y, mm.y, vv.y, c);
        adam_one(p.z, g.z, mm.z, vv.z, c); adam_one(p.w, g.w, mm.w, vv.w, c);
        p4[i] = p; m4[i] = mm; v4[i] = vv;
    }
    if (blockIdx.x == 0 && 4 * n4 + tid < n) {          // the tail of an n that is not a multiple of 4
        const long i = 4 * n4 + tid;
        float p = param[i], mm = m[i], vv = v[i];
        adam_one(p, __ldg(grad + i), mm, vv, c);
        param[i] = p; m[i] = mm; v[i] = vv;
    }
    __syncthreads();
    if (tid == 0) {
        if (last_block_done(state)) {                   // every block has read the old state: publish the new one
            state->beta1_power = __fmul_rn(b1p, beta1);
            state->beta2_power = __fmul_rn(b2p, beta2);
            state->lr_used = lr;
            state->global_step = s_step + 1;
        }
    }
}

__device__ __forceinline__ void momentum_one(float &p, float g, float &a, float mom, float lr)
{
    a = __fadd_rn(__fmul_rn(a, mom), g);
    p = __fsub_rn(p, __fmul_rn(a, lr));
}

__global__ void __launch_bounds__(ADAM_THREADS)
momentum_step_kernel(float *__restrict__ param, const float *__restrict__ grad, float *__restrict__ accum, long n, AdamState *state,
                     float momentum, const AdamSchedule sch)
{
    __shared__ long long s_step;
    __shared__ float s_b1p, s_b2p, s_lr;
    const int tid = threadIdx.x;
    if (tid == 0) s_lr = read_state(state, sch, s_step, s_b1p, s_b2p);
    __syncthreads();
    const float lr = s_lr;

    const long n4 = n / 4, stride = (long)gridDim.x * ADAM_THREADS;
    float4 *p4 = reinterpret_cast<float4 *>(param), *a4 = reinterpret_cast<float4 *>(accum);
    const float4 *g4 = reinterpret_cast<const float4 *>(grad);
    for (long i = (long)blockIdx.x * ADAM_THREADS + tid; i < n4; i += stride) {
        float4 p = p4[i], a = a4[i];
        const float4 g = __ldg(g4 + i);
        momentum_one(p.x, g.x, a.x, momentum, lr); momentum_one(p.y, g.y, a.y, momentum, lr);
        momentum_one(p.z, g.z, a.z, momentum, lr); momentum_one(p.w, g.w, a.w, momentum, lr);
        p4[i] = p; a4[i] = a;
    }
    if (blockIdx.x == 0 && 4 * n4 + tid < n) {          // the tail of an n that is not a multiple of 4
        const long i = 4 * n4 + tid;
        float p = param[i], a = accum[i];
        momentum_one(p, __ldg(grad + i), a, momentum, lr);
        param[i] = p; accum[i] = a;
    }
    __syncthreads();
    if (tid == 0 && last_block_done(state)) {           // the beta powers are Adam's: left as they are
        state->lr_used = lr;
        state->global_step = s_step + 1;
    }
}

// Block b works on tile (b - tile_start) of the weight whose descriptor row has the largest tile_start <= b.
__global__ void __launch_bounds__(WOP_TILE *WOP_ROWS)
weight_operands_kernel(const float *__restrict__ param, const long long *__restrict__ table, int nw, __nv_bfloat16 *__restrict__ arena)
{
    __shared__ float tile[WOP_TILE][WOP_TILE + 1];
    const long long blk = blockIdx.x;
    int lo = 0, hi = nw - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(table + (size_t)mid * WOP_COLS + 7) <= blk) lo = mid; else hi = mid - 1;
    }
    const long long *row = table + (size_t)lo * WOP_COLS;
    const float *w = param + __ldg(row + 0);
    const int cin = (int)__ldg(row + 1), cout = (int)__ldg(row + 2);
    __nv_bfloat16 *f_hi = arena + __ldg(row + 3), *f_lo = arena + __ldg(row + 4);
    __nv_bfloat16 *b_hi = arena + __ldg(row + 5), *b_lo = arena + __ldg(row + 6);
    const int kp_in = (cin + 15) / 16 * 16, kp_out = (cout + 15) / 16 * 16;
    const int tiles_j = (kp_out + WOP_TILE - 1) / WOP_TILE;
    const int t = (int)(blk - __ldg(row + 7));
    const int i0 = t / tiles_j * WOP_TILE, j0 = t % tiles_j * WOP_TILE;
    const int tx = threadIdx.x, ty = threadIdx.y;

    for (int r = ty; r < WOP_TILE; r += WOP_ROWS) {     // W rows i0.., columns j0..: the grad-x operand, row-major like W
        const int i = i0 + r, j = j0 + tx;
        const float x = (i < cin && j < cout) ? w[(size_t)i * cout + j] : 0.0f;
        tile[r][tx] = x;
        if (i < cin && j < kp_out) split_store(x, b_hi + (size_t)i * kp_out + j, b_lo + (size_t)i * kp_out + j);
    }
    __syncthreads();
    for (int r = ty; r < WOP_TILE; r += WOP_ROWS) {     // the forward operand: W^T, K-major
        const int j = j0 + r, i = i0 + tx;
        if (j < cout && i < kp_in) split_store(tile[tx][r], f_hi + (size_t)j * kp_in + i, f_lo + (size_t)j * kp_in + i);
    }
}

}  // namespace ssd3d

using namespace ssd3d;

// The schedule of both solver entries, checked and packed into the launch's parameters; 0 or the error's return code.
static int pack_schedule(const char *what, int nb, const long long *boundaries, const float *values, AdamSchedule &sch)
{
    SSD3D_REQUIRE(values && nb >= 0 && nb <= ADAM_MAX_BOUNDARIES && (nb == 0 || boundaries), "%s: nb=%d must be in [0, %d]",
                  what, nb, ADAM_MAX_BOUNDARIES);
    sch = AdamSchedule{};
    sch.nb = nb;
    for (int i = 0; i < nb; i++) {
        SSD3D_REQUIRE(i == 0 || boundaries[i] > boundaries[i - 1], "%s: boundaries must increase", what);
        sch.boundaries[i] = boundaries[i];
    }
    for (int i = 0; i <= nb; i++) sch.values[i] = values[i];
    return 0;
}

static int solver_blocks(long n)
{
    const long want = (n / 4 + ADAM_THREADS - 1) / ADAM_THREADS;
    return (int)(want < 1 ? 1 : (want < (long)kNumSMs * 8 ? want : (long)kNumSMs * 8));
}

extern "C" int ssd3d_adam_step(float *param, const float *grad, float *m, float *v, long n, void *state, float beta1,
                               float beta2, float epsilon, int nb, const long long *boundaries, const float *values,
                               ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(n > 0, "adam_step: n=%ld must be > 0", n);
    SSD3D_REQUIRE(param && grad && m && v && state && values, "adam_step: null pointer");
    SSD3D_REQUIRE(((reinterpret_cast<uintptr_t>(param) | reinterpret_cast<uintptr_t>(grad) | reinterpret_cast<uintptr_t>(m) |
                    reinterpret_cast<uintptr_t>(v)) & 15u) == 0, "adam_step: param, grad, m and v must be 16-byte aligned");
    SSD3D_REQUIRE((reinterpret_cast<uintptr_t>(state) & 7u) == 0, "adam_step: state must be 8-byte aligned");
    SSD3D_REQUIRE(beta1 >= 0.0f && beta1 < 1.0f && beta2 >= 0.0f && beta2 < 1.0f && epsilon >= 0.0f,
                  "adam_step: beta1=%g, beta2=%g must be in [0, 1) and epsilon=%g >= 0", beta1, beta2, epsilon);
    AdamSchedule sch;
    if (const int rc = pack_schedule("adam_step", nb, boundaries, values, sch)) return rc;
    const int blocks = solver_blocks(n);
    const float omb1 = 1.0f - beta1, omb2 = 1.0f - beta2;    // float32 differences, rounded once
    adam_step_kernel<<<blocks, ADAM_THREADS, 0, (cudaStream_t)stream>>>(param, grad, m, v, n, (AdamState *)state, beta1, beta2,
                                                                        omb1, omb2, epsilon, sch);
    SSD3D_LAUNCH_CHECK("adam_step_kernel");
}

extern "C" int ssd3d_momentum_step(float *param, const float *grad, float *accum, long n, void *state, float momentum, int nb,
                                   const long long *boundaries, const float *values, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(n > 0, "momentum_step: n=%ld must be > 0", n);
    SSD3D_REQUIRE(param && grad && accum && state, "momentum_step: null pointer");
    SSD3D_REQUIRE(((reinterpret_cast<uintptr_t>(param) | reinterpret_cast<uintptr_t>(grad) | reinterpret_cast<uintptr_t>(accum)) &
                   15u) == 0, "momentum_step: param, grad and accum must be 16-byte aligned");
    SSD3D_REQUIRE((reinterpret_cast<uintptr_t>(state) & 7u) == 0, "momentum_step: state must be 8-byte aligned");
    SSD3D_REQUIRE(momentum >= 0.0f && momentum <= 1.0f, "momentum_step: momentum=%g must be in [0, 1]", momentum);
    AdamSchedule sch;
    if (const int rc = pack_schedule("momentum_step", nb, boundaries, values, sch)) return rc;
    momentum_step_kernel<<<solver_blocks(n), ADAM_THREADS, 0, (cudaStream_t)stream>>>(param, grad, accum, n, (AdamState *)state,
                                                                                      momentum, sch);
    SSD3D_LAUNCH_CHECK("momentum_step_kernel");
}

extern "C" int ssd3d_weight_operands(const float *param, const long long *table, int nw, long tiles, void *arena,
                                     ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(nw > 0 && tiles >= nw && tiles < (1L << 31), "weight_operands: nw=%d weights in %ld tiles", nw, tiles);
    SSD3D_REQUIRE(param && table && arena, "weight_operands: null pointer");
    SSD3D_REQUIRE((reinterpret_cast<uintptr_t>(arena) & 15u) == 0 && (reinterpret_cast<uintptr_t>(table) & 7u) == 0,
                  "weight_operands: arena must be 16-byte and table 8-byte aligned");
    weight_operands_kernel<<<(unsigned)tiles, dim3(WOP_TILE, WOP_ROWS), 0, (cudaStream_t)stream>>>(
        param, table, nw, reinterpret_cast<__nv_bfloat16 *>(arena));
    SSD3D_LAUNCH_CHECK("weight_operands_kernel");
}
