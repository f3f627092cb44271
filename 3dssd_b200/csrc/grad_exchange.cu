// grad_exchange.cu -- the per-step gradient exchange of data-parallel training (DESIGN.md section 3.9).
//
// The reference trains on towers (lib/core/trainer.py:143-154, lib/utils/trainer_utils.py:23-46): every tower clips its
// own gradients to global norm 5 (tf.clip_by_global_norm), the clipped gradients are averaged over the towers, and every
// tower's forward applies its own batch statistics to the shared BatchNorm moving averages (tf_util.py:438-443,
// updates_collections=None).  Three kernels restate that with pinned arithmetic, so every rank holds the same bits:
//
//   grad_clip_scale       n_r = float32(sqrt(sum g^2 in double)) over a fixed reduction tree, and TF 1.4's float32 scale
//                         scale_r = rn(clip * minimum(rn(1 / use_norm), rn(1 / clip))), use_norm = n_r if finite else NaN
//                         (minimum propagates the NaN: a non-finite norm poisons that rank's clipped gradient, as in TF).
//   peer_allreduce_mean   m[i] = float32((sum over r = 0..G-1 in rank order of (double) rn(g_r[i] * scale_r)) / G),
//                         written back into every rank's flat gradient buffer.
//   bn_moving_update_ranks  for r = 0..G-1: v = rn(v - rn(rn(v - b_r) * rn(1 - decay))), bn.cu's own update, per rank in
//                         rank order (the towers' unlocked assign_subs of the reference have no fixed order).
//
// peer_allreduce_mean is a reduce-scatter plus all-gather over NVLink peer memory in ONE launch (the protocol of
// peer_gather.cu, widened to three phases).  The flat buffer of n floats is cut into `world` chunks of `chunk` floats
// (a multiple of 4: 16-byte boundaries; indices >= n are zero padding), rank p owns chunk p, and each chunk into `ctas`
// sub-slices of `sub` floats.  CTA j of every rank handles sub-slice j of every chunk in all three phases, so CTA j of
// rank A depends only on CTA j of the other ranks and every flag is per (source rank, sub-slice).  Replay s (counted on
// the device in state[0]) uses parity par = s & 1.  In every rank's symmetric buffer, per parity:
//     R1[par][q][chunk]   rank q's clipped sub-slices of MY chunk        F1[par][q][ctas]  (int32)
//     R2[par][q][chunk]   rank q's reduced chunk q                        F2[par][q][ctas]
//   phase 1  for every peer p: rn(g * scale_me) of sub-slice j of chunk p -> peer p's R1[par][me][j];
//            __threadfence_system(); st.release.sys peer p's F1[par][me][j] = s
//   phase 2  wait until my F1[par][q][j] >= s for every q; reduce sub-slice j of my chunk over q in rank order (double,
//            one division, one rounding); store it into every peer's R2[par][me][j]; fence; release peer's F2[par][me][j]
//   phase 3  wait until my F2[par][q][j] >= s for every q; copy R2[par][q][j] (L1 bypassed) into my gradient buffer
//   the last CTA to finish publishes state[0] = s.
// Reuse: rank A writes parity par again only in replay s+2.  Before that it has finished replay s+1, whose phase 2 waited
// for every peer's F1 of replay s+1 (CTA j waits for every peer's CTA j); a peer publishes its F1 of s+1 only inside its
// launch of replay s+1, which starts after its launch of replay s -- every read of R1[par] and R2[par] included -- has
// finished (same stream).  So neither R1[par] nor R2[par] is overwritten before its reader is done, without any
// acknowledgement.  Every rank must make the same sequence of calls.  CTA j spins on other ranks' CTA j, so all `ctas`
// CTAs of a launch must be co-resident on their device (ssd3d_peer_allreduce_resident_ctas); a wait of ~4 s gives up,
// counts itself in state[2] instead of hanging the GPU, and that CTA writes NaN into its part of the gradient.
#include "common.cuh"
#include "peer_sync.cuh"

namespace ssd3d {

constexpr int CLIP_BLOCKS = 256, CLIP_THREADS = 256;   // the fixed reduction tree of the norm (ssd3d.h)
constexpr int AR_THREADS = 256;
static_assert(CLIP_BLOCKS == CLIP_THREADS, "the finalize reads one partial per thread");

// s[0..CLIP_THREADS) -> s[0], halving strides: the same tree in every block and in the finalize
__device__ __forceinline__ double tree_sum(double *s, int tid)
{
    __syncthreads();
#pragma unroll
    for (int w = CLIP_THREADS / 2; w > 0; w >>= 1) {
        if (tid < w) s[tid] += s[tid + w];
        __syncthreads();
    }
    return s[0];
}

// thread t of block b sums g[i]^2 (exact in double) for i = b*256 + t, + 65536, ... in index order; then the block tree
__global__ void __launch_bounds__(CLIP_THREADS)
grad_sumsq_partial_kernel(const float *__restrict__ g, long n, double *__restrict__ partial)
{
    __shared__ double s[CLIP_THREADS];
    const int tid = threadIdx.x;
    double acc = 0.0;
    for (long i = (long)blockIdx.x * CLIP_THREADS + tid; i < n; i += (long)CLIP_BLOCKS * CLIP_THREADS) {
        const double v = (double)__ldg(g + i);
        acc += v * v;
    }
    s[tid] = acc;
    const double tot = tree_sum(s, tid);
    if (tid == 0) partial[blockIdx.x] = tot;
}

__global__ void __launch_bounds__(CLIP_THREADS)
grad_clip_finalize_kernel(const double *__restrict__ partial, float clip, float *__restrict__ norm, float *__restrict__ scale)
{
    __shared__ double s[CLIP_THREADS];
    const int tid = threadIdx.x;
    s[tid] = partial[tid];                                   // CLIP_BLOCKS == CLIP_THREADS
    const double tot = tree_sum(s, tid);
    if (tid == 0) {
        const float nr = (float)sqrt(tot);
        const float use = isfinite(nr) ? nr : __int_as_float(0x7fc00000);
        const float inv = __fdiv_rn(1.0f, use), cap = __fdiv_rn(1.0f, clip);
        const float m = isnan(inv) ? inv : (inv < cap ? inv : cap);       // tf.minimum: NaN propagates (not fminf)
        *norm = nr;
        *scale = __fmul_rn(clip, m);
    }
}

struct AllreduceParams {
    float *grad;                 // [n] this rank's flat gradient buffer, overwritten with the mean
    const float *scale;          // device scalar: this rank's clip scale
    uint8_t *const *peer_base;   // DEVICE array [world]: every rank's symmetric allocation as mapped here
    int *state;                  // [0] replays done, [1] CTAs of the current replay that have finished, [2] time-outs
    size_t n, chunk, sub;        // floats
    size_t r1[2], r2[2], f1[2], f2[2];   // byte offsets inside every rank's symmetric allocation, per parity
    int world, rank;
};

// returns 1 when the peer arrived, 0 when the wait gave up (counted in state[2])
__device__ __forceinline__ int ar_wait(const int *flag, int seq, int *state)
{
    const long long t0 = clock64();
    while (ld_acquire_sys(flag) < seq) {
        if (clock64() - t0 > kPeerSpinLimit) { atomicAdd(state + 2, 1); return 0; }   // a peer never came: counted, not hung
    }
    return 1;
}

__global__ void __launch_bounds__(AR_THREADS)
peer_allreduce_mean_kernel(const AllreduceParams p)
{
    const int j = blockIdx.x, tid = threadIdx.x, me = p.rank, G = p.world;
    __shared__ int s_seq, s_ok;
    if (tid == 0) { s_seq = *reinterpret_cast<volatile int *>(p.state) + 1; s_ok = 1; }   // state[0] changes only after every CTA read it
    __syncthreads();
    const int seq = s_seq, par = seq & 1;
    const size_t lo = (size_t)j * p.sub;                     // sub-slice j of a chunk: [lo, hi) inside the chunk
    const size_t hi = lo + p.sub < p.chunk ? lo + p.sub : p.chunk;
    const size_t len4 = hi > lo ? (hi - lo) / 4 : 0;         // chunk and sub are multiples of 4
    uint8_t *mine = p.peer_base[me];
    const float sc = *p.scale;
    const size_t r1o = par ? p.r1[1] : p.r1[0], r2o = par ? p.r2[1] : p.r2[0];   // selects, not a local-memory index
    const size_t f1o = par ? p.f1[1] : p.f1[0], f2o = par ? p.f2[1] : p.f2[0];

    // phase 1: my clipped sub-slice j of chunk q -> rank q's R1[par][me][j]
#pragma unroll 1
    for (int k = 0; k < G; k++) {
        const int q = (me + 1 + k) % G;                      // spread the first stores over the links
        float4 *dst = reinterpret_cast<float4 *>(p.peer_base[q] + r1o) + ((size_t)me * p.chunk + lo) / 4;
        const size_t gbase = (size_t)q * p.chunk + lo;
        for (size_t i = tid; i < len4; i += AR_THREADS) {
            const size_t e = gbase + 4 * i;
            float4 v;
            if (e + 3 < p.n) {
                v = *reinterpret_cast<const float4 *>(p.grad + e);   // plain load: phase 3 writes grad
            } else {
                v.x = e < p.n ? p.grad[e] : 0.0f;
                v.y = e + 1 < p.n ? p.grad[e + 1] : 0.0f;
                v.z = e + 2 < p.n ? p.grad[e + 2] : 0.0f;
                v.w = 0.0f;
            }
            v.x = __fmul_rn(v.x, sc); v.y = __fmul_rn(v.y, sc); v.z = __fmul_rn(v.z, sc); v.w = __fmul_rn(v.w, sc);
            dst[i] = v;
        }
    }
    __threadfence_system();
    __syncthreads();
    if (tid == 0) {
        for (int q = 0; q < G; q++) st_release_sys(reinterpret_cast<int *>(p.peer_base[q] + f1o) + (size_t)me * gridDim.x + j, seq);
        for (int q = 0; q < G; q++) s_ok &= ar_wait(reinterpret_cast<const int *>(mine + f1o) + (size_t)q * gridDim.x + j, seq, p.state);
    }
    __syncthreads();

    // phase 2: sub-slice j of my chunk, reduced in rank order -> every rank's R2[par][me][j]
    const float4 *r1 = reinterpret_cast<const float4 *>(mine + r1o);
    const double gd = (double)G;
    for (size_t i = tid; i < len4; i += AR_THREADS) {
        const size_t o = lo / 4 + i;
        float4 c = __ldcg(r1 + o);                           // written by another GPU: not through L1
        double ax = c.x, ay = c.y, az = c.z, aw = c.w;
#pragma unroll 1
        for (int q = 1; q < G; q++) {
            c = __ldcg(r1 + (size_t)q * (p.chunk / 4) + o);
            ax += (double)c.x; ay += (double)c.y; az += (double)c.z; aw += (double)c.w;
        }
        const float4 m = make_float4((float)(ax / gd), (float)(ay / gd), (float)(az / gd), (float)(aw / gd));
#pragma unroll 1
        for (int k = 0; k < G; k++) {
            const int q = (me + 1 + k) % G;
            reinterpret_cast<float4 *>(p.peer_base[q] + r2o)[(size_t)me * (p.chunk / 4) + o] = m;
        }
    }
    __threadfence_system();
    __syncthreads();
    if (tid == 0) {
        for (int q = 0; q < G; q++) st_release_sys(reinterpret_cast<int *>(p.peer_base[q] + f2o) + (size_t)me * gridDim.x + j, seq);
        for (int q = 0; q < G; q++) s_ok &= ar_wait(reinterpret_cast<const int *>(mine + f2o) + (size_t)q * gridDim.x + j, seq, p.state);
    }
    __syncthreads();

    // phase 3: every rank's reduced sub-slice j -> my gradient buffer.  After a wait that gave up the data may be stale:
    // the CTA writes NaN instead, so a broken exchange poisons the step visibly rather than silently.
    const float4 *r2 = reinterpret_cast<const float4 *>(mine + r2o);
    const bool ok = s_ok != 0;
    const float qnan = __int_as_float(0x7fc00000);
#pragma unroll 1
    for (int q = 0; q < G; q++) {
        const size_t gbase = (size_t)q * p.chunk + lo;
        for (size_t i = tid; i < len4; i += AR_THREADS) {
            const size_t e = gbase + 4 * i;
            if (e >= p.n) break;
            const float4 v = ok ? __ldcg(r2 + ((size_t)q * p.chunk + lo) / 4 + i) : make_float4(qnan, qnan, qnan, qnan);
            if (e + 3 < p.n) {
                *reinterpret_cast<float4 *>(p.grad + e) = v;
            } else {
                p.grad[e] = v.x;
                if (e + 1 < p.n) p.grad[e + 1] = v.y;
                if (e + 2 < p.n) p.grad[e + 2] = v.z;
            }
        }
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

__global__ void bn_moving_update_ranks_kernel(float *__restrict__ stats, long n, const float *__restrict__ batch, long ld,
                                              int world, float om)
{
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
        float v = stats[i];
        for (int r = 0; r < world; r++) v = __fsub_rn(v, __fmul_rn(__fsub_rn(v, batch[(size_t)r * ld + i]), om));
        stats[i] = v;
    }
}

}  // namespace ssd3d

using namespace ssd3d;

extern "C" size_t ssd3d_grad_clip_scale_workspace(long n) { return n > 0 ? (size_t)CLIP_BLOCKS * sizeof(double) : 0; }

extern "C" int ssd3d_grad_clip_scale(const float *grad, long n, float clip_norm, void *workspace, float *norm, float *scale,
                                     ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(n > 0, "grad_clip_scale: n=%ld must be > 0", n);
    SSD3D_REQUIRE(grad && workspace && norm && scale, "grad_clip_scale: null pointer");
    SSD3D_REQUIRE(clip_norm > 0.0f && clip_norm < INFINITY, "grad_clip_scale: clip_norm=%g must be positive and finite", clip_norm);
    SSD3D_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 7u) == 0, "grad_clip_scale: workspace must be 8-byte aligned");
    cudaStream_t st = (cudaStream_t)stream;
    grad_sumsq_partial_kernel<<<CLIP_BLOCKS, CLIP_THREADS, 0, st>>>(grad, n, (double *)workspace);
    const int rc = cuda_status(cudaGetLastError(), "grad_sumsq_partial_kernel");
    if (rc) return rc;
    grad_clip_finalize_kernel<<<1, CLIP_THREADS, 0, st>>>((const double *)workspace, clip_norm, norm, scale);
    SSD3D_LAUNCH_CHECK("grad_clip_finalize_kernel");
}

extern "C" int ssd3d_peer_allreduce_resident_ctas(void)
{
    int dev = 0, sms = 0, per_sm = 0;
    int rc = cuda_status(cudaGetDevice(&dev), "peer_allreduce_resident_ctas");
    if (rc) return rc;
    rc = cuda_status(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev), "peer_allreduce_resident_ctas");
    if (rc) return rc;
    rc = cuda_status(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, peer_allreduce_mean_kernel, AR_THREADS, 0),
                     "peer_allreduce_resident_ctas");
    if (rc) return rc;
    return sms * per_sm;
}

extern "C" int ssd3d_peer_allreduce_mean(float *grad, size_t n, const float *scale, void *const *peer_base, int world, int rank,
                                         int ctas, size_t chunk, size_t sub, size_t r1_off0, size_t r1_off1, size_t r2_off0,
                                         size_t r2_off1, size_t f1_off0, size_t f1_off1, size_t f2_off0, size_t f2_off1,
                                         int *state, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(world >= 1 && world <= 64 && rank >= 0 && rank < world, "peer_allreduce_mean: bad world=%d rank=%d", world, rank);
    SSD3D_REQUIRE(ctas >= 1 && ctas <= 1024, "peer_allreduce_mean: ctas=%d must be in [1, 1024]", ctas);
    SSD3D_REQUIRE(grad && scale && peer_base && state, "peer_allreduce_mean: null pointer");
    SSD3D_REQUIRE(n > 0 && chunk % 4 == 0 && sub % 4 == 0 && sub > 0 && chunk * (size_t)world >= n && sub * (size_t)ctas >= chunk,
                  "peer_allreduce_mean: chunk=%zu / sub=%zu must be multiples of 4 covering n=%zu over world=%d, ctas=%d",
                  chunk, sub, n, world, ctas);
    SSD3D_REQUIRE(r1_off0 % 16 == 0 && r1_off1 % 16 == 0 && r2_off0 % 16 == 0 && r2_off1 % 16 == 0 && f1_off0 % 4 == 0 &&
                  f1_off1 % 4 == 0 && f2_off0 % 4 == 0 && f2_off1 % 4 == 0,
                  "peer_allreduce_mean: data offsets must be 16-byte and flag offsets 4-byte multiples");
    SSD3D_REQUIRE((reinterpret_cast<uintptr_t>(grad) & 15u) == 0, "peer_allreduce_mean: grad must be 16-byte aligned");
    AllreduceParams p = {};
    p.grad = grad; p.scale = scale; p.peer_base = (uint8_t *const *)peer_base; p.state = state;
    p.n = n; p.chunk = chunk; p.sub = sub;
    p.r1[0] = r1_off0; p.r1[1] = r1_off1; p.r2[0] = r2_off0; p.r2[1] = r2_off1;
    p.f1[0] = f1_off0; p.f1[1] = f1_off1; p.f2[0] = f2_off0; p.f2[1] = f2_off1;
    p.world = world; p.rank = rank;
    peer_allreduce_mean_kernel<<<ctas, AR_THREADS, 0, (cudaStream_t)stream>>>(p);
    SSD3D_LAUNCH_CHECK("peer_allreduce_mean_kernel");
}

extern "C" int ssd3d_bn_moving_update_ranks(float *stats, long n, const float *batch, long ld_batch, int world, float decay,
                                            ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(n > 0 && world >= 1 && ld_batch >= n, "bn_moving_update_ranks: bad shape n=%ld world=%d ld_batch=%ld", n, world,
                  ld_batch);
    SSD3D_REQUIRE(stats && batch, "bn_moving_update_ranks: null pointer");
    SSD3D_REQUIRE(decay >= 0.0f && decay <= 1.0f, "bn_moving_update_ranks: decay=%g must be in [0,1]", decay);
    const float om = 1.0f - decay;                           // bn.cu computes the same float32 difference
    const int blocks = (int)((n + 255) / 256 < (long)kNumSMs * 4 ? (n + 255) / 256 : (long)kNumSMs * 4);
    bn_moving_update_ranks_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(stats, n, batch, ld_batch, world, om);
    SSD3D_LAUNCH_CHECK("bn_moving_update_ranks_kernel");
}
