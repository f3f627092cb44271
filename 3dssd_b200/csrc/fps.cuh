// fps.cuh -- the round protocol shared by the FPS kernels (fps.cu, fps_bucket.cu).
#pragma once
#include "common.cuh"
#include "fps_plan.h"

namespace ssd3d {

constexpr uint32_t KEY_INVALID = 0x7FFFFFFFu;

// Where a launch reads and writes (the *_ex entry points of include/ssd3d.h): scene strides of the inputs in
// elements (so a [:, a:b] slice of a dense [b,N,c] tensor needs no copy), row stride + value offset of the index
// output (so the segments of a fusion-sampling layer land directly in the concatenated fps_idx tensor with the
// segment offset already added, layers_util.py:109-111), and -- resumable kernels only -- the range of rounds
// [j0, j1) this launch runs, the running distances travelling through `temp` between launches.
struct FpsIO {
    long long sa, sb;   // scene stride of inp / fa (sa) and fb (sb), in floats
    int ldo, ioff;      // out row stride (ints), offset added to every stored index
    int j0, j1;         // rounds [j0, j1) of 0..m (round 0 = "sample point 0")
    float *temp;        // [b, n] running distances (resume state; NULL when j0 == 0 && j1 == m)
};

__device__ __forceinline__ uint32_t fps_key(int k) { return ((uint32_t)(k & 1023) << 21) | (uint32_t)(k >> 10); }
__device__ __forceinline__ int fps_key_to_k(uint32_t key) { return (int)(((key & 0x1FFFFFu) << 10) | (key >> 21)); }

// (value,key) arg-max across a warp: max value, then min key among the lanes holding it.
__device__ __forceinline__ void warp_argmax(uint32_t u, uint32_t key_if_valid, uint32_t &mx, uint32_t &kmin)
{
    mx = __reduce_max_sync(0xffffffffu, u);
    kmin = __reduce_min_sync(0xffffffffu, (u == mx) ? key_if_valid : KEY_INVALID);
}

// A thread's candidate as the (value bits, key) pair the reductions order: values are >= 0, so their bits order like
// the floats; a thread left with padding slots only (best < 0) never wins.
__device__ __forceinline__ uint2 fps_candidate(float best, uint32_t key)
{
    return make_uint2(__float_as_uint(fmaxf(best, 0.0f)), best >= 0.0f ? key : KEY_INVALID);
}

// The reference's contracted distance d = fma(dz,dz, fma(dy,dy, dx*dx)), pinned against re-association; the pair
// form runs the same IEEE operations on two points.
__device__ __forceinline__ float fps_d2(float dx, float dy, float dz)
{
    return __fmaf_rn(dz, dz, __fmaf_rn(dy, dy, __fmul_rn(dx, dx)));
}
__device__ __forceinline__ float2 fps_d2(float2 dx, float2 dy, float2 dz) { return fma2_rn(dz, dz, fma2_rn(dy, dy, mul2_rn(dx, dx))); }

// Ascending scan of a thread's slots: visited in ascending key order, "first strictly greater" keeps the smallest key
// among the thread's maxima.
struct FpsScan {
    float best = -1.0f;
    int at = 0;
    __device__ __forceinline__ void see(float t, int i)
    {
        if (t > best) { best = t; at = i; }
    }
};

// The same answer as a tree of depth log2 P over slots in ascending key order: a higher slot wins only when STRICTLY
// greater.  Leaves the maximum in v[0] and its k in k[0].
template <int P>
__device__ __forceinline__ void fps_tree_argmax(float (&v)[P], int (&k)[P])
{
#pragma unroll
    for (int s = 1; s < P; s *= 2) {
#pragma unroll
        for (int i = 0; i + s < P; i += 2 * s) {
            const bool up = v[i + s] > v[i];
            v[i] = up ? v[i + s] : v[i];
            k[i] = up ? k[i + s] : k[i];
        }
    }
}

// Scene context of a thread of the cluster kernels: its CTA's rank in the scene's cluster, its scene and its global
// thread index g in the scene.
template <int CL>
struct FpsScene {
    int tid;
    uint32_t rank;
    int scene, g;
    __device__ __forceinline__ FpsScene()
        : tid(threadIdx.x), rank(CL > 1 ? cluster_ctarank() : 0u), scene(blockIdx.x / CL), g((int)rank * FPS_T + tid) {}
    // this scene's part of a [b, ...] input with scene stride `stride` floats, and its row of the index output
    __device__ __forceinline__ const float *in(const float *base, long long stride) const { return base + (size_t)scene * stride; }
    __device__ __forceinline__ int *row(int *out, const FpsIO &io) const { return out + (size_t)scene * io.ldo; }
};

// The rounds one launch runs, [jbeg, jend) of 1..m-1, and the scene's index output.  A launch that does not start at
// round 0 reloads the running distances from `dist` (the scene's part of temp) and the last winner from the index
// output; one that stops before m saves the distances there.
struct FpsRounds {
    int jbeg, jend;
    bool resume, save;
    int *idxs;
    int ioff;
    float *dist;
    __device__ __forceinline__ FpsRounds(const FpsIO &io, int m, int scene, int *out, long long temp_stride)
        : jbeg(io.j0 > 1 ? io.j0 : 1), jend(io.j1 < m ? io.j1 : m), resume(io.j0 > 0), save(io.j1 < m),
          idxs(out + (size_t)scene * io.ldo), ioff(io.ioff), dist(io.temp + (size_t)scene * temp_stride) {}
    // starting distance of point k (padding slots start at -1: min(d,-1) stays -1, valid values are >= 0)
    __device__ __forceinline__ float start(int k, bool valid) const { return valid ? (resume ? dist[k] : 1e38f) : -1.0f; }
    // the sample the launch starts from: the previous launch's last winner, or point 0, which `writer` then stores
    __device__ __forceinline__ int first(bool writer) const
    {
        if (resume) return idxs[jbeg - 1] - ioff;
        if (writer) idxs[0] = ioff;
        return 0;
    }
    __device__ __forceinline__ void put(int j, int k) const { idxs[j] = k + ioff; }
    // save the P running distances of the thread; where(i) is the point of slot i, < 0 for none
    template <int P, class Where>
    __device__ __forceinline__ void save_dist(const float (&td)[P], Where where) const
    {
        if (!save) return;
#pragma unroll
        for (int i = 0; i < P; i++) {
            const int k = where(i);
            if (k >= 0) dist[k] = td[i];
        }
    }
};

// The two-parity mbarrier ring of the per-round exchange.  Round r, counted from 1 at the launch's first round, uses
// buffer and barrier r & 1 and waits for phase ((r - 1) >> 1) & 1 of that barrier; peers complete its tx-bytes with
// st.async.  Every kernel keeps its own packets and send pattern.
struct FpsRing {
    unsigned long long bar[2];
    // thread 0: both barriers, fenced for the cluster together with the thread's earlier barrier inits
    __device__ __forceinline__ void init()
    {
        mbar_init(smem_u32(&bar[0]), 1);
        mbar_init(smem_u32(&bar[1]), 1);
        fence_mbar_init_cluster();
    }
    // init + every CTA's barriers exist before any peer st.async targets them
    template <int CL>
    __device__ __forceinline__ void start()
    {
        if (threadIdx.x == 0) init();
        __syncthreads();
        if (CL > 1) cluster_sync_all();
    }
    __device__ __forceinline__ uint32_t at(int r) { return smem_u32(&bar[r & 1]); }
    __device__ __forceinline__ void expect(int r, uint32_t bytes) { mbar_arrive_expect_tx(at(r), bytes); }
    __device__ __forceinline__ void wait(int r) { mbar_wait_cta(at(r), ((r - 1) >> 1) & 1); }
};

// fps_bucket.cu: single-CTA D-FPS with spatial pruning for large xyz scenes
int launch_fps3_bucket(int b, int n, int m, const float *inp, int *out, const FpsIO &io, cudaStream_t st);

}  // namespace ssd3d
