// fps_bucket.cu -- the pruned FPS kernels, which skip the points a new sample cannot reach: fps3_bucket_kernel (D-FPS,
// 8192 < n <= 16384 on one CTA: 3DSSD layer 1) and ffps_bucket_kernel (F-FPS, 2048 < n <= 4096 on four: layer 2).
//
// fps3_bucket_kernel.  Same function as fps3_direct_kernel (fps.cu), i.e. farthestpointsamplingKernel of
// /root/reference/lib/utils/tf_ops/sampling/tf_sampling_g.cu:124-178 for c == 3, same indices bit for bit.
//
// Why another kernel.  A round of FPS is  dist[k] = min(dist[k], d(k, last sample))  for every point, then an arg-max.
// The cluster kernel does the full update with the points spread over 4-8 SMs and pays a DSMEM exchange per round
// (~390 ns per round, 4095 rounds, 32-64 SMs busy per batch of 8 scenes).  But after a few dozen rounds a new sample
// can only LOWER the running distance of points in its own neighbourhood: dist[k] is already the distance to the
// nearest of j samples, so only points closer to the new sample than that change.  With the points grouped into
// spatially compact buckets of 32 (2-D Morton order of the two widest axes) and an axis-aligned box per bucket,
//     lower bound of d(any point of the box, s)  >=  max running distance inside the bucket
// proves that the round leaves the bucket untouched -- no distance needs to be computed, and its cached (max, arg-max)
// stays valid.  On the benchmark's layer-1 scenes a round touches 1.4 % of the 512 buckets (tools/fps_prune_stats.py).
// A whole scene then fits ONE CTA: coordinates in shared memory (SoA, 192 KiB), running distances in registers (32 per
// thread), no cluster, no DSMEM; a round is  bucket test -> update of the (usually one) affected bucket of a warp -> one
// __syncthreads -> 16-entry arg-max.  The reductions carry (value, key) only, and the key word holds the point's place
// in bucket order below its tie-break fields, so the winner's coordinates are one shared-memory read away: a ballot +
// find-first to track lanes costs as much as the two REDUX of a stage (tools/ubench/warp_ops.cu).  One SM per scene
// instead of 4-8.
//
// Exactness.  Skipping is the only approximation-shaped step and it is one-sided: a bucket is skipped only when
// lb * (1 - 1e-5) >= bucket max, where lb is the squared distance from the sample to the box computed in fp32; the
// reference's fp32 distance of any point inside the box is >= lb * (1 - 8 * 2^-24) (every operation rounds to nearest
// and all terms are non-negative), so a skipped point satisfies d >= dist[k] and min() would not have changed it.
// Tiny values (lb < 1e-30, where denormal rounding breaks relative bounds) never skip.  Everything that IS computed
// uses the reference's contracted recipe d = fma(dz,dz, fma(dy,dy, dx*dx)) and the arg-max order
// (value desc, k mod 1024 asc, k asc) of fps.cu.  The bucket assignment itself cannot change a result.
//
// Resumable like fps3_direct_kernel (rounds [j0, j1)): running distances travel through temp[scene][0:n] in ORIGINAL
// point order, the bucket permutation through temp[scene][n:2n], so a resumed launch skips the sort.
#include "common.cuh"
#include "fps.cuh"

namespace ssd3d {

constexpr int FB_T = 512;                    // threads per CTA (one CTA per scene)
constexpr int FB_NW = FB_T / 32;             // 16 warps
constexpr int FB_SLOTS = 32;                 // buckets per warp: lane l OWNS the meta data of the warp's slot l
constexpr int FB_NBUCKET = FB_NW * FB_SLOTS; // 512
static_assert(FB_NBUCKET * 32 == FB_MAXN, "one point per lane of every bucket slot (fps_plan.h)");
constexpr uint32_t FB_PAD_KEY = 0xFFFFFFFFu;

__device__ __forceinline__ uint32_t fb_spread9(uint32_t v)   // 9 bits -> every second bit
{
    v &= 0x1ffu;
    v = (v | (v << 8)) & 0x00ff00ffu;
    v = (v | (v << 4)) & 0x0f0f0f0fu;
    v = (v | (v << 2)) & 0x33333333u;
    v = (v | (v << 1)) & 0x55555555u;
    return v;
}

// position of (warp w, slot i, lane l) in bucket order: consecutive buckets belong to different warps, so the buckets a
// sample touches (neighbours in Morton order) are worked on in parallel
__device__ __forceinline__ int fb_pos(int w, int i, int lane) { return ((i * FB_NW + w) << 5) + lane; }


#define FB_CASE(I)                                                              \
    case I:                                                                     \
        nd = fminf(d, dist[I]);                                                 \
        dist[I] = nd;                                                           \
        break;

__global__ void __launch_bounds__(FB_T, 1)
fps3_bucket_kernel(int n, int m, const float *__restrict__ inp, int *__restrict__ out, const FpsIO io)
{
    extern __shared__ float4 fb_dyn[];
    float *xs = reinterpret_cast<float *>(fb_dyn);          // [FB_MAXN] sorted x          (first 64 KiB: sort keys during setup)
    float *ys = xs + FB_MAXN, *zs = ys + FB_MAXN;
    uint32_t *skey = reinterpret_cast<uint32_t *>(fb_dyn);
    __shared__ __align__(8) uint2 slots[2][FB_NW];          // per round parity: (max bits, key) of every warp's best point
    __shared__ uint32_t red[6][FB_NW];
    __shared__ uint16_t orig_of[FB_MAXN];                   // position in bucket order -> original index (0xffff: no point)

    const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
    const int scene = blockIdx.x;
    const float *data = inp + (size_t)scene * io.sa;
    const FpsRounds rounds(io, m, scene, out, 2LL * n);
    uint32_t *perm = io.temp ? reinterpret_cast<uint32_t *>(rounds.dist + n) : nullptr;

    float dist[FB_SLOTS];

    if (!rounds.resume) {
        // ---- scene box -> 2-D Morton keys of the two widest axes -> bitonic sort (key = morton18 : index14)
        float lo[3], hi[3], ext[3];
        fps_scene_box<FB_T>(n, [&](int k, int a) { return __ldg(data + 3 * k + a); }, red, lo, hi);
#pragma unroll
        for (int a = 0; a < 3; a++) ext[a] = hi[a] - lo[a];
        // the two widest axes (a0 widest), square cells sized by the widest; non-finite extents just give poor buckets
        int a0 = 0, a1 = 1;
        if (ext[1] > ext[a0]) a0 = 1;
        if (ext[2] > ext[a0]) a0 = 2;
        a1 = a0 == 0 ? 1 : 0;
        for (int a = 0; a < 3; a++)
            if (a != a0 && ext[a] > ext[a1]) a1 = a;
        const float scale = ext[a0] > 0.0f ? 511.999f / ext[a0] : 0.0f;
        int np = 1024;
        while (np < n) np <<= 1;                                  // sort size (n <= FB_MAXN)
        for (int k = tid; k < np; k += FB_T) {
            uint32_t key = FB_PAD_KEY;
            if (k < n) {
                const float u = (__ldg(data + 3 * k + a0) - lo[a0]) * scale, v = (__ldg(data + 3 * k + a1) - lo[a1]) * scale;
                const uint32_t qu = (uint32_t)min(511, max(0, (int)u)), qv = (uint32_t)min(511, max(0, (int)v));
                key = ((fb_spread9(qu) | (fb_spread9(qv) << 1)) << 14) | (uint32_t)k;
            }
            skey[k] = key;
        }
        __syncthreads();
        fps_bitonic_sort<uint32_t, FB_T, FB_MAXN>(skey, np);
#pragma unroll
        for (int i = 0; i < FB_SLOTS; i++) {
            const int p = fb_pos(w, i, lane);
            uint32_t o = 0xffffu;                                  // 0xffff marks "no point" (n <= 16384 < 0xffff)
            if (p < n) o = skey[p] & 0x3fffu;
            orig_of[p] = (uint16_t)o;
            if (perm != nullptr && p < n) perm[p] = o;
        }
        __syncthreads();                                           // sort buffer consumed: xs may be overwritten
    } else {
#pragma unroll
        for (int i = 0; i < FB_SLOTS; i++) {
            const int p = fb_pos(w, i, lane);
            orig_of[p] = (uint16_t)(p < n ? (perm[p] & 0xffffu) : 0xffffu);
        }
    }

    // ---- coordinates into bucket order, bucket boxes, running distances
    float bminx = 0, bminy = 0, bminz = 0, bmaxx = 0, bmaxy = 0, bmaxz = 0;   // box of the slot this lane owns
    uint32_t bmaxu = 0u, bkey = KEY_INVALID;                                  // its max (bits) and the key of the point holding it
#pragma unroll
    for (int i = 0; i < FB_SLOTS; i++) {
        const int p = fb_pos(w, i, lane);
        const uint32_t o = orig_of[p];                             // written by this thread above
        const bool valid = o != 0xffffu;
        float x = 0.0f, y = 0.0f, z = 0.0f;
        if (valid) { x = __ldg(data + 3 * o); y = __ldg(data + 3 * o + 1); z = __ldg(data + 3 * o + 2); }
        xs[p] = x; ys[p] = y; zs[p] = z;
        dist[i] = rounds.start(o, valid);                          // tf_sampling_g.cu:136
        const uint32_t mnx = __reduce_min_sync(0xffffffffu, valid ? fps_ord(x) : 0xffffffffu);
        const uint32_t mny = __reduce_min_sync(0xffffffffu, valid ? fps_ord(y) : 0xffffffffu);
        const uint32_t mnz = __reduce_min_sync(0xffffffffu, valid ? fps_ord(z) : 0xffffffffu);
        const uint32_t mxx = __reduce_max_sync(0xffffffffu, valid ? fps_ord(x) : 0u);
        const uint32_t mxy = __reduce_max_sync(0xffffffffu, valid ? fps_ord(y) : 0u);
        const uint32_t mxz = __reduce_max_sync(0xffffffffu, valid ? fps_ord(z) : 0u);
        // arg-max of the slot as it stands (a fresh start has 1e38 everywhere: every bucket is "affected" in round 1)
        const uint32_t u = valid ? __float_as_uint(fmaxf(dist[i], 0.0f)) : 0u;
        const uint32_t key = valid ? fps_place_key<4>(o, (uint32_t)p) : KEY_INVALID;
        uint32_t mx, kmin;
        warp_argmax(u, key, mx, kmin);
        if (lane == i) {
            bminx = fps_unord(mnx); bminy = fps_unord(mny); bminz = fps_unord(mnz);
            bmaxx = fps_unord(mxx); bmaxy = fps_unord(mxy); bmaxz = fps_unord(mxz);
            bmaxu = mx; bkey = kmin;
        }
    }

    const int old0 = rounds.first(tid == 0);
    float sx = __ldg(data + 3 * old0), sy = __ldg(data + 3 * old0 + 1), sz = __ldg(data + 3 * old0 + 2);
    // the warp's best over its 32 slots, cached between rounds (valid while none of its buckets changes)
    uint32_t wm = 0u, wk = KEY_INVALID;
    bool wdirty = true;
    __syncthreads();                                               // xs / ys / zs complete

    for (int j = rounds.jbeg; j < rounds.jend; j++) {
        const int par = j & 1;
        // ---- which of this warp's buckets can the new sample change?  (lane l tests slot l)
        const float gx = fmaxf(fmaxf(bminx - sx, sx - bmaxx), 0.0f);
        const float gy = fmaxf(fmaxf(bminy - sy, sy - bmaxy), 0.0f);
        const float gz = fmaxf(fmaxf(bminz - sz, sz - bmaxz), 0.0f);
        const float lb = gx * gx + gy * gy + gz * gz;
        const bool skip = bmaxu == 0u || (lb * 0.99999f >= __uint_as_float(bmaxu) && lb >= 1e-30f);
        uint32_t mask = __ballot_sync(0xffffffffu, !skip);
        wdirty = wdirty || mask != 0u;
        while (mask) {
            const int i = 31 - __clz(mask);                        // warp-uniform; any order (find-leading-one is the cheaper one)
            mask &= ~(1u << i);
            const int p = fb_pos(w, i, lane);
            const uint32_t kk = orig_of[p];
            const float dx = xs[p] - sx, dy = ys[p] - sy, dz = zs[p] - sz;
            const float d = fps_d2(dx, dy, dz);
            float nd;
            switch (i) {
                FB_CASE(0) FB_CASE(1) FB_CASE(2) FB_CASE(3) FB_CASE(4) FB_CASE(5) FB_CASE(6) FB_CASE(7)
                FB_CASE(8) FB_CASE(9) FB_CASE(10) FB_CASE(11) FB_CASE(12) FB_CASE(13) FB_CASE(14) FB_CASE(15)
                FB_CASE(16) FB_CASE(17) FB_CASE(18) FB_CASE(19) FB_CASE(20) FB_CASE(21) FB_CASE(22) FB_CASE(23)
                FB_CASE(24) FB_CASE(25) FB_CASE(26) FB_CASE(27) FB_CASE(28) FB_CASE(29) FB_CASE(30)
                default: nd = fminf(d, dist[31]); dist[31] = nd; break;
            }
            const bool valid = kk != 0xffffu;
            const uint32_t u = valid ? __float_as_uint(fmaxf(nd, 0.0f)) : 0u;
            const uint32_t key = valid ? fps_place_key<4>(kk, (uint32_t)p) : KEY_INVALID;
            uint32_t mx, kmin;
            warp_argmax(u, key, mx, kmin);
            if (lane == i) { bmaxu = mx; bkey = kmin; }
        }
        if (wdirty) {                                              // warp-uniform
            warp_argmax(bmaxu, bkey, wm, wk);
            wdirty = false;
        }
        if (lane == 0) slots[par][w] = make_uint2(wm, wk);
        __syncthreads();
        // ---- scene-wide arg-max of the 16 warp candidates (every warp, redundantly: no second barrier); the winning key
        // carries the winner's place
        const uint2 c = slots[par][lane & (FB_NW - 1)];
        uint32_t m3, k3;
        warp_argmax(c.x, c.y, m3, k3);
        const int p = (int)(k3 & 0x3fffu);
        sx = xs[p]; sy = ys[p]; sz = zs[p];
        if (tid == 0) rounds.put(j, fps_place_key_to_k<4>(k3));
    }

    rounds.save_dist(dist, [&](int i) {
        const uint32_t o = orig_of[fb_pos(w, i, lane)];
        return o != 0xffffu ? (int)o : -1;
    });
}

int launch_fps3_bucket(int b, int n, int m, const float *inp, int *out, const FpsIO &io, cudaStream_t st)
{
    cudaError_t e = cudaFuncSetAttribute((const void *)fps3_bucket_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)FB_SMEM);
    if (e != cudaSuccess) return (int)e;
    fps3_bucket_kernel<<<b, FB_T, FB_SMEM, st>>>(n, m, inp, out, io);
    return (int)cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------------
// ffps_bucket_kernel: matrix-free F-FPS on FOUR CTAs per scene with bucket pruning (plan_ffps: a capped cluster request,
// full range, 2048 < n <= 4096, c <= 68).  Same indices as ffps_cluster_kernel (fps.cu), which needs 8 CTAs for these scenes.
//
// Layout.  4 point slots per thread: slots 0-1 in registers (as ffps_cluster_kernel), slots 2-3 as rows in shared
// memory.  The points are placed in 3-D Morton order of xyz (channels 0-2), and a BUCKET is the 32 lanes of one
// (warp, slot): bucket B (0..127, Morton order) lives in CTA B % 4, warp (B / 4) % 8, slot B / 32, so the few
// neighbouring buckets a sample reaches are spread over CTAs and warps.  Every bucket has a centre c (the mean row), a
// radius rho >= max |x - c| and the largest squared norm of its rows; lane 8i of a warp holds slot i's bounds and its
// cached (value, key) arg-max.
//
// Skip rule.  A new sample w can only lower the running distance td of a point x when the computed value
//     v = (sq_w + sq_x) - 2 dot(w, x)           (sqdist's pinned fma chains, 68 terms)
// is below td.  With D = |w - x|^2 exactly, the chains' rounding gives |v - D| <= (2 gamma_68 + 3u)(|w|^2 + |x|^2)
// (u = 2^-24, gamma_68 = 68u / (1 - 68u): gamma_68 |w|^2 and gamma_68 |x|^2 from the two norm chains, gamma_68 * 2|w||x|
// <= gamma_68 (|w|^2 + |x|^2) from the dot chain, u from the addition and 2u from the final subtraction, whose operand is
// below 2 (|w|^2 + |x|^2)), plus an absolute term below 1e-40 for denormal products.  So with E = 8.4e-6 (sq_w + sqmax_b)
// + 1e-36 (8.4e-6 > 139u = 8.29e-6 and absorbs the first-order (1 + gamma) factors of the computed norms) and
//     D >= (|w - c| - rho)^2                      (triangle inequality, when |w - c| > rho),
// lb = (|w - c|_lo - rho_hi)^2 * 0.9999 - E is a lower bound of v for every point of the bucket; |w - c|_lo and rho_hi
// are fp32 sums of squares shrunk / grown by 1e-4 (relative error of a 72-term sum of non-negative terms < 72u) and 1e-36
// (denormals).  lb >= (cached max td of the bucket) proves fminf(v, td) == td for all its points: the bucket is skipped,
// keeps its cached arg-max, and neither its rows are read nor its products computed.  An empty bucket has rho = -inf.
// On the layer-2 operands of the benchmark a round touches 10 % of the 128 buckets (tools/fps_prune_stats.py).
//
// Keys.  fps_place_key<2>(o, place) carries the point's place in its CTA (slot * 256 + thread), so the arg-max itself
// says where the winner's row is.  Before the round's barrier every warp stages its best point (squared norm, and the
// row when it is in registers) into a per-warp row of the round's parity; after it warps 0-3 push the CTA candidate's
// packet (header + row, 18 pieces of 16 bytes) to CTA 0-3 with st.async, as ffps_cluster_kernel does.
// ---------------------------------------------------------------------------------------------------
constexpr int FFB_CP = 68, FFB_CEN = 72, FFB_NP = 1 + FFB_CP / 4;
static_assert(FFB_CL * FPS_T * 4 == FFB_MAXN && FFB_MAXN == 4096, "2 bits of o div 1024 in the place key (fps_plan.h)");
static_assert(ffps_bucket_smem() == (size_t)2 * FPS_T * FFB_CP * 4 + (size_t)FFB_MAXN * 8 + (size_t)FPS_NW * 4 * FFB_CEN * 4 +
                                        (size_t)2 * FPS_NW * (FFB_CP + 4) * 4 + 2 * FFB_CL * sizeof(FfpsPacket<FFB_CP>),
              "ffps_bucket_smem (fps_plan.h)");

__device__ __forceinline__ uint32_t ffb_spread10(uint32_t v)   // 10 bits -> every third bit
{
    v &= 0x3ffu;
    v = (v | (v << 16)) & 0x030000ffu;
    v = (v | (v << 8)) & 0x0300f00fu;
    v = (v | (v << 4)) & 0x030c30c3u;
    v = (v | (v << 2)) & 0x09249249u;
    return v;
}

__device__ __forceinline__ float warp_sum8(float v)   // sum over the aligned group of 8 lanes
{
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    return v;
}

__global__ void __launch_bounds__(FPS_T, 1)
ffps_bucket_kernel(int n, int ca, int cb, int m, const float *__restrict__ fa, const float *__restrict__ fb,
                   int *__restrict__ out, const FpsIO io)
{
    using Packet = FfpsPacket<FFB_CP>;
    extern __shared__ float4 dyn_smem[];
    float *rows = reinterpret_cast<float *>(dyn_smem);                          // [2][FPS_T][68] slots 2-3
    unsigned long long *skey = reinterpret_cast<unsigned long long *>(rows + 2 * FPS_T * FFB_CP);   // [4096] sort
    float *cen = reinterpret_cast<float *>(skey + FFB_MAXN);                     // [8 warps][4 slots][72]
    float *stage = cen + FPS_NW * 4 * FFB_CEN;                                   // [2][8 warps][68 + 4]
    Packet *cl_pk = reinterpret_cast<Packet *>(stage + 2 * FPS_NW * (FFB_CP + 4));   // [2][4]
    __shared__ uint32_t warp_val[2][FPS_NW], warp_key[2][FPS_NW];
    __shared__ uint32_t red[6][FPS_NW];
    __shared__ FpsRing ring;

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, gi = lane >> 3, gl = lane & 7;
    const FpsScene<FFB_CL> s;
    const int c = ca + cb;
    const float *A = s.in(fa, io.sa);
    const float *B = s.in(fb, io.sb);
    int *idxs = s.row(out, io);
    auto chan = [&](int k, int l) -> float {
        return l < ca ? __ldg(A + (size_t)k * ca + l) : (l < c ? __ldg(B + (size_t)k * cb + (l - ca)) : 0.0f);
    };

    // ---- 3-D Morton order of xyz (every CTA sorts the whole scene: 4096 64-bit keys, a few microseconds)
    {
        float lo[3], hi[3], ext = 0.0f;
        fps_scene_box<FPS_T>(n, chan, red, lo, hi);
#pragma unroll
        for (int a = 0; a < 3; a++) ext = fmaxf(ext, hi[a] - lo[a]);
        const float scale = ext > 0.0f ? 1023.999f / ext : 0.0f;   // cubic cells sized by the widest axis
#pragma unroll 8
        for (int k = s.tid; k < FFB_MAXN; k += FPS_T) {
            unsigned long long key = ~0ull;
            if (k < n) {
                uint32_t mc = 0;
#pragma unroll
                for (int a = 0; a < 3; a++)
                    mc |= ffb_spread10((uint32_t)min(1023, max(0, (int)((chan(k, a) - lo[a]) * scale)))) << a;
                key = ((unsigned long long)mc << 12) | (unsigned long long)k;
            }
            skey[k] = key;
        }
        __syncthreads();
        fps_bitonic_sort<unsigned long long, FPS_T, FFB_MAXN>(skey, FFB_MAXN);
    }
    // Morton position of slot i of thread t of this CTA; the point there (-1: none)
    auto point_at = [&](int i, int t) -> int {
        const int q = (((i * 32 + (t >> 5) * 4 + (int)s.rank)) << 5) | (t & 31);
        return q < n ? (int)(skey[q] & 4095ull) : -1;
    };

    // ---- rows, norms, keys, running distances and bucket bounds, two slots per pass through `rows`
    float f[2][FFB_CP], td[4], sq[4];
    uint32_t key[4];
    float rho_hi = 0.0f, sqmax = 0.0f;        // lane 8i: bounds of slot i's bucket
    uint32_t bval = 0u, bkey = KEY_INVALID;   // lane 8i: its cached arg-max
#pragma unroll
    for (int pass = 0; pass < 2; pass++) {
        // rows[q][l] of the pass's two slots, 8 loads per thread in flight; consecutive threads read along a row
        constexpr int EL = 2 * FPS_T * FFB_CP, U = 8;
        static_assert(EL % (U * FPS_T) == 0, "whole batches");
        for (int e0 = s.tid; e0 < EL; e0 += U * FPS_T) {
            float v[U];
#pragma unroll
            for (int u = 0; u < U; u++) {
                const int e = e0 + u * FPS_T, q = e / FFB_CP, l = e % FFB_CP;
                const int o = point_at(2 * pass + q / FPS_T, q % FPS_T);
                v[u] = o >= 0 ? chan(o, l) : 0.0f;
            }
#pragma unroll
            for (int u = 0; u < U; u++) rows[e0 + u * FPS_T] = v[u];
        }
        __syncthreads();
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const int i = 2 * pass + h;
            const int o = point_at(i, s.tid);
            const float *row = rows + (h * FPS_T + s.tid) * FFB_CP;
            float s2 = 0.0f;
#pragma unroll
            for (int l = 0; l < FFB_CP; l++) {
                const float v = row[l];
                if (pass == 0) f[h][l] = v;
                s2 = __fmaf_rn(v, v, s2);                                  // sqdist's squared-norm chain
            }
            sq[i] = s2;
            td[i] = o >= 0 ? 1e38f : -1.0f;                                // tf_sampling_g.cu:188
            key[i] = o >= 0 ? fps_place_key<2>((uint32_t)o, (uint32_t)(i * FPS_T + s.tid)) : KEY_INVALID;
            // bucket centre: lane l averages channels l, l + 32, l + 64 over the warp's 32 rows of this slot
            const int cnt = __popc(__ballot_sync(0xffffffffu, o >= 0));
            float *cw = cen + (warp * 4 + i) * FFB_CEN;
            for (int l = lane; l < FFB_CEN; l += 32) {
                float acc = 0.0f;
                if (l < FFB_CP)
#pragma unroll
                    for (int t = 0; t < 32; t++) acc += rows[(h * FPS_T + warp * 32 + t) * FFB_CP + l];
                cw[l] = cnt > 0 ? acc / (float)cnt : 0.0f;
            }
            __syncwarp();
            float r2 = 0.0f;
#pragma unroll
            for (int l = 0; l < FFB_CP; l++) { const float d = row[l] - cw[l]; r2 = __fmaf_rn(d, d, r2); }
            const uint32_t r2max = __reduce_max_sync(0xffffffffu, o >= 0 ? __float_as_uint(r2) : 0u);
            const uint32_t sqm = __reduce_max_sync(0xffffffffu, o >= 0 ? __float_as_uint(s2) : 0u);
            const uint2 cd = fps_candidate(td[i], key[i]);
            uint32_t mx, kmin;
            warp_argmax(cd.x, cd.y, mx, kmin);
            if (lane == 8 * i) {
                rho_hi = cnt > 0 ? sqrtf(__uint_as_float(r2max) * 1.0001f + 1e-36f) * 1.0001f : -INFINITY;
                sqmax = __uint_as_float(sqm);
                bval = mx; bkey = kmin;
            }
        }
        if (pass == 0) __syncthreads();                                    // rows of slots 0-1 consumed
    }
    if (s.tid == 0) ring.init();
    // point 0 is the first sample: every CTA reads its row from global memory
    {
        Packet &p0 = cl_pk[0];
        for (int l = s.tid; l < FFB_CP; l += FPS_T) p0.feat[l] = chan(0, l);
        __syncthreads();
        if (s.tid == 0) {
            float s2 = 0.0f;
            for (int l = 0; l < FFB_CP; l++) s2 = __fmaf_rn(p0.feat[l], p0.feat[l], s2);
            p0.sq = s2;
        }
        if (s.g == 0) idxs[0] = io.ioff;
    }
    __syncthreads();                          // `rows` keeps slots 2-3 from the second pass
    cluster_sync_all();                       // every CTA's barriers exist before any peer st.async targets them

    uint32_t wm = 0u, wk = KEY_INVALID;       // the warp's best over its 4 buckets
    uint32_t staged0 = ~0u, staged1 = ~0u;    // key of the point in the warp's staging row of parity 0 / 1 (~0: none)
    warp_argmax((lane & 7) == 0 ? bval : 0u, (lane & 7) == 0 ? bkey : KEY_INVALID, wm, wk);
    const Packet *oldp = &cl_pk[0];
    for (int j = 1; j < m; j++) {
        const int par = j & 1;
        // ---- bucket test: lanes 8i..8i+7 measure |w - c_i| over channels gl, gl + 8, ...
        const float so = oldp->sq;
        uint32_t mask;
        {
            const float *cw = cen + (warp * 4 + gi) * FFB_CEN;
            float dc2 = 0.0f;
#pragma unroll
            for (int t = 0; t < 9; t++) {
                const int l = gl + 8 * t;
                if (l < FFB_CP) { const float d = oldp->feat[l] - cw[l]; dc2 = __fmaf_rn(d, d, dc2); }
            }
            dc2 = warp_sum8(dc2);
            const float dc_lo = sqrtf(fmaxf(dc2 * 0.9999f - 1e-36f, 0.0f)) * 0.9999f;
            const float g = fmaxf(dc_lo - rho_hi, 0.0f);
            const float lb = g * g * 0.9999f - (8.4e-6f * (so + sqmax) + 1e-36f);
            mask = __ballot_sync(0xffffffffu, gl == 0 && !(lb >= __uint_as_float(bval)));
        }
        // ---- touched buckets: distance update and a fresh arg-max (the bucket index is warp-uniform)
        if (mask != 0u) {
            const float4 *of4 = reinterpret_cast<const float4 *>(oldp->feat);
#pragma unroll
            for (int i = 0; i < 4; i++) {
                if ((mask >> (8 * i)) & 1u) {
                    float dot = 0.0f;
                    if (i < 2) {
#pragma unroll
                        for (int l4 = 0; l4 < FFB_CP / 4; l4++) {
                            const float4 o = of4[l4];
                            dot = __fmaf_rn(o.x, f[i & 1][4 * l4 + 0], dot);
                            dot = __fmaf_rn(o.y, f[i & 1][4 * l4 + 1], dot);
                            dot = __fmaf_rn(o.z, f[i & 1][4 * l4 + 2], dot);
                            dot = __fmaf_rn(o.w, f[i & 1][4 * l4 + 3], dot);
                        }
                    } else {
                        const float4 *x4 = reinterpret_cast<const float4 *>(rows + ((i - 2) * FPS_T + s.tid) * FFB_CP);
#pragma unroll
                        for (int l4 = 0; l4 < FFB_CP / 4; l4++) {
                            const float4 o = of4[l4], x = x4[l4];
                            dot = __fmaf_rn(o.x, x.x, dot);
                            dot = __fmaf_rn(o.y, x.y, dot);
                            dot = __fmaf_rn(o.z, x.z, dot);
                            dot = __fmaf_rn(o.w, x.w, dot);
                        }
                    }
                    const float d = __fsub_rn(__fadd_rn(so, sq[i]), __fmul_rn(2.0f, dot));
                    td[i] = fminf(d, td[i]);
                    const uint2 cd = fps_candidate(td[i], key[i]);
                    uint32_t mx, kmin;
                    warp_argmax(cd.x, cd.y, mx, kmin);
                    if (lane == 8 * i) { bval = mx; bkey = kmin; }
                }
            }
            warp_argmax(gl == 0 ? bval : 0u, gl == 0 ? bkey : KEY_INVALID, wm, wk);
        }
        // ---- the warp's best into this parity's staging row (squared norm, and the row itself when it lives in
        // registers), so that any warp can send it after the barrier.  Written only when it changed since this parity
        // was last written; the other parity is still being read by the previous round's senders.
        if (wk != (par ? staged1 : staged0)) {
            if (par) staged1 = wk;
            else staged0 = wk;
            const int place = wk != KEY_INVALID ? (int)(wk & 1023u) : 2 * FPS_T + warp * 32;
            const int oslot = place >> 8;
            if (lane == (place & 31)) {
                float *st = stage + (par * FPS_NW + warp) * (FFB_CP + 4);
                st[FFB_CP] = oslot == 0 ? sq[0] : oslot == 1 ? sq[1] : oslot == 2 ? sq[2] : sq[3];
                if (oslot < 2) {
                    float4 *d4 = reinterpret_cast<float4 *>(st);
#pragma unroll
                    for (int l4 = 0; l4 < FFB_CP / 4; l4++)
                        d4[l4] = oslot == 0 ? make_float4(f[0][4 * l4], f[0][4 * l4 + 1], f[0][4 * l4 + 2], f[0][4 * l4 + 3])
                                            : make_float4(f[1][4 * l4], f[1][4 * l4 + 1], f[1][4 * l4 + 2], f[1][4 * l4 + 3]);
                }
            }
        }
        if (lane == 0) { warp_val[par][warp] = wm; warp_key[par][warp] = wk; }
        __syncthreads();
        // ---- CTA candidate (every warp reduces redundantly); warp w sends header + row to CTA w, one piece per lane
        if (s.tid == 0) ring.expect(j, FFB_CL * FFB_NP * 16);
        if (warp < FFB_CL) {
            const uint32_t v = lane < FPS_NW ? warp_val[par][lane] : 0u;
            const uint32_t kk = lane < FPS_NW ? warp_key[par][lane] : KEY_INVALID;
            uint32_t m2, k2;
            warp_argmax(v, kk, m2, k2);
            const int place = k2 != KEY_INVALID ? (int)(k2 & 1023u) : 2 * FPS_T;   // nothing valid left: warp 0's entry
            const int ow = (place & (FPS_T - 1)) >> 5;
            const int oslot = place >> 8, ot = place & (FPS_T - 1);
            const float *st = stage + (par * FPS_NW + ow) * (FFB_CP + 4);
            const float4 *src = reinterpret_cast<const float4 *>(oslot < 2 ? st : rows + ((oslot - 2) * FPS_T + ot) * FFB_CP);
            if (lane < FFB_NP) {
                const float4 v4 = lane == 0 ? make_float4(__uint_as_float(m2), __uint_as_float(k2), st[FFB_CP], 0.0f) : src[lane - 1];
                st_async_v4(mapa(smem_u32(&cl_pk[par * FFB_CL + s.rank]) + lane * 16, (uint32_t)warp), mapa(ring.at(j), (uint32_t)warp),
                            make_uint4(__float_as_uint(v4.x), __float_as_uint(v4.y), __float_as_uint(v4.z), __float_as_uint(v4.w)));
            }
        }
        ring.wait(j);
        {
            const uint32_t v = lane < FFB_CL ? cl_pk[par * FFB_CL + lane].val : 0u;
            const uint32_t kk = lane < FFB_CL ? cl_pk[par * FFB_CL + lane].key : KEY_INVALID;
            uint32_t m3, k3;
            warp_argmax(v, kk, m3, k3);
            const uint32_t bal = __ballot_sync(0xffffffffu, lane < FFB_CL && v == m3 && kk == k3);
            oldp = &cl_pk[par * FFB_CL + (__ffs(bal) - 1)];
            if (s.g == 0) idxs[j] = (k3 != KEY_INVALID ? fps_place_key_to_k<2>(k3) : 0) + io.ioff;
        }
    }
    cluster_sync_all();                       // peers may still be storing into this CTA's shared memory
}

int launch_ffps_bucket(int b, int n, int ca, int cb, int m, const float *fa, const float *fb, int *out, const FpsIO &io,
                       cudaStream_t st)
{
    void *args[] = {&n, &ca, &cb, &m, &fa, &fb, &out, (void *)&io};
    return (int)launch_cluster(ffps_bucket_kernel, FFB_CL, b, ffps_bucket_smem(), st, args);
}

}  // namespace ssd3d
