// fps.cu -- farthest point sampling for sm_90a.
//
// Replaces the reference kernels farthestpointsamplingKernel / farthestpointsamplingwithdistKernel
// (/root/reference/lib/utils/tf_ops/sampling/tf_sampling_g.cu:124-178, :181-230).
//
// Design (DESIGN.md "FPS"): FPS is a chain of m-1 dependent rounds, so the kernel is built to
// minimise the latency of ONE round instead of streaming bandwidth:
//   * one thread-block CLUSTER per scene (CL CTAs x 256 threads); every thread keeps its P points
//     and their running min-distance in REGISTERS for the whole kernel -- no global/shared traffic
//     for the distance update (the reference re-reads xyz and read-modify-writes `temp` in global
//     memory every round);
//   * per-round arg-max = two redux.sync per warp -> one 32-byte packet per warp in shared memory
//     -> one packet per CTA pushed to every peer with st.async (DSMEM store + mbarrier complete_tx,
//     a one-way message, no cluster barrier) -> every warp reduces the CL packets redundantly;
//   * the winner's coordinates travel inside the packet, so the next round starts immediately.
//
// Bit-exactness: the reference's result is the arg-max under the order
//     (value desc, k mod 1024 asc, k asc)            [1024-thread strided scan + left-biased tree]
// which is reproduced by reducing the pair (value bits, key) with key = (k mod 1024, k div 1024).
// Distances use the reference's contracted arithmetic: d = fma(dz,dz, fma(dy,dy, dx*dx)).
#include "common.cuh"
#include "fps.cuh"

namespace ssd3d {

constexpr int FPS_T = 256;  // threads per CTA
constexpr int FPS_NW = FPS_T / 32;
// Ownership map: slot i of global thread g (g = cta_rank*256 + tid, TT = CL*256 threads per scene).
// Each thread owns points of one residue class mod 1024 (or 1024/TT classes when TT < 1024), visited
// in ascending key order, so "first strictly greater" inside a thread == smallest key among its maxima.
template <int TT, int P>
struct FpsMap {
    static constexpr int S = TT >= 1024 ? TT / 1024 : 1;  // threads sharing one residue class
    static constexpr int R = TT >= 1024 ? 1 : 1024 / TT;  // residue classes per thread
    static constexpr int J = P / R;
    static_assert(P % R == 0 && J >= 1, "P must be a multiple of the residue classes per thread");
    __device__ static __forceinline__ int k_of(int g, int i)
    {
        const int a = i / J, jj = i % J;
        return (g & 1023) + a * TT + 1024 * ((g >> 10) + S * jj);
    }
    // inverse: (global thread, slot) that own point k
    __device__ static __forceinline__ void owner_of(int k, int &g, int &i)
    {
        const int r = k & 1023, q = k >> 10;
        if (TT >= 1024) { g = r + 1024 * (q % S); i = q / S; }
        else { g = r % TT; i = (r / TT) * J + q; }
    }
};

struct __align__(16) FpsPacket {
    uint32_t val;  // bits of the (non-negative) candidate distance
    uint32_t key;  // fps_key(k); smaller wins ties
    float x, y, z; // coordinates of the candidate (c==3 kernel only)
    uint32_t pad[3];
};
static_assert(sizeof(FpsPacket) == 32, "packet must be two 16-byte pieces");

// ---------------------------------------------------------------------------------------------------
// Shared per-round machinery: given this thread's candidate (best value, slot, key), produce the
// scene-wide winner.  MODE 0: packets carry xyz (c==3); MODE 1: (value,key) only.
// ---------------------------------------------------------------------------------------------------
template <int CL>
struct FpsShared {
    FpsPacket warp_pk[2][FPS_NW];
    FpsPacket cl_pk[2][CL];
    unsigned long long mbar[2];
};

// pf_rows != nullptr (with-distance kernel): while the CTA's candidate travels to the peers, warp 0 prefetches that
// candidate's matrix row into L2 -- the winner of the round is one of the CL candidates, so the row every CTA reads
// next round is (almost always) an L2 hit instead of a DRAM-latency miss on the critical path.
template <int CL, bool WITH_XYZ>
__device__ __forceinline__ void fps_exchange(FpsShared<CL> &sh, int j, uint32_t rank, float best, uint32_t my_key,
                                             float cx, float cy, float cz, uint32_t &win_key, float &ox, float &oy,
                                             float &oz, const float *pf_rows = nullptr, int pf_n = 0)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int par = j & 1;
    const uint32_t u = __float_as_uint(fmaxf(best, 0.0f));
    uint32_t mx, kmin;
    warp_argmax(u, best >= 0.0f ? my_key : KEY_INVALID, mx, kmin);
    {
        const uint32_t bal = __ballot_sync(0xffffffffu, (u == mx) && ((best >= 0.0f ? my_key : KEY_INVALID) == kmin));
        if (lane == __ffs(bal) - 1) {
            uint4 *dst = reinterpret_cast<uint4 *>(&sh.warp_pk[par][warp]);
            dst[0] = make_uint4(mx, kmin, __float_as_uint(cx), __float_as_uint(cy));
            if (WITH_XYZ) dst[1] = make_uint4(__float_as_uint(cz), 0u, 0u, 0u);
        }
    }
    __syncthreads();
    if (CL == 1 || warp == 0) {
        const uint32_t v = lane < FPS_NW ? sh.warp_pk[par][lane].val : 0u;
        const uint32_t kk = lane < FPS_NW ? sh.warp_pk[par][lane].key : KEY_INVALID;
        uint32_t m2, k2;
        warp_argmax(v, kk, m2, k2);
        const uint32_t bal = __ballot_sync(0xffffffffu, lane < FPS_NW && v == m2 && kk == k2);
        const int ww = __ffs(bal) - 1;
        if (CL == 1) {
            win_key = k2;
            if (WITH_XYZ) {
                const uint4 a = reinterpret_cast<const uint4 *>(&sh.warp_pk[par][ww])[0];
                ox = __uint_as_float(a.z); oy = __uint_as_float(a.w);
                oz = sh.warp_pk[par][ww].z;
            }
            return;
        }
        constexpr int PIECES = WITH_XYZ ? 2 : 1;
        if (lane == 0) mbar_arrive_expect_tx(smem_u32(&sh.mbar[par]), CL * PIECES * 16);
        if (lane < PIECES * CL) {
            const int piece = WITH_XYZ ? (lane & 1) : 0;
            const uint32_t peer = WITH_XYZ ? (lane >> 1) : lane;
            const uint4 v4 = reinterpret_cast<const uint4 *>(&sh.warp_pk[par][ww])[piece];
            st_async_v4(mapa(smem_u32(&sh.cl_pk[par][rank]) + piece * 16, peer), mapa(smem_u32(&sh.mbar[par]), peer), v4);
        }
        if (pf_rows != nullptr && k2 != KEY_INVALID) {
            const float *row = pf_rows + (size_t)fps_key_to_k(k2) * pf_n;
            for (int e = lane * 32; e < pf_n; e += 32 * 32)          // one 128-byte line per prefetch
                asm volatile("prefetch.global.L2 [%0];" ::"l"(row + e) : "memory");
        }
    }
    if (CL > 1) {
        mbar_wait_cta(smem_u32(&sh.mbar[par]), ((j - 1) >> 1) & 1);
        const uint32_t v = lane < CL ? sh.cl_pk[par][lane].val : 0u;
        const uint32_t kk = lane < CL ? sh.cl_pk[par][lane].key : KEY_INVALID;
        uint32_t m3, k3;
        warp_argmax(v, kk, m3, k3);
        win_key = k3;
        if (WITH_XYZ) {
            const uint32_t bal = __ballot_sync(0xffffffffu, lane < CL && v == m3 && kk == k3);
            const int wr = __ffs(bal) - 1;
            const uint4 a = reinterpret_cast<const uint4 *>(&sh.cl_pk[par][wr])[0];
            ox = __uint_as_float(a.z); oy = __uint_as_float(a.w);
            oz = sh.cl_pk[par][wr].z;
        }
    }
}

template <int CL>
__device__ __forceinline__ void fps_shared_init(FpsShared<CL> &sh)
{
    if (threadIdx.x == 0) {
        mbar_init(smem_u32(&sh.mbar[0]), 1);
        mbar_init(smem_u32(&sh.mbar[1]), 1);
        fence_mbar_init_cluster();
    }
    __syncthreads();
    if (CL > 1) cluster_sync_all();  // every CTA's barriers exist before any peer st.async targets them
}

// ---------------------------------------------------------------------------------------------------
// D-FPS on xyz (c == 3): points + running distances live in registers.
// ---------------------------------------------------------------------------------------------------
template <int CL, int P>
__global__ void __launch_bounds__(FPS_T, 1)
fps3_cluster_kernel(int n, int m, const float *__restrict__ inp, int *__restrict__ out, const FpsIO io)
{
    using Map = FpsMap<CL * FPS_T, P>;
    extern __shared__ float4 own_pts[];  // [P][FPS_T] xyz of this CTA's points (lookup by the round winner)
    __shared__ FpsShared<CL> sh;

    const int tid = threadIdx.x;
    const uint32_t rank = CL > 1 ? cluster_ctarank() : 0u;
    const int scene = blockIdx.x / CL;
    const int g = (int)rank * FPS_T + tid;
    const float *data = inp + (size_t)scene * io.sa;
    int *idxs = out + (size_t)scene * io.ldo;

    float px[P], py[P], pz[P], td[P];
#pragma unroll
    for (int i = 0; i < P; i++) {
        const int k = Map::k_of(g, i);
        if (k < n) {
            px[i] = data[3 * k]; py[i] = data[3 * k + 1]; pz[i] = data[3 * k + 2];
            td[i] = 1e38f;  // tf_sampling_g.cu:136
        } else {
            px[i] = py[i] = pz[i] = 0.0f;
            td[i] = -1.0f;  // padding slot: can never win (min(d,-1) stays -1, valid values are >= 0)
        }
        own_pts[i * FPS_T + tid] = make_float4(px[i], py[i], pz[i], 0.0f);
    }
    fps_shared_init<CL>(sh);

    float ox = data[0], oy = data[1], oz = data[2];  // first sample is point 0 (:131-133)
    if (g == 0) idxs[0] = io.ioff;

    for (int j = 1; j < m; j++) {
        float best = -1.0f;
        int bi = 0;
#pragma unroll
        for (int i = 0; i < P; i++) {
            const float dx = px[i] - ox, dy = py[i] - oy, dz = pz[i] - oz;
            float d = __fmul_rn(dx, dx);
            d = __fmaf_rn(dy, dy, d);
            d = __fmaf_rn(dz, dz, d);
            const float t = fminf(d, td[i]);
            td[i] = t;
            if (t > best) { best = t; bi = i; }
        }
        const float4 c = own_pts[bi * FPS_T + tid];
        uint32_t wkey;
        fps_exchange<CL, true>(sh, j, rank, best, fps_key(Map::k_of(g, bi)), c.x, c.y, c.z, wkey, ox, oy, oz);
        if (g == 0) idxs[j] = fps_key_to_k(wkey) + io.ioff;
    }
    if (CL > 1) cluster_sync_all();  // peers may still be storing into this CTA's shared memory
}

// ---------------------------------------------------------------------------------------------------
// D-FPS, "direct" variant for scenes whose xyz fit in one CTA's shared memory (n <= ~18k, the 3DSSD sizes):
// every CTA keeps a full copy of the scene's coordinates (one bulk TMA copy), so a packet is just (value, key)
// = 8 bytes and EVERY WARP pushes its candidate straight to all peers -- the intra-CTA reduction stage and its
// barrier disappear; a round is: register update -> 2 redux -> st.async -> mbarrier wait -> 2 redux -> 3 LDS.
// ---------------------------------------------------------------------------------------------------
template <int CL, int P>
__global__ void __launch_bounds__(FPS_T, 1)
fps3_direct_kernel(int n, int m, const float *__restrict__ inp, int *__restrict__ out, const FpsIO io)
{
    using Map = FpsMap<CL * FPS_T, P>;
    constexpr int NSLOT = CL * FPS_NW;                   // packets received per round
    extern __shared__ float4 dyn_smem[];
    float *sxyz = reinterpret_cast<float *>(dyn_smem);   // [n][3] raw copy of the scene
    __shared__ __align__(16) unsigned long long slots[2][NSLOT];
    __shared__ __align__(8) unsigned long long mbar[2], load_bar;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t rank = CL > 1 ? cluster_ctarank() : 0u;
    const int scene = blockIdx.x / CL;
    const int g = (int)rank * FPS_T + tid;
    const float *data = inp + (size_t)scene * io.sa;
    int *idxs = out + (size_t)scene * io.ldo;
    // Resumable: this launch runs rounds [jbeg, jend) of 1..m-1.  A launch that does not start at round 0 reloads the
    // running distances from io.temp and the last winner from the index output; one that stops before m saves them.
    const int jbeg = io.j0 > 1 ? io.j0 : 1, jend = io.j1 < m ? io.j1 : m;
    const bool resume = io.j0 > 0, save = io.j1 < m;
    float *tsave = io.temp + (size_t)scene * n;

    if (tid == 0) {
        mbar_init(smem_u32(&mbar[0]), 1);
        mbar_init(smem_u32(&mbar[1]), 1);
        mbar_init(smem_u32(&load_bar), 1);
        fence_mbar_init_cluster();
        mbar_arrive_expect_tx(smem_u32(&load_bar), (uint32_t)n * 12u);
        bulk_g2s(smem_u32(sxyz), data, (uint32_t)n * 12u, smem_u32(&load_bar));
    }
    __syncthreads();
    mbar_wait_cta(smem_u32(&load_bar), 0);

    float px[P], py[P], pz[P], td[P];
#pragma unroll
    for (int i = 0; i < P; i++) {
        const int k = Map::k_of(g, i);
        if (k < n) {
            px[i] = sxyz[3 * k]; py[i] = sxyz[3 * k + 1]; pz[i] = sxyz[3 * k + 2];
            td[i] = resume ? tsave[k] : 1e38f;
        } else { px[i] = py[i] = pz[i] = 0.0f; td[i] = -1.0f; }
    }
    if (CL > 1) cluster_sync_all();                      // all peers' barriers are initialised

    int old0 = 0;
    if (resume) old0 = idxs[jbeg - 1] - io.ioff;         // written by the previous launch of this scene
    else if (g == 0) idxs[0] = io.ioff;
    float ox = sxyz[3 * old0], oy = sxyz[3 * old0 + 1], oz = sxyz[3 * old0 + 2];

    for (int j = jbeg; j < jend; j++) {
        const int r = j - jbeg + 1;                      // 1-based round of THIS launch: slot parity / barrier phase
        const int par = r & 1;
        if (tid == 0) mbar_arrive_expect_tx(smem_u32(&mbar[par]), NSLOT * 8);
        // ---- distance update of the thread's P points, then their arg-max as a TREE (depth log2 P) instead of a serial
        // "first strictly greater" scan (depth P): the scan's compare + select chain was ~150 of the ~830 cycles of a
        // round.  Ties keep the lower slot (a higher slot wins only when STRICTLY greater), i.e. the scan's answer.
        float tv[P];
        {
            // fp32 pairs: same IEEE operations as d = fma(dz,dz, fma(dy,dy, dx*dx))
            const float2 nox = make_float2(-ox, -ox), noy = make_float2(-oy, -oy), noz = make_float2(-oz, -oz);
#pragma unroll
            for (int i = 0; i + 1 < P; i += 2) {
                const float2 dx = add2_rn(make_float2(px[i], px[i + 1]), nox);
                const float2 dy = add2_rn(make_float2(py[i], py[i + 1]), noy);
                const float2 dz = add2_rn(make_float2(pz[i], pz[i + 1]), noz);
                float2 d = mul2_rn(dx, dx);
                d = fma2_rn(dy, dy, d);
                d = fma2_rn(dz, dz, d);
                td[i] = fminf(d.x, td[i]); td[i + 1] = fminf(d.y, td[i + 1]);
                tv[i] = td[i]; tv[i + 1] = td[i + 1];
            }
            if (P & 1) {
                constexpr int i = P - 1;
                const float dx = px[i] - ox, dy = py[i] - oy, dz = pz[i] - oz;
                float d = __fmul_rn(dx, dx);
                d = __fmaf_rn(dy, dy, d);
                d = __fmaf_rn(dz, dz, d);
                td[i] = fminf(d, td[i]);
                tv[i] = td[i];
            }
        }
        int tk[P];                                       // k of slot i (compile-time offsets from the thread's base)
#pragma unroll
        for (int i = 0; i < P; i++) tk[i] = Map::k_of(g, i);
#pragma unroll
        for (int sdist = 1; sdist < P; sdist *= 2) {
#pragma unroll
            for (int i = 0; i + sdist < P; i += 2 * sdist) {
                const bool up = tv[i + sdist] > tv[i];
                tv[i] = up ? tv[i + sdist] : tv[i];
                tk[i] = up ? tk[i + sdist] : tk[i];
            }
        }
        const float best = tv[0];
        const uint32_t u = __float_as_uint(fmaxf(best, 0.0f));
        uint32_t mx, kmin;
        warp_argmax(u, best >= 0.0f ? fps_key(tk[0]) : KEY_INVALID, mx, kmin);
        if (lane < CL) {
            const unsigned long long pk = ((unsigned long long)mx << 32) | (unsigned long long)kmin;
            st_async_b64(mapa(smem_u32(&slots[par][rank * FPS_NW + warp]), (uint32_t)lane),
                         mapa(smem_u32(&mbar[par]), (uint32_t)lane), pk);
        }
        mbar_wait_cta(smem_u32(&mbar[par]), ((r - 1) >> 1) & 1);
        // reduce the NSLOT packets: value desc, key asc
        unsigned long long a = lane < NSLOT ? slots[par][lane] : 0x00000000ffffffffull;
#pragma unroll
        for (int sidx = 32; sidx < NSLOT; sidx += 32) {
            const unsigned long long b2 = slots[par][lane + sidx];
            const uint32_t av = (uint32_t)(a >> 32), bv = (uint32_t)(b2 >> 32);
            if (bv > av || (bv == av && (uint32_t)b2 < (uint32_t)a)) a = b2;
        }
        uint32_t m3, k3;
        warp_argmax((uint32_t)(a >> 32), (uint32_t)a, m3, k3);
        const int old = fps_key_to_k(k3);
        ox = sxyz[3 * old]; oy = sxyz[3 * old + 1]; oz = sxyz[3 * old + 2];
        if (g == 0) idxs[j] = old + io.ioff;
    }
    if (save) {
#pragma unroll
        for (int i = 0; i < P; i++) {
            const int k = Map::k_of(g, i);
            if (k < n) tsave[k] = td[i];
        }
    }
    if (CL > 1) cluster_sync_all();
}

// ---------------------------------------------------------------------------------------------------
// F-FPS given a precomputed distance matrix (tf_sampling_g.cu:181-230): one coalesced row read per round.
// ---------------------------------------------------------------------------------------------------
template <int CL, int P>
__global__ void __launch_bounds__(FPS_T, 1)
fpsdist_cluster_kernel(int n, int m, const float *__restrict__ dist, int *__restrict__ out, const FpsIO io)
{
    using Map = FpsMap<CL * FPS_T, P>;
    __shared__ FpsShared<CL> sh;
    const int tid = threadIdx.x;
    const uint32_t rank = CL > 1 ? cluster_ctarank() : 0u;
    const int scene = blockIdx.x / CL;
    const int g = (int)rank * FPS_T + tid;
    const float *mat = dist + (size_t)scene * io.sa;
    int *idxs = out + (size_t)scene * io.ldo;

    float td[P];
    int kk[P];
#pragma unroll
    for (int i = 0; i < P; i++) {
        kk[i] = Map::k_of(g, i);
        td[i] = kk[i] < n ? 1e38f : -1.0f;
    }
    fps_shared_init<CL>(sh);
    int old = 0;
    if (g == 0) idxs[0] = io.ioff;
    for (int j = 1; j < m; j++) {
        const float *row = mat + (size_t)old * n;
        float dv[P];
#pragma unroll
        for (int i = 0; i < P; i++) dv[i] = kk[i] < n ? __ldg(row + kk[i]) : 0.0f;
        float best = -1.0f;
        int bi = 0;
#pragma unroll
        for (int i = 0; i < P; i++) {
            const float t = fminf(dv[i], td[i]);
            td[i] = t;
            if (t > best) { best = t; bi = i; }
        }
        uint32_t wkey;
        float ux, uy, uz;
        fps_exchange<CL, false>(sh, j, rank, best, fps_key(Map::k_of(g, bi)), 0.f, 0.f, 0.f, wkey, ux, uy, uz, mat, n);
        old = fps_key_to_k(wkey);
        if (g == 0) idxs[j] = old + io.ioff;
    }
    if (CL > 1) cluster_sync_all();
}

// ---------------------------------------------------------------------------------------------------
// FPS on generic c-dimensional points (the reference kernel's generic path, :146-150), used as the
// matrix-free F-FPS on concat[xyz, features]: the scene's features stay in the cluster's shared memory
// ([c][NL] per CTA), the winner's feature vector is fetched from its owner CTA through DSMEM.
// ---------------------------------------------------------------------------------------------------
template <int CL, int P>
__global__ void __launch_bounds__(FPS_T, 1)
fpsc_cluster_kernel(int n, int c, int m, const float *__restrict__ inp, int *__restrict__ out, const FpsIO io)
{
    using Map = FpsMap<CL * FPS_T, P>;
    constexpr int NL = P * FPS_T;
    constexpr int NLP = NL + 1;  // +1 pitch: conflict-free staging writes, reads stay conflict-free
    extern __shared__ float4 dyn_smem[];
    float *feat = reinterpret_cast<float *>(dyn_smem);  // [c][NLP]
    float *old_f = feat + (size_t)c * NLP;               // [c]
    __shared__ FpsShared<CL> sh;

    const int tid = threadIdx.x;
    const uint32_t rank = CL > 1 ? cluster_ctarank() : 0u;
    const int scene = blockIdx.x / CL;
    const int g = (int)rank * FPS_T + tid;
    const float *data = inp + (size_t)scene * io.sa;
    int *idxs = out + (size_t)scene * io.ldo;

    float td[P];
#pragma unroll
    for (int i = 0; i < P; i++) td[i] = Map::k_of(g, i) < n ? 1e38f : -1.0f;
    // stage features: one warp per point row for coalesced global reads
    for (int s = tid >> 5; s < NL; s += FPS_NW) {
        const int st = s % FPS_T, si = s / FPS_T;
        const int k = Map::k_of((int)rank * FPS_T + st, si);
        for (int l = tid & 31; l < c; l += 32) feat[(size_t)l * NLP + s] = k < n ? data[(size_t)k * c + l] : 0.0f;
    }
    for (int l = tid; l < c; l += FPS_T) old_f[l] = data[l];  // first sample is point 0
    fps_shared_init<CL>(sh);  // contains __syncthreads
    if (g == 0) idxs[0] = io.ioff;

    for (int j = 1; j < m; j++) {
        float d[P];
#pragma unroll
        for (int i = 0; i < P; i++) d[i] = 0.0f;
        for (int l = 0; l < c; l++) {
            const float o = old_f[l];
            const float *fl = feat + (size_t)l * NLP + tid;
#pragma unroll
            for (int i = 0; i < P; i++) {
                const float diff = fl[i * FPS_T] - o;
                d[i] = __fmaf_rn(diff, diff, d[i]);
            }
        }
        float best = -1.0f;
        int bi = 0;
#pragma unroll
        for (int i = 0; i < P; i++) {
            const float t = fminf(d[i], td[i]);
            td[i] = t;
            if (t > best) { best = t; bi = i; }
        }
        uint32_t wkey;
        float ux, uy, uz;
        fps_exchange<CL, false>(sh, j, rank, best, fps_key(Map::k_of(g, bi)), 0.f, 0.f, 0.f, wkey, ux, uy, uz);
        const int old = fps_key_to_k(wkey);
        if (g == 0) idxs[j] = old + io.ioff;
        // fetch the winner's feature vector from its owner CTA (all threads passed the __syncthreads inside
        // fps_exchange, so nobody still reads old_f of this round)
        int og, oi;
        Map::owner_of(old, og, oi);
        const uint32_t orank = (uint32_t)(og / FPS_T);
        const int oslot = oi * FPS_T + (og % FPS_T);
        for (int l = tid; l < c; l += FPS_T) {
            const uint32_t a = smem_u32(feat + (size_t)l * NLP + oslot);
            old_f[l] = CL > 1 ? ld_dsmem_f32(mapa(a, orank)) : feat[(size_t)l * NLP + oslot];
        }
        __syncthreads();
    }
    if (CL > 1) cluster_sync_all();
}

// ---------------------------------------------------------------------------------------------------
// F-FPS without the distance matrix: farthest_point_sample_with_distance(m, calc_square_dist(feat)) evaluated row by
// row, on the fly (layers_util.py:94-96 / :102-104 of the reference build the [B,N,N] matrix with a GEMM and then
// read one row of it per round).  Bit-identical to the matrix route: the value used for point k in the round after
// `old` was picked is exactly sqdist's entry  (sq[old] + sq[k]) - 2 * dot(old, k)  with the pinned fma chains.
//
// Every thread keeps the features of its P points in REGISTERS (P*CP <= 136 values); a copy of the CTA's rows lives
// in shared memory so that warp 0 can attach the CTA candidate's whole feature row (+ its squared norm) to the
// arg-max packet it pushes to the peers with st.async.  After the one mbarrier wait of the round every CTA therefore
// already holds the winner's features locally: no second hop, no global memory, no [B,N,N] tensor (0.5 GB per step
// at layer 2) and no kernel to produce it.
// ---------------------------------------------------------------------------------------------------
template <int CP>
struct __align__(16) FfpsPacket {
    uint32_t val, key;
    float sq;
    uint32_t pad;
    float feat[CP];
};

template <int CL, int P, int CP>
__global__ void __launch_bounds__(FPS_T, 1)
ffps_cluster_kernel(int n, int ca, int cb, int m, const float *__restrict__ fa, const float *__restrict__ fb,
                    int *__restrict__ out, const FpsIO io)
{
    constexpr int TT = CL * FPS_T, NL = P * FPS_T, NP = 1 + CP / 4;   // pieces of 16 bytes per packet
    using Packet = FfpsPacket<CP>;
    extern __shared__ float4 dyn_smem[];
    float *featS = reinterpret_cast<float *>(dyn_smem);               // [NL][CP] rows of this CTA's points
    float *sqS = featS + (size_t)NL * CP;                             // [NL]
    Packet *cl_pk = reinterpret_cast<Packet *>(sqS + NL);             // [2][CL]
    __shared__ uint32_t warp_val[2][FPS_NW], warp_key[2][FPS_NW];
    __shared__ unsigned long long mbar[2];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t rank = CL > 1 ? cluster_ctarank() : 0u;
    const int scene = blockIdx.x / CL;
    const int g = (int)rank * FPS_T + tid;
    const int c = ca + cb;
    const float *A = fa + (size_t)scene * io.sa;
    const float *B = fb + (size_t)scene * io.sb;
    int *idxs = out + (size_t)scene * io.ldo;

    // ---- stage this CTA's rows: local point s = i*256 + t  <->  k = rank*256 + t + i*TT (zero rows beyond n)
    for (int s = warp; s < NL; s += FPS_NW) {
        const int k = (int)rank * FPS_T + (s % FPS_T) + (s / FPS_T) * TT;
        for (int l = lane; l < CP; l += 32) {
            float v = 0.0f;
            if (k < n && l < c) v = l < ca ? __ldg(A + (size_t)k * ca + l) : __ldg(B + (size_t)k * cb + (l - ca));
            featS[(size_t)s * CP + l] = v;
        }
    }
    if (tid == 0) {
        mbar_init(smem_u32(&mbar[0]), 1);
        mbar_init(smem_u32(&mbar[1]), 1);
        fence_mbar_init_cluster();
    }
    __syncthreads();
    // Resumable like fps3_direct_kernel: rounds [jbeg, jend); the running distances travel through io.temp, the last
    // winner is re-read from the index output and its feature row from global memory.
    const int jbeg = io.j0 > 1 ? io.j0 : 1, jend = io.j1 < m ? io.j1 : m;
    const bool resume = io.j0 > 0, save = io.j1 < m;
    float *tsave = io.temp + (size_t)scene * n;
    float f[P][CP], td[P], sq[P];
    uint32_t key[P];
#pragma unroll
    for (int i = 0; i < P; i++) {
        const int k = g + i * TT;
        const float4 *row = reinterpret_cast<const float4 *>(featS + (size_t)(i * FPS_T + tid) * CP);
        float s2 = 0.0f;
#pragma unroll
        for (int l4 = 0; l4 < CP / 4; l4++) {
            const float4 v = row[l4];
            f[i][4 * l4 + 0] = v.x; f[i][4 * l4 + 1] = v.y; f[i][4 * l4 + 2] = v.z; f[i][4 * l4 + 3] = v.w;
        }
#pragma unroll
        for (int l = 0; l < CP; l++) s2 = __fmaf_rn(f[i][l], f[i][l], s2);     // sqdist's squared-norm chain
        sq[i] = s2;
        sqS[i * FPS_T + tid] = s2;
        td[i] = k < n ? (resume ? tsave[k] : 1e38f) : -1.0f;
        key[i] = fps_key(k);
    }
    // the point picked last (point 0 at the start of the sampling): its row is read from global memory by every CTA
    {
        const int old0 = resume ? idxs[jbeg - 1] - io.ioff : 0;
        Packet &p0 = cl_pk[0];
        for (int l = tid; l < CP; l += FPS_T) {
            float v = 0.0f;
            if (l < c) v = l < ca ? __ldg(A + (size_t)old0 * ca + l) : __ldg(B + (size_t)old0 * cb + (l - ca));
            p0.feat[l] = v;
        }
        __syncthreads();
        if (tid == 0) {
            float s2 = 0.0f;
            for (int l = 0; l < CP; l++) s2 = __fmaf_rn(p0.feat[l], p0.feat[l], s2);
            p0.sq = s2;
        }
    }
    __syncthreads();
    if (CL > 1) cluster_sync_all();       // every CTA's barriers exist before any peer st.async targets them
    if (g == 0 && !resume) idxs[0] = io.ioff;

    const Packet *oldp = &cl_pk[0];
    for (int j = jbeg; j < jend; j++) {
        const int r = j - jbeg + 1;       // 1-based round of THIS launch: buffer parity / barrier phase
        const int par = r & 1;
        // ---- row `old` of the distance matrix for this thread's points
        float dot[P];
#pragma unroll
        for (int i = 0; i < P; i++) dot[i] = 0.0f;
        const float4 *of4 = reinterpret_cast<const float4 *>(oldp->feat);
#pragma unroll
        for (int l4 = 0; l4 < CP / 4; l4++) {
            const float4 o = of4[l4];
#pragma unroll
            for (int i = 0; i < P; i++) {
                dot[i] = __fmaf_rn(o.x, f[i][4 * l4 + 0], dot[i]);
                dot[i] = __fmaf_rn(o.y, f[i][4 * l4 + 1], dot[i]);
                dot[i] = __fmaf_rn(o.z, f[i][4 * l4 + 2], dot[i]);
                dot[i] = __fmaf_rn(o.w, f[i][4 * l4 + 3], dot[i]);
            }
        }
        const float so = oldp->sq;
        float best = -1.0f;
        uint32_t bkey = KEY_INVALID;
#pragma unroll
        for (int i = 0; i < P; i++) {
            const float d = __fsub_rn(__fadd_rn(so, sq[i]), __fmul_rn(2.0f, dot[i]));
            const float t = fminf(d, td[i]);
            td[i] = t;
            if (t > best || (t == best && key[i] < bkey)) { best = t; bkey = key[i]; }
        }
        // ---- CTA candidate
        const uint32_t u = __float_as_uint(fmaxf(best, 0.0f));
        uint32_t mx, kmin;
        warp_argmax(u, best >= 0.0f ? bkey : KEY_INVALID, mx, kmin);
        if (lane == 0) { warp_val[par][warp] = mx; warp_key[par][warp] = kmin; }
        __syncthreads();
        uint32_t win_key;
        {
            // every warp reduces the 8 warp candidates redundantly; warp w then pushes the CTA candidate's packet
            // (header + feature row, one 16-byte piece per lane) to peer w -- no serial section in one warp
            const uint32_t v = lane < FPS_NW ? warp_val[par][lane] : 0u;
            const uint32_t kk = lane < FPS_NW ? warp_key[par][lane] : KEY_INVALID;
            uint32_t m2, k2;
            warp_argmax(v, kk, m2, k2);
            // the candidate's row in this CTA's shared memory (k2 == KEY_INVALID: nothing valid left, send row 0)
            const int kc = k2 != KEY_INVALID ? fps_key_to_k(k2) : (int)rank * FPS_T;
            const int ls = ((kc - (int)rank * FPS_T) / TT) * FPS_T + ((kc - (int)rank * FPS_T) % TT);
            const float4 *crow = reinterpret_cast<const float4 *>(featS + (size_t)ls * CP);
            if (CL == 1) {
                if (warp == 0) {
                    Packet &dst = cl_pk[par];
                    for (int e = lane; e < NP; e += 32) {
                        const float4 v4 = e == 0 ? make_float4(__uint_as_float(m2), __uint_as_float(k2), sqS[ls], 0.0f) : crow[e - 1];
                        reinterpret_cast<float4 *>(&dst)[e] = v4;
                    }
                }
            } else {
                if (tid == 0) mbar_arrive_expect_tx(smem_u32(&mbar[par]), CL * NP * 16);
                for (int peer = warp; peer < CL; peer += FPS_NW) {
                    const uint32_t dst = mapa(smem_u32(&cl_pk[par * CL + rank]), (uint32_t)peer);
                    const uint32_t dbar = mapa(smem_u32(&mbar[par]), (uint32_t)peer);
                    for (int piece = lane; piece < NP; piece += 32) {
                        const float4 v4 = piece == 0 ? make_float4(__uint_as_float(m2), __uint_as_float(k2), sqS[ls], 0.0f) : crow[piece - 1];
                        st_async_v4(dst + piece * 16, dbar,
                                    make_uint4(__float_as_uint(v4.x), __float_as_uint(v4.y), __float_as_uint(v4.z), __float_as_uint(v4.w)));
                    }
                }
            }
            win_key = k2;
        }
        if (CL == 1) {
            __syncthreads();
            oldp = &cl_pk[par];
            win_key = oldp->key;
        } else {
            mbar_wait_cta(smem_u32(&mbar[par]), ((r - 1) >> 1) & 1);
            const uint32_t v = lane < CL ? cl_pk[par * CL + lane].val : 0u;
            const uint32_t kk = lane < CL ? cl_pk[par * CL + lane].key : KEY_INVALID;
            uint32_t m3, k3;
            warp_argmax(v, kk, m3, k3);
            const uint32_t bal = __ballot_sync(0xffffffffu, lane < CL && v == m3 && kk == k3);
            oldp = &cl_pk[par * CL + (__ffs(bal) - 1)];
            win_key = k3;
        }
        if (g == 0) idxs[j] = (win_key != KEY_INVALID ? fps_key_to_k(win_key) : 0) + io.ioff;
    }
    if (save) {
#pragma unroll
        for (int i = 0; i < P; i++) {
            const int k = g + i * TT;
            if (k < n) tsave[k] = td[i];
        }
    }
    if (CL > 1) cluster_sync_all();
}

// ---------------------------------------------------------------------------------------------------
// Fallback for shapes the on-chip kernels do not cover (very large n or c): one 1024-thread CTA per
// scene, running distances in the caller's `temp` like the reference, warp-redux arg-max.
// ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024, 1)
fps_fallback_kernel(int n, int c, int m, const float *__restrict__ inp, const float *__restrict__ dist,
                    float *__restrict__ temp, int *__restrict__ out, const FpsIO io)
{
    __shared__ uint32_t s_val[32], s_key[32];
    __shared__ int s_old;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int scene = blockIdx.x;
    const float *data = inp ? inp + (size_t)scene * io.sa : nullptr;
    const float *mat = dist ? dist + (size_t)scene * io.sa : nullptr;
    float *td = temp + (size_t)scene * n;
    int *idxs = out + (size_t)scene * io.ldo;
    for (int k = tid; k < n; k += 1024) td[k] = 1e38f;
    if (tid == 0) idxs[0] = io.ioff;
    int old = 0;
    __syncthreads();
    for (int j = 1; j < m; j++) {
        float best = -1.0f;
        int bk = 0;
        for (int k = tid; k < n; k += 1024) {
            float d;
            if (mat) d = mat[(size_t)old * n + k];
            else {
                d = 0.0f;
                for (int l = 0; l < c; l++) {
                    const float diff = data[(size_t)k * c + l] - data[(size_t)old * c + l];
                    d = __fmaf_rn(diff, diff, d);
                }
            }
            const float t = fminf(d, td[k]);
            td[k] = t;
            if (t > best) { best = t; bk = k; }
        }
        const uint32_t u = __float_as_uint(fmaxf(best, 0.0f));
        const uint32_t key = best >= 0.0f ? fps_key(bk) : KEY_INVALID;
        uint32_t mx, kmin;
        warp_argmax(u, key, mx, kmin);
        if (lane == 0) { s_val[warp] = mx; s_key[warp] = kmin; }
        __syncthreads();
        if (warp == 0) {
            uint32_t m2, k2;
            warp_argmax(s_val[lane], s_key[lane], m2, k2);
            if (lane == 0) { s_old = fps_key_to_k(k2); idxs[j] = s_old + io.ioff; }
        }
        __syncthreads();
        old = s_old;
    }
}

// ---------------------------------------------------------------------------------------------------
// Launch logic
// ---------------------------------------------------------------------------------------------------
template <typename K>
static cudaError_t launch_cluster(K kernel, int cl, int b, size_t dyn_smem, cudaStream_t stream, void **args)
{
    cudaError_t e = cudaFuncSetAttribute((const void *)kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn_smem);
    if (e != cudaSuccess) return e;
    if (cl > 8) {
        e = cudaFuncSetAttribute((const void *)kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
        if (e != cudaSuccess) return e;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(b * cl));
    cfg.blockDim = dim3(FPS_T);
    cfg.dynamicSmemBytes = dyn_smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)cl;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelExC(&cfg, (const void *)kernel, args);
}

// smallest power of two P >= need with P >= residue classes per thread
static int pick_p(int n, int cl)
{
    const int tt = cl * FPS_T;
    const int r = tt >= 1024 ? 1 : 1024 / tt;
    int need = (n + tt - 1) / tt;
    // a residue class holds ceil(n/1024) points; slots per class J = P/R must cover them
    const int per_class = (n + 1023) / 1024;
    const int s = tt >= 1024 ? tt / 1024 : 1;
    const int j = (per_class + s - 1) / s;
    need = r * j;
    int p = r;
    while (p < need) p *= 2;
    return p;
}

// Cluster-size request of one call (the `cluster` argument of the *_ex entry points): 0 = heuristic, > 0 = exactly
// that many CTAs per scene, < 0 = heuristic capped at -cluster (throughput mode: FPS is latency-bound, so fewer SMs
// per scene cost little time and free SMs for work running concurrently).
static int cap_cl(int cl, int n, int hint)
{
    if (hint < 0)
        while (cl > -hint && cl > 1 && (n + (cl / 2) * FPS_T - 1) / ((cl / 2) * FPS_T) <= 16) cl /= 2;
    return cl;
}

static int pick_cl_xyz(int n, int hint)
{
    if (hint > 0) return hint;
    int cl;
    if (n <= 1024) cl = 1;
    else if (n <= 2048) cl = 2;
    else if (n <= 4096) cl = 4;
    else if (n <= 32768) cl = 8;
    else cl = 16;
    return cap_cl(cl, n, hint);
}

}  // namespace ssd3d

using namespace ssd3d;

// The P values legal for a cluster size are the multiples of R = max(1, 1024/(CL*256)):
//   CL=1 -> P in {4,8,16}; CL=2 -> {2,4,8,16}; CL>=4 -> {1,2,4,8,16}.
#define SSD3D_FPS_SWITCH(KERNEL, SMEM_OF_P)                                                               \
    do {                                                                                                  \
        cudaError_t e = cudaErrorInvalidValue;                                                            \
        const int p = pick_p(n, cl);                                                                      \
        const size_t smem = (SMEM_OF_P);                                                                  \
        if (cl == 1) {                                                                                    \
            if (p == 4) e = launch_cluster(KERNEL<1, 4>, 1, b, smem, st, args);                           \
            else if (p == 8) e = launch_cluster(KERNEL<1, 8>, 1, b, smem, st, args);                      \
            else if (p == 16) e = launch_cluster(KERNEL<1, 16>, 1, b, smem, st, args);                    \
            else return -100;                                                                             \
        } else if (cl == 2) {                                                                             \
            if (p == 2) e = launch_cluster(KERNEL<2, 2>, 2, b, smem, st, args);                           \
            else if (p == 4) e = launch_cluster(KERNEL<2, 4>, 2, b, smem, st, args);                      \
            else if (p == 8) e = launch_cluster(KERNEL<2, 8>, 2, b, smem, st, args);                      \
            else if (p == 16) e = launch_cluster(KERNEL<2, 16>, 2, b, smem, st, args);                    \
            else return -100;                                                                             \
        } else if (cl == 4) {                                                                             \
            if (p == 1) e = launch_cluster(KERNEL<4, 1>, 4, b, smem, st, args);                           \
            else if (p == 2) e = launch_cluster(KERNEL<4, 2>, 4, b, smem, st, args);                      \
            else if (p == 4) e = launch_cluster(KERNEL<4, 4>, 4, b, smem, st, args);                      \
            else if (p == 8) e = launch_cluster(KERNEL<4, 8>, 4, b, smem, st, args);                      \
            else if (p == 16) e = launch_cluster(KERNEL<4, 16>, 4, b, smem, st, args);                    \
            else return -100;                                                                             \
        } else if (cl == 8) {                                                                             \
            if (p == 1) e = launch_cluster(KERNEL<8, 1>, 8, b, smem, st, args);                           \
            else if (p == 2) e = launch_cluster(KERNEL<8, 2>, 8, b, smem, st, args);                      \
            else if (p == 4) e = launch_cluster(KERNEL<8, 4>, 8, b, smem, st, args);                      \
            else if (p == 8) e = launch_cluster(KERNEL<8, 8>, 8, b, smem, st, args);                      \
            else if (p == 16) e = launch_cluster(KERNEL<8, 16>, 8, b, smem, st, args);                    \
            else return -100;                                                                             \
        } else if (cl == 16) {                                                                            \
            if (p == 1) e = launch_cluster(KERNEL<16, 1>, 16, b, smem, st, args);                         \
            else if (p == 2) e = launch_cluster(KERNEL<16, 2>, 16, b, smem, st, args);                    \
            else if (p == 4) e = launch_cluster(KERNEL<16, 4>, 16, b, smem, st, args);                    \
            else if (p == 8) e = launch_cluster(KERNEL<16, 8>, 16, b, smem, st, args);                    \
            else if (p == 16) e = launch_cluster(KERNEL<16, 16>, 16, b, smem, st, args);                  \
            else return -100;                                                                             \
        } else return -100;                                                                               \
        return (int)e;                                                                                    \
    } while (0)

static int launch_fps3(int b, int n, int m, int cl, const float *inp, int *out, const FpsIO &io, cudaStream_t st)
{
    void *args[] = {&n, &m, (void *)&inp, (void *)&out, (void *)&io};
    SSD3D_FPS_SWITCH(fps3_cluster_kernel, (size_t)p * FPS_T * sizeof(float4));
}
static int launch_fps3_direct(int b, int n, int m, int cl, const float *inp, int *out, const FpsIO &io, cudaStream_t st)
{
    void *args[] = {&n, &m, (void *)&inp, (void *)&out, (void *)&io};
    SSD3D_FPS_SWITCH(fps3_direct_kernel, (size_t)n * 12 + 16);
}
static int launch_fpsdist(int b, int n, int m, int cl, const float *dist, int *out, const FpsIO &io, cudaStream_t st)
{
    void *args[] = {&n, &m, (void *)&dist, (void *)&out, (void *)&io};
    SSD3D_FPS_SWITCH(fpsdist_cluster_kernel, (size_t)0);
}
static int launch_fpsc(int b, int n, int c, int m, int cl, const float *inp, int *out, const FpsIO &io, cudaStream_t st)
{
    void *args[] = {&n, &c, &m, (void *)&inp, (void *)&out, (void *)&io};
    SSD3D_FPS_SWITCH(fpsc_cluster_kernel, ((size_t)c * (p * FPS_T + 1) + c) * sizeof(float) + 16);
}

// cluster size for the generic-c kernel: smallest CL whose per-CTA feature slab fits in shared memory
static int pick_cl_generic(int n, int c, int hint)
{
    if (hint > 0) return hint;
    const size_t budget = 200 * 1024;
    for (int cl = 1; cl <= 16; cl *= 2) {
        const int p = pick_p(n, cl);
        if (p > 16) continue;
        if (((size_t)c * (p * FPS_T + 1) + c) * sizeof(float) + 16 <= budget && (cl >= 8 || n <= cl * 1024)) return cl;
    }
    for (int cl = 1; cl <= 16; cl *= 2) {
        const int p = pick_p(n, cl);
        if (p <= 16 && ((size_t)c * (p * FPS_T + 1) + c) * sizeof(float) + 16 <= budget) return cl;
    }
    return 0;
}

extern "C" int ssd3d_fps_needs_temp(int n, int c)
{
    if (c == 3) return pick_p(n, 16) > 16;
    return pick_cl_generic(n, c, 0) == 0;
}

// (c == 3) does the resumable direct kernel cover n?  It needs the scene resident in one CTA's shared memory.
static bool fps3_direct_fits(int n, int cl, const float *inp, long long sa)
{
    return cl >= 2 && (size_t)n * 12 + 16 <= 200 * 1024 && (n % 4) == 0 &&
           (reinterpret_cast<uintptr_t>(inp) & 15u) == 0 && (sa % 4) == 0 && pick_p(n, cl) <= 16;
}

// floats of `temp` per scene a partial range of rounds needs: the running distances, plus (bucket kernel) the permutation
extern "C" long ssd3d_fps_temp_elems(int n, int c, int m, int flags)
{
    if (n <= 0) return 0;
    if (c == 3 && fps3_bucket_applies(n, m, nullptr, 0, flags)) return 2L * n;
    return n;
}

extern "C" int ssd3d_fps_supports_rounds(int n, int c)
{
    if (c != 3) return 0;
    int cl = pick_cl_xyz(n, 0);
    while (cl < 16 && pick_p(n, cl) > 16) cl *= 2;
    return cl >= 2 && (size_t)n * 12 + 16 <= 200 * 1024 && (n % 4) == 0 && pick_p(n, cl) <= 16;
}

extern "C" int ssd3d_farthest_point_sample_ex(int b, int n, int c, int m, const float *inp, long long in_stride,
                                              float *temp, int *out, int ldo, int idx_offset, int j0, int j1,
                                              int cluster, int flags, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && n > 0 && c > 0 && m >= 0, "farthest_point_sample: bad shape b=%d n=%d c=%d m=%d", b, n, c, m);
    SSD3D_REQUIRE(ldo >= m && in_stride >= (long long)n * c, "farthest_point_sample: strides smaller than a row (ldo=%d, in_stride=%lld)", ldo, in_stride);
    SSD3D_REQUIRE(0 <= j0 && j0 <= j1 && j1 <= m, "farthest_point_sample: rounds [%d,%d) outside [0,%d]", j0, j1, m);
    SSD3D_REQUIRE(cluster == 0 || cluster == 1 || cluster == 2 || cluster == 4 || cluster == 8 || cluster == 16 ||
                  cluster == -1 || cluster == -2 || cluster == -4 || cluster == -8 || cluster == -16,
                  "farthest_point_sample: cluster must be 0, +-1, +-2, +-4, +-8 or +-16, got %d", cluster);
    if (b == 0 || m == 0 || j0 == j1) return 0;  // tf_sampling_g.cu:126-127
    SSD3D_REQUIRE(inp && out, "farthest_point_sample: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const bool partial = j0 > 0 || j1 < m;
    FpsIO io = {in_stride, 0, ldo, idx_offset, j0, j1, temp};
    int rc = -100;
    if (c == 3 && fps3_bucket_applies(n, m, inp, in_stride, flags)) {
        // large scenes: one CTA per scene with spatial pruning (fps_bucket.cu); `cluster` does not apply
        SSD3D_REQUIRE(!partial || temp != nullptr, "farthest_point_sample: a partial range of rounds carries its state in temp[b, 2n] "
                      "(ssd3d_fps_temp_elems)");
        rc = launch_fps3_bucket(b, n, m, inp, out, io, st);
    } else if (c == 3) {
        int cl = pick_cl_xyz(n, cluster);
        while (cl < 16 && pick_p(n, cl) > 16) cl *= 2;
        // direct variant: whole scene resident in every CTA (bulk copy needs 16-byte aligned source and size)
        const bool direct_ok = (flags & 1) == 0 && fps3_direct_fits(n, cl, inp, in_stride);
        if (partial) {
            SSD3D_REQUIRE(direct_ok, "farthest_point_sample: a partial range of rounds needs the resident-scene kernel "
                          "(c == 3, n %% 4 == 0, n <= 17000, 16-byte aligned input); see ssd3d_fps_supports_rounds");
            SSD3D_REQUIRE(temp != nullptr, "farthest_point_sample: a partial range of rounds carries its state in temp[b,n]");
        }
        if (direct_ok) rc = launch_fps3_direct(b, n, m, cl, inp, out, io, st);
        else if (pick_p(n, cl) <= 16) rc = launch_fps3(b, n, m, cl, inp, out, io, st);
    } else {
        SSD3D_REQUIRE(!partial, "farthest_point_sample: a partial range of rounds is only built for c == 3");
        const int cl = pick_cl_generic(n, c, cluster);
        if (cl > 0) rc = launch_fpsc(b, n, c, m, cl, inp, out, io, st);
    }
    if (rc == -100) {
        SSD3D_REQUIRE(temp != nullptr, "farthest_point_sample: n=%d c=%d needs the temp[b,n] workspace", n, c);
        fps_fallback_kernel<<<b, 1024, 0, st>>>(n, c, m, inp, nullptr, temp, out, io);
        SSD3D_LAUNCH_CHECK("fps_fallback_kernel");
    }
    return cuda_status((cudaError_t)rc, "farthest_point_sample launch");
}

extern "C" int ssd3d_farthest_point_sample(int b, int n, int c, int m, const float *inp, float *temp, int *out,
                                           ssd3d_stream_t stream)
{
    return ssd3d_farthest_point_sample_ex(b, n, c, m, inp, (long long)n * c, temp, out, m, 0, 0, m, 0, 0, stream);
}

extern "C" int ssd3d_farthest_point_sample_with_distance_ex(int b, int n, int m, const float *dist, float *temp,
                                                            int *out, int ldo, int idx_offset, int cluster,
                                                            ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && n > 0 && m >= 0, "farthest_point_sample_with_distance: bad shape b=%d n=%d m=%d", b, n, m);
    SSD3D_REQUIRE(ldo >= m, "farthest_point_sample_with_distance: ldo=%d smaller than m=%d", ldo, m);
    if (b == 0 || m == 0) return 0;
    SSD3D_REQUIRE(dist && out, "farthest_point_sample_with_distance: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    FpsIO io = {(long long)n * n, 0, ldo, idx_offset, 0, m, nullptr};
    // the per-round row read is a DRAM-latency-bound gather: more CTAs per scene = more loads in flight
    int cl = cluster > 0 ? cluster : cap_cl(n <= 1024 ? 1 : (n <= 2048 ? 4 : 8), n, cluster);
    while (cl < 16 && pick_p(n, cl) > 16) cl *= 2;
    if (pick_p(n, cl) <= 16) return cuda_status((cudaError_t)launch_fpsdist(b, n, m, cl, dist, out, io, st), "fpsdist launch");
    SSD3D_REQUIRE(temp != nullptr, "farthest_point_sample_with_distance: n=%d needs the temp[b,n] workspace", n);
    fps_fallback_kernel<<<b, 1024, 0, st>>>(n, 0, m, nullptr, dist, temp, out, io);
    SSD3D_LAUNCH_CHECK("fps_fallback_kernel");
}

extern "C" int ssd3d_farthest_point_sample_with_distance(int b, int n, int m, const float *dist, float *temp,
                                                         int *out, ssd3d_stream_t stream)
{
    return ssd3d_farthest_point_sample_with_distance_ex(b, n, m, dist, temp, out, m, 0, 0, stream);
}

// ---- matrix-free F-FPS dispatch: CP = 68 (P = 2 points per thread) or 132 (P = 1); smallest cluster that holds n
template <int CL, int P, int CP>
static int launch_ffps_t(int b, int n, int ca, int cb, int m, const float *fa, const float *fb, int *out, const FpsIO &io,
                         cudaStream_t st)
{
    const size_t smem = (size_t)P * FPS_T * CP * 4 + (size_t)P * FPS_T * 4 + (size_t)2 * CL * sizeof(FfpsPacket<CP>);
    void *args[] = { &n, &ca, &cb, &m, &fa, &fb, &out, (void *)&io };
    return (int)launch_cluster(ffps_cluster_kernel<CL, P, CP>, CL, b, smem, st, args);
}
static int ffps_cluster_for(int n, int c)
{
    const int per_cta = c <= 68 ? 2 * FPS_T : (c <= 132 ? FPS_T : 0);
    if (per_cta == 0) return 0;
    for (int cl = 1; cl <= 8; cl *= 2)
        if (n <= cl * per_cta) return cl;
    return 0;
}

// 1 when the matrix-free F-FPS kernel covers (n points, c = channels of the concatenated feature), else 0.
extern "C" int ssd3d_ffps_supported(int n, int c) { return n > 0 && c > 0 && ffps_cluster_for(n, c) > 0 ? 1 : 0; }

// farthest_point_sample_with_distance(m, calc_square_dist(concat[fa, fb])) without the [b,n,n] matrix; same indices.
extern "C" int ssd3d_farthest_point_sample_features_ex(int b, int n, int ca, int cb, int m, const float *fa,
                                                       long long fa_stride, const float *fb, long long fb_stride,
                                                       float *temp, int *out, int ldo, int idx_offset, int j0, int j1,
                                                       ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(0 <= j0 && j0 <= j1 && j1 <= m, "farthest_point_sample_features: rounds [%d,%d) outside [0,%d]", j0, j1, m);
    SSD3D_REQUIRE((j0 == 0 && j1 == m) || temp != nullptr, "farthest_point_sample_features: a partial range of rounds carries its state in temp[b,n]");
    if (j0 == j1) return 0;
    SSD3D_REQUIRE(b >= 0 && n > 0 && m >= 0 && ca > 0 && cb >= 0, "farthest_point_sample_features: bad shape b=%d n=%d m=%d c=%d+%d", b, n, m, ca, cb);
    SSD3D_REQUIRE(ldo >= m && fa_stride >= (long long)n * ca && fb_stride >= (long long)n * cb,
                  "farthest_point_sample_features: strides smaller than a row");
    if (b == 0 || m == 0) return 0;
    SSD3D_REQUIRE(fa && out && (fb || cb == 0), "farthest_point_sample_features: null pointer");
    const int c = ca + cb;
    const int cl = ffps_cluster_for(n, c);
    if (cl == 0) {
        set_error("farthest_point_sample_features: n=%d c=%d not covered (use calc_square_dist + farthest_point_sample_with_distance)", n, c);
        return SSD3D_ERR_UNSUPPORTED;
    }
    cudaStream_t st = (cudaStream_t)stream;
    const FpsIO io = {fa_stride, fb_stride, ldo, idx_offset, j0, j1, temp};
    int rc;
    if (c <= 68) {
        rc = cl == 1 ? launch_ffps_t<1, 2, 68>(b, n, ca, cb, m, fa, fb, out, io, st)
           : cl == 2 ? launch_ffps_t<2, 2, 68>(b, n, ca, cb, m, fa, fb, out, io, st)
           : cl == 4 ? launch_ffps_t<4, 2, 68>(b, n, ca, cb, m, fa, fb, out, io, st)
                     : launch_ffps_t<8, 2, 68>(b, n, ca, cb, m, fa, fb, out, io, st);
    } else {
        rc = cl == 1 ? launch_ffps_t<1, 1, 132>(b, n, ca, cb, m, fa, fb, out, io, st)
           : cl == 2 ? launch_ffps_t<2, 1, 132>(b, n, ca, cb, m, fa, fb, out, io, st)
           : cl == 4 ? launch_ffps_t<4, 1, 132>(b, n, ca, cb, m, fa, fb, out, io, st)
                     : launch_ffps_t<8, 1, 132>(b, n, ca, cb, m, fa, fb, out, io, st);
    }
    return cuda_status((cudaError_t)rc, "ffps launch");
}

extern "C" int ssd3d_farthest_point_sample_features(int b, int n, int ca, int cb, int m, const float *fa, const float *fb,
                                                    int *out, ssd3d_stream_t stream)
{
    return ssd3d_farthest_point_sample_features_ex(b, n, ca, cb, m, fa, (long long)n * ca, fb, (long long)n * cb, nullptr, out,
                                                   m, 0, 0, m, stream);
}
