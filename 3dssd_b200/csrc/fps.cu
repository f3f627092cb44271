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
    FpsRing ring;
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
    const uint2 cd = fps_candidate(best, my_key);
    uint32_t mx, kmin;
    warp_argmax(cd.x, cd.y, mx, kmin);
    {
        const uint32_t bal = __ballot_sync(0xffffffffu, cd.x == mx && cd.y == kmin);
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
        if (lane == 0) sh.ring.expect(j, CL * PIECES * 16);
        if (lane < PIECES * CL) {
            const int piece = WITH_XYZ ? (lane & 1) : 0;
            const uint32_t peer = WITH_XYZ ? (lane >> 1) : lane;
            const uint4 v4 = reinterpret_cast<const uint4 *>(&sh.warp_pk[par][ww])[piece];
            st_async_v4(mapa(smem_u32(&sh.cl_pk[par][rank]) + piece * 16, peer), mapa(sh.ring.at(j), peer), v4);
        }
        if (pf_rows != nullptr && k2 != KEY_INVALID) {
            const float *row = pf_rows + (size_t)fps_key_to_k(k2) * pf_n;
            for (int e = lane * 32; e < pf_n; e += 32 * 32)          // one 128-byte line per prefetch
                asm volatile("prefetch.global.L2 [%0];" ::"l"(row + e) : "memory");
        }
    }
    if (CL > 1) {
        sh.ring.wait(j);
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
    const FpsScene<CL> s;
    const float *data = s.in(inp, io.sa);
    int *idxs = s.row(out, io);

    float px[P], py[P], pz[P], td[P];
#pragma unroll
    for (int i = 0; i < P; i++) {
        const int k = Map::k_of(s.g, i);
        if (k < n) {
            px[i] = data[3 * k]; py[i] = data[3 * k + 1]; pz[i] = data[3 * k + 2];
            td[i] = 1e38f;  // tf_sampling_g.cu:136
        } else {
            px[i] = py[i] = pz[i] = 0.0f;
            td[i] = -1.0f;  // padding slot: can never win (min(d,-1) stays -1, valid values are >= 0)
        }
        own_pts[i * FPS_T + s.tid] = make_float4(px[i], py[i], pz[i], 0.0f);
    }
    sh.ring.template start<CL>();

    float ox = data[0], oy = data[1], oz = data[2];  // first sample is point 0 (:131-133)
    if (s.g == 0) idxs[0] = io.ioff;

    for (int j = 1; j < m; j++) {
        FpsScan scan;
#pragma unroll
        for (int i = 0; i < P; i++) {
            td[i] = fminf(fps_d2(px[i] - ox, py[i] - oy, pz[i] - oz), td[i]);
            scan.see(td[i], i);
        }
        const float4 c = own_pts[scan.at * FPS_T + s.tid];
        uint32_t wkey;
        fps_exchange<CL, true>(sh, j, s.rank, scan.best, fps_key(Map::k_of(s.g, scan.at)), c.x, c.y, c.z, wkey, ox, oy, oz);
        if (s.g == 0) idxs[j] = fps_key_to_k(wkey) + io.ioff;
    }
    if (CL > 1) cluster_sync_all();  // peers may still be storing into this CTA's shared memory
}

// ---------------------------------------------------------------------------------------------------
// D-FPS, "direct" variant for scenes whose xyz fit in one CTA's shared memory (n <= ~18k, the 3DSSD sizes):
// every CTA keeps a full copy of the scene's coordinates (one bulk TMA copy), so a packet is just (value, key)
// = 8 bytes and EVERY WARP pushes its candidate straight to all peers -- the intra-CTA reduction stage and its
// barrier disappear; a round is: register update -> 2 redux -> st.async -> mbarrier wait -> 2 redux -> 3 LDS.
// Resumable (FpsRounds): the running distances travel through temp[b, n].
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
    __shared__ FpsRing ring;
    __shared__ __align__(8) unsigned long long load_bar;

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const FpsScene<CL> s;
    const FpsRounds rounds(io, m, s.scene, out, n);

    if (s.tid == 0) {
        mbar_init(smem_u32(&load_bar), 1);
        ring.init();
        mbar_arrive_expect_tx(smem_u32(&load_bar), (uint32_t)n * 12u);
        bulk_g2s(smem_u32(sxyz), s.in(inp, io.sa), (uint32_t)n * 12u, smem_u32(&load_bar));
    }
    __syncthreads();
    mbar_wait_cta(smem_u32(&load_bar), 0);

    float px[P], py[P], pz[P], td[P];
#pragma unroll
    for (int i = 0; i < P; i++) {
        const int k = Map::k_of(s.g, i);
        if (k < n) { px[i] = sxyz[3 * k]; py[i] = sxyz[3 * k + 1]; pz[i] = sxyz[3 * k + 2]; }
        else { px[i] = py[i] = pz[i] = 0.0f; }
        td[i] = rounds.start(k, k < n);
    }
    if (CL > 1) cluster_sync_all();                      // all peers' barriers are initialised

    const int old0 = rounds.first(s.g == 0);
    float ox = sxyz[3 * old0], oy = sxyz[3 * old0 + 1], oz = sxyz[3 * old0 + 2];

    for (int j = rounds.jbeg; j < rounds.jend; j++) {
        const int r = j - rounds.jbeg + 1;               // round of THIS launch: slot parity / barrier phase
        const int par = r & 1;
        if (s.tid == 0) ring.expect(r, NSLOT * 8);
        // ---- distance update of the thread's P points, then their arg-max as a TREE (depth log2 P) instead of a serial
        // scan (depth P): the scan's compare + select chain was ~150 of the ~830 cycles of a round.
        float tv[P];
        {
            const float2 nox = make_float2(-ox, -ox), noy = make_float2(-oy, -oy), noz = make_float2(-oz, -oz);
#pragma unroll
            for (int i = 0; i + 1 < P; i += 2) {
                const float2 d = fps_d2(add2_rn(make_float2(px[i], px[i + 1]), nox), add2_rn(make_float2(py[i], py[i + 1]), noy),
                                        add2_rn(make_float2(pz[i], pz[i + 1]), noz));
                td[i] = fminf(d.x, td[i]); td[i + 1] = fminf(d.y, td[i + 1]);
                tv[i] = td[i]; tv[i + 1] = td[i + 1];
            }
            if (P & 1) {
                constexpr int i = P - 1;
                td[i] = fminf(fps_d2(px[i] - ox, py[i] - oy, pz[i] - oz), td[i]);
                tv[i] = td[i];
            }
        }
        int tk[P];                                       // k of slot i (compile-time offsets from the thread's base)
#pragma unroll
        for (int i = 0; i < P; i++) tk[i] = Map::k_of(s.g, i);
        fps_tree_argmax(tv, tk);
        const uint2 cd = fps_candidate(tv[0], fps_key(tk[0]));
        uint32_t mx, kmin;
        warp_argmax(cd.x, cd.y, mx, kmin);
        if (lane < CL) {
            const unsigned long long pk = ((unsigned long long)mx << 32) | (unsigned long long)kmin;
            st_async_b64(mapa(smem_u32(&slots[par][s.rank * FPS_NW + warp]), (uint32_t)lane), mapa(ring.at(r), (uint32_t)lane), pk);
        }
        ring.wait(r);
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
        if (s.g == 0) rounds.put(j, old);
    }
    rounds.save_dist(td, [&](int i) {
        const int k = Map::k_of(s.g, i);
        return k < n ? k : -1;
    });
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
    const FpsScene<CL> s;
    const float *mat = s.in(dist, io.sa);
    int *idxs = s.row(out, io);

    float td[P];
    int kk[P];
#pragma unroll
    for (int i = 0; i < P; i++) {
        kk[i] = Map::k_of(s.g, i);
        td[i] = kk[i] < n ? 1e38f : -1.0f;
    }
    sh.ring.template start<CL>();
    int old = 0;
    if (s.g == 0) idxs[0] = io.ioff;
    for (int j = 1; j < m; j++) {
        const float *row = mat + (size_t)old * n;
        float dv[P];
#pragma unroll
        for (int i = 0; i < P; i++) dv[i] = kk[i] < n ? __ldg(row + kk[i]) : 0.0f;
        FpsScan scan;
#pragma unroll
        for (int i = 0; i < P; i++) {
            td[i] = fminf(dv[i], td[i]);
            scan.see(td[i], i);
        }
        uint32_t wkey;
        float ux, uy, uz;
        fps_exchange<CL, false>(sh, j, s.rank, scan.best, fps_key(Map::k_of(s.g, scan.at)), 0.f, 0.f, 0.f, wkey, ux, uy, uz,
                                mat, n);
        old = fps_key_to_k(wkey);
        if (s.g == 0) idxs[j] = old + io.ioff;
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
    const FpsScene<CL> s;
    const float *data = s.in(inp, io.sa);
    int *idxs = s.row(out, io);

    float td[P];
#pragma unroll
    for (int i = 0; i < P; i++) td[i] = Map::k_of(s.g, i) < n ? 1e38f : -1.0f;
    // stage features: one warp per point row for coalesced global reads
    for (int q = s.tid >> 5; q < NL; q += FPS_NW) {
        const int st = q % FPS_T, si = q / FPS_T;
        const int k = Map::k_of((int)s.rank * FPS_T + st, si);
        for (int l = s.tid & 31; l < c; l += 32) feat[(size_t)l * NLP + q] = k < n ? data[(size_t)k * c + l] : 0.0f;
    }
    for (int l = s.tid; l < c; l += FPS_T) old_f[l] = data[l];  // first sample is point 0
    sh.ring.template start<CL>();  // contains __syncthreads
    if (s.g == 0) idxs[0] = io.ioff;

    for (int j = 1; j < m; j++) {
        float d[P];
#pragma unroll
        for (int i = 0; i < P; i++) d[i] = 0.0f;
        for (int l = 0; l < c; l++) {
            const float o = old_f[l];
            const float *fl = feat + (size_t)l * NLP + s.tid;
#pragma unroll
            for (int i = 0; i < P; i++) {
                const float diff = fl[i * FPS_T] - o;
                d[i] = __fmaf_rn(diff, diff, d[i]);
            }
        }
        FpsScan scan;
#pragma unroll
        for (int i = 0; i < P; i++) {
            td[i] = fminf(d[i], td[i]);
            scan.see(td[i], i);
        }
        uint32_t wkey;
        float ux, uy, uz;
        fps_exchange<CL, false>(sh, j, s.rank, scan.best, fps_key(Map::k_of(s.g, scan.at)), 0.f, 0.f, 0.f, wkey, ux, uy, uz);
        const int old = fps_key_to_k(wkey);
        if (s.g == 0) idxs[j] = old + io.ioff;
        // fetch the winner's feature vector from its owner CTA (all threads passed the __syncthreads inside
        // fps_exchange, so nobody still reads old_f of this round)
        int og, oi;
        Map::owner_of(old, og, oi);
        const uint32_t orank = (uint32_t)(og / FPS_T);
        const int oslot = oi * FPS_T + (og % FPS_T);
        for (int l = s.tid; l < c; l += FPS_T) {
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
// at layer 2) and no kernel to produce it.  Resumable (FpsRounds): the last winner's feature row is re-read from
// global memory.
// ---------------------------------------------------------------------------------------------------
template <int CP>
struct __align__(16) FfpsPacket {
    uint32_t val, key;
    float sq;
    uint32_t pad;
    float feat[CP];
};
static_assert(sizeof(FfpsPacket<68>) == 16 + 4 * 68 && sizeof(FfpsPacket<132>) == 16 + 4 * 132, "ffps_smem (fps_plan.h)");

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
    __shared__ FpsRing ring;

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const FpsScene<CL> s;
    const int c = ca + cb;
    const float *A = s.in(fa, io.sa);
    const float *B = s.in(fb, io.sb);
    const FpsRounds rounds(io, m, s.scene, out, n);

    // ---- stage this CTA's rows: local point q = i*256 + t  <->  k = rank*256 + t + i*TT (zero rows beyond n)
    for (int q = warp; q < NL; q += FPS_NW) {
        const int k = (int)s.rank * FPS_T + (q % FPS_T) + (q / FPS_T) * TT;
        for (int l = lane; l < CP; l += 32) {
            float v = 0.0f;
            if (k < n && l < c) v = l < ca ? __ldg(A + (size_t)k * ca + l) : __ldg(B + (size_t)k * cb + (l - ca));
            featS[(size_t)q * CP + l] = v;
        }
    }
    if (s.tid == 0) ring.init();
    __syncthreads();
    float f[P][CP], td[P], sq[P];
    uint32_t key[P];
#pragma unroll
    for (int i = 0; i < P; i++) {
        const int k = s.g + i * TT;
        const float4 *row = reinterpret_cast<const float4 *>(featS + (size_t)(i * FPS_T + s.tid) * CP);
        float s2 = 0.0f;
#pragma unroll
        for (int l4 = 0; l4 < CP / 4; l4++) {
            const float4 v = row[l4];
            f[i][4 * l4 + 0] = v.x; f[i][4 * l4 + 1] = v.y; f[i][4 * l4 + 2] = v.z; f[i][4 * l4 + 3] = v.w;
        }
#pragma unroll
        for (int l = 0; l < CP; l++) s2 = __fmaf_rn(f[i][l], f[i][l], s2);     // sqdist's squared-norm chain
        sq[i] = s2;
        sqS[i * FPS_T + s.tid] = s2;
        td[i] = rounds.start(k, k < n);
        key[i] = fps_key(k);
    }
    // the point picked last (point 0 at the start of the sampling): its row is read from global memory by every CTA
    {
        const int old0 = rounds.first(s.g == 0);
        Packet &p0 = cl_pk[0];
        for (int l = s.tid; l < CP; l += FPS_T) {
            float v = 0.0f;
            if (l < c) v = l < ca ? __ldg(A + (size_t)old0 * ca + l) : __ldg(B + (size_t)old0 * cb + (l - ca));
            p0.feat[l] = v;
        }
        __syncthreads();
        if (s.tid == 0) {
            float s2 = 0.0f;
            for (int l = 0; l < CP; l++) s2 = __fmaf_rn(p0.feat[l], p0.feat[l], s2);
            p0.sq = s2;
        }
    }
    __syncthreads();
    if (CL > 1) cluster_sync_all();       // every CTA's barriers exist before any peer st.async targets them

    const Packet *oldp = &cl_pk[0];
    for (int j = rounds.jbeg; j < rounds.jend; j++) {
        const int r = j - rounds.jbeg + 1; // round of THIS launch: buffer parity / barrier phase
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
        const uint2 cd = fps_candidate(best, bkey);
        uint32_t mx, kmin;
        warp_argmax(cd.x, cd.y, mx, kmin);
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
            const int kc = k2 != KEY_INVALID ? fps_key_to_k(k2) : (int)s.rank * FPS_T;
            const int ls = ((kc - (int)s.rank * FPS_T) / TT) * FPS_T + ((kc - (int)s.rank * FPS_T) % TT);
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
                if (s.tid == 0) ring.expect(r, CL * NP * 16);
                for (int peer = warp; peer < CL; peer += FPS_NW) {
                    const uint32_t dst = mapa(smem_u32(&cl_pk[par * CL + s.rank]), (uint32_t)peer);
                    const uint32_t dbar = mapa(ring.at(r), (uint32_t)peer);
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
            ring.wait(r);
            const uint32_t v = lane < CL ? cl_pk[par * CL + lane].val : 0u;
            const uint32_t kk = lane < CL ? cl_pk[par * CL + lane].key : KEY_INVALID;
            uint32_t m3, k3;
            warp_argmax(v, kk, m3, k3);
            const uint32_t bal = __ballot_sync(0xffffffffu, lane < CL && v == m3 && kk == k3);
            oldp = &cl_pk[par * CL + (__ffs(bal) - 1)];
            win_key = k3;
        }
        if (s.g == 0) rounds.put(j, win_key != KEY_INVALID ? fps_key_to_k(win_key) : 0);
    }
    rounds.save_dist(td, [&](int i) {
        const int k = s.g + i * TT;
        return k < n ? k : -1;
    });
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
        FpsScan scan;
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
            scan.see(t, k);
        }
        const uint2 cd = fps_candidate(scan.best, fps_key(scan.at));
        uint32_t mx, kmin;
        warp_argmax(cd.x, cd.y, mx, kmin);
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
// Launch logic: the entry points validate, ask fps_plan.h for the route and launch what it says.
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

// Kernel families of the (CL, P) dispatch: fn<CL, P> is the instantiation, has(CL, P) whether it is built.  The
// cluster kernels take P a multiple of the residue classes per thread, max(1, 1024 / (CL * 256)).
struct ClusterFamily {
    static constexpr bool has(int cl, int p) { return cl * p >= 4; }
};
struct Fps3Packet : ClusterFamily {
    template <int CL, int P> static constexpr auto fn = fps3_cluster_kernel<CL, P>;
};
struct Fps3Direct : ClusterFamily {
    template <int CL, int P> static constexpr auto fn = fps3_direct_kernel<CL, P>;
};
struct FpsDist : ClusterFamily {
    template <int CL, int P> static constexpr auto fn = fpsdist_cluster_kernel<CL, P>;
};
struct FpsGeneric : ClusterFamily {
    template <int CL, int P> static constexpr auto fn = fpsc_cluster_kernel<CL, P>;
};
// matrix-free F-FPS: P = 2 points of CP = 68 channels per thread, or P = 1 of 132, on up to 8 CTAs
struct FfpsFamily {
    static constexpr bool has(int cl, int p) { return cl <= 8 && p <= 2; }
    template <int CL, int P> static constexpr auto fn = ffps_cluster_kernel<CL, P, P == 2 ? 68 : 132>;
};

// launch K::fn<plan.cl, plan.p> over CL, P in {1, 2, 4, 8, 16}
template <class K, int CL = 1, int P = 1>
static cudaError_t launch_planned(const FpsPlan &pl, int b, cudaStream_t st, void **args)
{
    if constexpr (CL > 16) {
        return cudaErrorInvalidValue;
    } else if constexpr (P > 16) {
        return launch_planned<K, CL * 2>(pl, b, st, args);
    } else {
        if constexpr (K::has(CL, P))
            if (pl.cl == CL && pl.p == P) return launch_cluster(K::template fn<CL, P>, CL, b, pl.smem, st, args);
        return launch_planned<K, CL, P * 2>(pl, b, st, args);
    }
}

}  // namespace ssd3d

using namespace ssd3d;

// The queries read the plan at the defaults of ssd3d_farthest_point_sample: dense 16-byte aligned input, heuristic
// cluster size.  Whether a route needs temp does not depend on m.
extern "C" int ssd3d_fps_needs_temp(int n, int c)
{
    return plan_fps(n, c, 2, 0, 0, true, (long long)n * c, false).kind == FpsKind::Fallback;
}

// whether the resident-scene kernel runs partial ranges of n points (flags bit 1: the pruned kernel, which also
// does, is chosen by its own flags)
extern "C" int ssd3d_fps_supports_rounds(int n, int c) { return plan_fps(n, c, 2, 0, 2, true, (long long)n * c, true).rounds; }

// floats of `temp` per scene a partial range of rounds needs: the running distances, plus (bucket kernel) the permutation
extern "C" long ssd3d_fps_temp_elems(int n, int c, int m, int flags)
{
    return n <= 0 ? 0 : plan_fps(n, c, m, 0, flags, true, (long long)n * c, true).temp;
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
    const bool partial = j0 > 0 || j1 < m;
    const FpsPlan pl = plan_fps(n, c, m, cluster, flags, (reinterpret_cast<uintptr_t>(inp) & 15u) == 0, in_stride, partial);
    if (partial) {
        SSD3D_REQUIRE(c == 3, "farthest_point_sample: a partial range of rounds is only built for c == 3");
        SSD3D_REQUIRE(pl.rounds, "farthest_point_sample: a partial range of rounds needs the resident-scene kernel "
                      "(c == 3, n %% 4 == 0, n <= 17000, 16-byte aligned input); see ssd3d_fps_supports_rounds");
        if (pl.kind == FpsKind::Bucket)
            SSD3D_REQUIRE(temp != nullptr, "farthest_point_sample: a partial range of rounds carries its state in temp[b, 2n] "
                          "(ssd3d_fps_temp_elems)");
        SSD3D_REQUIRE(temp != nullptr, "farthest_point_sample: a partial range of rounds carries its state in temp[b,n]");
    }
    SSD3D_REQUIRE(pl.kind != FpsKind::Fallback || temp != nullptr, "farthest_point_sample: n=%d c=%d needs the temp[b,n] workspace", n, c);
    cudaStream_t st = (cudaStream_t)stream;
    FpsIO io = {in_stride, 0, ldo, idx_offset, j0, j1, temp};
    void *args[] = {&n, &m, (void *)&inp, (void *)&out, (void *)&io};
    void *args_c[] = {&n, &c, &m, (void *)&inp, (void *)&out, (void *)&io};
    cudaError_t e;
    switch (pl.kind) {
    case FpsKind::Bucket: e = (cudaError_t)launch_fps3_bucket(b, n, m, inp, out, io, st); break;
    case FpsKind::Direct: e = launch_planned<Fps3Direct>(pl, b, st, args); break;
    case FpsKind::Packet: e = launch_planned<Fps3Packet>(pl, b, st, args); break;
    case FpsKind::Generic: e = launch_planned<FpsGeneric>(pl, b, st, args_c); break;
    default:
        fps_fallback_kernel<<<b, 1024, 0, st>>>(n, c, m, inp, nullptr, temp, out, io);
        SSD3D_LAUNCH_CHECK("fps_fallback_kernel");
    }
    return cuda_status(e, "farthest_point_sample launch");
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
    const FpsPlan pl = plan_fps_dist(n, cluster);
    if (pl.kind == FpsKind::Dist) {
        void *args[] = {&n, &m, (void *)&dist, (void *)&out, (void *)&io};
        return cuda_status(launch_planned<FpsDist>(pl, b, st, args), "fpsdist launch");
    }
    SSD3D_REQUIRE(temp != nullptr, "farthest_point_sample_with_distance: n=%d needs the temp[b,n] workspace", n);
    fps_fallback_kernel<<<b, 1024, 0, st>>>(n, 0, m, nullptr, dist, temp, out, io);
    SSD3D_LAUNCH_CHECK("fps_fallback_kernel");
}

extern "C" int ssd3d_farthest_point_sample_with_distance(int b, int n, int m, const float *dist, float *temp,
                                                         int *out, ssd3d_stream_t stream)
{
    return ssd3d_farthest_point_sample_with_distance_ex(b, n, m, dist, temp, out, m, 0, 0, stream);
}

// 1 when the matrix-free F-FPS kernel covers (n points, c = channels of the concatenated feature), else 0.
extern "C" int ssd3d_ffps_supported(int n, int c) { return plan_ffps(n, c, false).kind == FpsKind::Features; }

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
    const FpsPlan pl = plan_ffps(n, c, j0 > 0 || j1 < m);
    if (pl.kind != FpsKind::Features) {
        set_error("farthest_point_sample_features: n=%d c=%d not covered (use calc_square_dist + farthest_point_sample_with_distance)", n, c);
        return SSD3D_ERR_UNSUPPORTED;
    }
    const FpsIO io = {fa_stride, fb_stride, ldo, idx_offset, j0, j1, temp};
    void *args[] = {&n, &ca, &cb, &m, &fa, &fb, &out, (void *)&io};
    return cuda_status(launch_planned<FfpsFamily>(pl, b, (cudaStream_t)stream, args), "ffps launch");
}

extern "C" int ssd3d_farthest_point_sample_features(int b, int n, int ca, int cb, int m, const float *fa, const float *fb,
                                                    int *out, ssd3d_stream_t stream)
{
    return ssd3d_farthest_point_sample_features_ex(b, n, ca, cb, m, fa, (long long)n * ca, fb, (long long)n * cb, nullptr, out,
                                                   m, 0, 0, m, stream);
}
