// mlp_tc.cu -- the grouped-MLP layers on the Hopper tensor cores (wgmma + TMA + mbarrier pipeline).
//
// One layer of the SA point MLP, y = act((x . W) * scale + shift) [+ max-pool over the neighbour axis], i.e. the
// conv2d/bias/BN/ReLU/reduce_max chain of /root/reference/lib/utils/tf_util.py:127-201, :424-444 and
// /root/reference/lib/utils/layers_util.py:167-180, as ONE persistent warp-specialised GEMM kernel.
//
// Precision (DESIGN.md "Grouped MLP"): the reference computes in fp32 and the parity budget is 1e-3 relative.
// A single TF32/BF16 pass does not hold that through three chained layers, so every fp32 operand is split into
// two bf16 terms, x = x_hi + x_lo (16 mantissa bits), and the product is evaluated as three bf16 MMAs
//     x.W ~= x_hi.W_hi + x_lo.W_hi + x_hi.W_lo          (error ~2^-16, fp32 accumulation in registers)
// at 3x the bf16 tensor rate instead of the 2x-slower TF32 pipe.  Activations travel between layers already
// split (two bf16 matrices, row-major == K-major), so every operand tile is a plain TMA box in the 128B-swizzled
// K-major layout the wgmma descriptors read, and no conversion happens on the load path.
//
// Two kernels, one per route of the A operand; both stream K in 64-element blocks through a multi-stage mbarrier ring
// (a stage is released as soon as the wgmma group that read it has retired, so the loads of the next k-blocks overlap the
// MMAs), and both run the same epilogue, tc_epilogue, on the accumulator fragments where they are (scale/shift/ReLU in
// place -> fp32 / split-bf16 through per-warp TMA tensor stores, or max-pool as a shuffle reduce-and-transpose butterfly
// over the fragment rows; only pools of 32-128 rows meet other warps, through a small exchange in shared memory).  Two
// consumer warpgroups; warpgroup g owns rows 64g..64g+63 of a 128-row tile and issues the wgmma chain into its registers.
// linear_tc_tma_kernel<BN> (A read from memory): 384 threads = 3 warpgroups; one thread of warp 0 issues the TMA boxes of
// A_hi/A_lo/B_hi/B_lo, warps 4-11 are the consumers.  Tiles of 128 x BN, BN = 32, 64 or 128: a wider tile reads each A
// row from L2 and from shared memory fewer times (see linear_tc_launch).  384 threads leave 168 registers per thread, so
// the 64 accumulators of a BN = 128 consumer fit next to the epilogue.
// linear_tc_kernel<BN> (gather modes): 640 threads = 5 warpgroups; warp 0 = TMA producer of the weights (warps 1-3 idle),
// warps 4-11 = operand producers, warps 12-19 = the consumers.  640 threads leave 96 registers per thread, so tiles stop
// at BN = 64.
// Gather modes (TcParams::gather): the operand tile is not read from memory but built in shared memory by the
// producer warps from neighbour indices (1: concat(features, xyz - centre); 2: the hoisted first conv) and kept
// resident across the n-tiles of its m-tile (TcParams::astat).
// Unit-list mode (TcParams::units, round 2): the grouped matrix holds only the 8-row units the ball query listed (rows
// that repeat a group's first neighbour cannot change the max-pool); the row count comes from the list at run time, the
// gather producers look their source up through it, and the last conv of a scale pools each unit and combines the units
// of a group with atomicMax (the unit_pool branch of the epilogue).  Same bits as the dense schedule.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cstdio>
#include <cstring>

#include "common.cuh"
#include "operand.cuh"
#include "pool.cuh"
#include "wgmma.cuh"

namespace ssd3d {

constexpr int TC_BM = 128;
constexpr int TC_BK = 64;                 // bf16 elements per k-block = one 128-byte swizzle row
constexpr int TC_PROD_WARP0 = 4;          // gather kernel, warps 4..11: A-operand producers: two threads per tile row, each
constexpr int TC_PROD_WARPS = 8;          // builds 4 of the 8 16-byte chunks of a k-block
constexpr int TC_EPI_WARP0 = TC_PROD_WARP0 + TC_PROD_WARPS;   // gather kernel, warps 12..19: the two consumer warpgroups
constexpr int TC_EPI_WARPS = 8;
constexpr int TC_THREADS = (TC_EPI_WARP0 + TC_EPI_WARPS) * 32;
constexpr int TC_GATHER_MAX_BN = 64;
constexpr int TC_TMA_EPI_WARP0 = 4;       // TMA kernel, warps 4..11: the two consumer warpgroups
constexpr int TC_TMA_THREADS = (TC_TMA_EPI_WARP0 + TC_EPI_WARPS) * 32;
constexpr int TC_MAX_BN = 128;
constexpr int TC_MAX_STAGES = 4;
constexpr int TC_MAX_AKB = 4;            // A-stationary mode: k-blocks of an m-tile resident at once (K <= 256)
constexpr uint32_t TC_A_BYTES = TC_BM * TC_BK * 2;   // one A tile (hi or lo): 16 KiB
constexpr uint32_t TC_STORE_BLOCK = 4096;            // per-warp TMA-store block: 16 rows x 64 fp32 (or 2 x 64 bf16) columns
// Shared memory per CTA: the planner hands out at most TC_DYN_SMEM of dynamic shared memory (1 KiB of it is the
// alignment slack of the carve); the kernels' static __shared__ (the mbarriers, allocated in 1 KiB granules) takes the
// rest of the 227 KiB opt-in limit.
constexpr size_t TC_DYN_SMEM = 224 * 1024;
constexpr size_t TC_STATIC_SMEM = (2 * TC_MAX_STAGES + 2 * TC_MAX_AKB) * 8;
static_assert(TC_DYN_SMEM + (TC_STATIC_SMEM + 1023) / 1024 * 1024 <= 227 * 1024, "linear_tc: shared memory over the opt-in limit");

struct TcParams {
    long rows;
    int kp;          // K padded to a multiple of 16
    int n;           // output channels
    int bn;          // tile width (32, 64 or 128)
    int n_tiles, m_tiles, stages;
    const float *scale, *shift;
    int relu, pool;
    const int *rowmask;
    float *out_f32; int ld_f32;
    __nv_bfloat16 *out_hi, *out_lo; int ld_split;
    int tma_store;   // non-pooled outputs leave through per-warp shared-memory blocks + TMA tensor stores
    // gather mode (first layer of an SA scale): the A operand is not read from memory but BUILT by two producer warps:
    // x[row] = concat(points[scene, idx[row], :], xyz[scene, idx[row], :] - new_xyz[scene, row/ns, :])  (layers_util.py:160-165)
    // gather == 2 ("hoisted first layer"): the operand of THIS layer is the OUTPUT of the scale's first conv, rebuilt per
    // grouped row from a per-point table instead of being computed per row:  with W1 = [Wf ; Wx] split by input rows,
    //   relu((concat(f_j, x_j - c_i) . W1) * s + t) = relu(z[j] + (x_j - c_i) . (Wx * s)),   z = (f . Wf) * s + t  [per point]
    // g_points = z (row pitch g_ldz, this scale's columns), g_c = first-layer width (= K of this layer), g_wx = Wx*s [3][g_c]
    // astat ("A-stationary", gather modes): the produced A tile of an m-tile (all its k-blocks) stays in shared memory
    // while the CTA sweeps that m-tile's n-tiles, so the producers build it once instead of once per n-tile; only the
    // weights travel through the ring.  Tiles are then enumerated m-major per CTA.
    int astat;       // 0: A through the ring; 1: the resident A tile
    int gather, g_n, g_c, g_m, g_ns, g_ldz;
    const float *g_xyz, *g_points, *g_new_xyz, *g_wx;
    const int *g_idx;
    // UNIT-LIST mode (include/ssd3d.h, ssd3d_query_ball_point_multi_ws_ex): units[0] = number of units, units[1 + u] =
    // (group << 4) | j names rows Wj .. Wj+W-1 of a group's neighbour list, W = 1 << unit_lg (8 or 4).  The matrix this
    // launch works on then has units[0] * W rows -- compact row Wu + e is neighbour slot Wj + e of that group -- instead of
    // `rows` (which stays the capacity of the buffers): the gather producers look their source up through the list, and
    // unit_pool max-pools each W-row unit and combines the units of a group with atomicMax on out_f32[group] (zero-filled
    // by the caller; values are post-ReLU, >= 0).
    const int *units;
    int unit_pool, unit_lg;
};

// ---- PTX wrappers ---------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap *map, int x, int y, uint32_t bar)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(dst), "l"(map), "r"(bar), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap *map, uint32_t src, int x, int y)
{
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(map), "r"(src), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---- epilogue on the accumulator fragment ---------------------------------------------------------------------
// Thread t of warp w (of its warpgroup) holds tile rows 64g + 16w + t/4 in d[4j], d[4j+1] and the row 8 below in
// d[4j+2], d[4j+3], columns 8j + 2(t%4) + {0, 1} (wgmma.cuh).  The max-pools reduce these fragments where they are
// (quad_rowmax_transpose, pool.cuh).

// 8-row max-pool of a warp's fragment (dense pool == 8 or the unit-list pool): the two 8-row halves stay apart.  On return
// lane t owns slots s = i + (BN/16)(t/4), i < BN/16, of d: column 8(s/4) + 2(t%4) + (s%2) of row half (s/2)%2.
template <int BN>
__device__ __forceinline__ void frag_pool8(float (&d)[BN / 2], int lane) { quad_rowmax_transpose<BN / 2>(d, lane); }

// 16-row max-pool of a warp's fragment: halves combined first, then the quad butterfly.  On return u[i], i < BN/32, holds
// column 8(s/2) + 2(t%4) + (s%2), s = i + (BN/32)(t/4), over the warp's 16 rows.
template <int BN>
__device__ __forceinline__ void frag_pool16(const float (&d)[BN / 2], float (&u)[BN / 4], int lane)
{
#pragma unroll
    for (int j = 0; j < BN / 8; j++) {
        u[2 * j] = fmaxf(d[4 * j], d[4 * j + 2]);
        u[2 * j + 1] = fmaxf(d[4 * j + 1], d[4 * j + 3]);
    }
    quad_rowmax_transpose<BN / 4>(u, lane);
}

// pooled row gg (group of POOL rows) of columns `col`: mask (layers_util.py:180), fp32 and / or split bf16 outputs
__device__ __forceinline__ void store_pooled(const TcParams &p, long gg, int col, float mx)
{
    if (col >= p.n) return;
    store_pooled_value(mx, p.rowmask && p.rowmask[gg] == 0, (size_t)gg, col, p.out_f32, p.ld_f32, p.out_hi, p.out_lo, p.ld_split);
}

// Developer instrumentation (nvcc -DTC_PROFILE): CTA 0 accumulates, per role, the cycles spent waiting on each barrier
// and the cycles spent working; printed by the launcher.  Slots: 1 tma wait-empty | 6 prod wait-slot |
// 7 prod load+math | 8 consumer waits + MMAs of a tile | 9 epi work
#ifdef TC_PROFILE
__device__ long long tc_prof[16];
#define TCP_DECL long long tcp_t = clock64(); const bool tcp_on = blockIdx.x == 0 && lane == 0
#define TCP(i) do { if (tcp_on) { const long long t_ = clock64(); atomicAdd((unsigned long long *)&tc_prof[i], (unsigned long long)(t_ - tcp_t)); tcp_t = t_; } } while (0)
#else
#define TCP_DECL do { } while (0)
#define TCP(i) do { } while (0)
#endif

// ---------------------------------------------------------------------------------------------------------
// The epilogue of one 128 x BN tile, run by consumer warp `we` (0..7: rows 16we..16we+15 of the tile, warpgroup we / 4) on
// its accumulator fragment: folded bias/BN scale/shift, ReLU, then store or pool.  out_stage: the per-warp TMA-store
// blocks (tma_store launches); pool_xs: [8 warps][BN] floats (pools of 32-128 rows).
template <int BN>
__device__ __forceinline__ void tc_epilogue(const TcParams &p, float (&d)[BN / 2], int mt, int nt, long rows, int nunits,
                                            const float *s_scale, const float *s_shift, uint8_t *out_stage,
                                            float *pool_xs, int we, int lane, const CUtensorMap *map_ohi,
                                            const CUtensorMap *map_olo, const CUtensorMap *map_of32)
{
    const int g = we >> 2;
    const int cq = 2 * (lane & 3);                                   // this thread's column pair inside each 8 columns
    const int col_t = nt * BN;
#pragma unroll
    for (int j = 0; j < BN / 8; j++) {
        const float2 sc = *reinterpret_cast<const float2 *>(s_scale + col_t + 8 * j + cq);
        const float2 sh = *reinterpret_cast<const float2 *>(s_shift + col_t + 8 * j + cq);
        d[4 * j] = fmaf(d[4 * j], sc.x, sh.x);
        d[4 * j + 1] = fmaf(d[4 * j + 1], sc.y, sh.y);
        d[4 * j + 2] = fmaf(d[4 * j + 2], sc.x, sh.x);
        d[4 * j + 3] = fmaf(d[4 * j + 3], sc.y, sh.y);
    }
    if (p.relu) {
#pragma unroll
        for (int j = 0; j < BN / 2; j++) d[j] = fmaxf(d[j], 0.0f);
    }
    const int row0 = mt * TC_BM + 16 * we;                           // first row of this warp's fragment
    const int rq = lane >> 2;                                        // fragment row of d[4j], d[4j+1]; +8 for the others
    if (p.pool <= 1 && p.tma_store) {
        // Each warp owns a 4 KiB block: its [16 rows x 32 columns] pieces are laid out in the TMA swizzle and one bulk
        // tensor store per piece writes whole 64/128-byte row segments (rows / columns beyond the tensor are clipped by
        // the hardware).  Up to 64 columns pass through the block at a time; it is reused once the previous stores
        // have read it.
        uint8_t *blk = out_stage + we * TC_STORE_BLOCK;
        constexpr int PIECES = BN < 64 ? BN / 32 : 2;
#pragma unroll
        for (int c64 = 0; c64 < BN / (32 * PIECES); c64++) {
            if (lane == 0) tma_store_wait_read();
            __syncwarp();
#pragma unroll
            for (int q = 0; q < PIECES; q++) {
                uint8_t *piece = blk + q * 2048;
                const int c32 = PIECES * c64 + q;
                if (p.out_f32) {                                     // 128-byte rows, SWIZZLE_128B: 2 KiB
#pragma unroll
                    for (int jj = 0; jj < 4; jj++) {
                        const int j = 4 * c32 + jj;
                        const uint32_t off = (uint32_t)rq * 128u + (uint32_t)(((2 * jj + (cq >> 2)) ^ rq) << 4) + (uint32_t)(cq & 2) * 4u;
                        *reinterpret_cast<float2 *>(piece + off) = make_float2(d[4 * j], d[4 * j + 1]);
                        *reinterpret_cast<float2 *>(piece + 1024 + off) = make_float2(d[4 * j + 2], d[4 * j + 3]);
                    }
                } else {                                             // 64-byte rows (hi | lo), SWIZZLE_64B: 1 KiB each
#pragma unroll
                    for (int jj = 0; jj < 4; jj++) {
                        const int j = 4 * c32 + jj;
                        const uint32_t off = (uint32_t)rq * 64u + (uint32_t)((jj ^ ((rq >> 1) & 3)) << 4) + (uint32_t)cq * 2u;
                        uint32_t hw, lw;
                        split_pair(d[4 * j], d[4 * j + 1], hw, lw);
                        *reinterpret_cast<uint32_t *>(piece + off) = hw;
                        *reinterpret_cast<uint32_t *>(piece + 1024 + off) = lw;
                        split_pair(d[4 * j + 2], d[4 * j + 3], hw, lw);
                        *reinterpret_cast<uint32_t *>(piece + 512 + off) = hw;
                        *reinterpret_cast<uint32_t *>(piece + 1536 + off) = lw;
                    }
                }
            }
            fence_async_smem();
            __syncwarp();
            if (lane == 0) {
#pragma unroll
                for (int q = 0; q < PIECES; q++) {
                    const uint32_t piece = smem_u32(blk + q * 2048);
                    const int col = col_t + 32 * (PIECES * c64 + q);
                    if (p.out_f32) {
                        tma_store_2d(map_of32, piece, col, row0);
                    } else {
                        tma_store_2d(map_ohi, piece, col, row0);
                        tma_store_2d(map_olo, piece + 1024, col, row0);
                    }
                }
                tma_store_commit();
            }
        }
    } else if (p.pool <= 1) {
#pragma unroll
        for (int hf = 0; hf < 2; hf++) {
            const long row = (long)row0 + rq + 8 * hf;
            if (row >= rows) continue;
#pragma unroll
            for (int j = 0; j < BN / 8; j++) {
                const int col = col_t + 8 * j + cq;
                const float x0 = d[4 * j + 2 * hf], x1 = d[4 * j + 2 * hf + 1];
                if (p.out_f32) {
                    float *dst = p.out_f32 + (size_t)row * p.ld_f32 + col;
                    if (col < p.n) dst[0] = x0;
                    if (col + 1 < p.n) dst[1] = x1;
                }
                // x = hi + lo (bf16 each); columns n..ld_split-1 come out as exact zeros (next layer's K padding)
                if (p.out_hi && col < p.ld_split) {
                    uint32_t hw, lw;
                    split_pair(x0, x1, hw, lw);
                    *reinterpret_cast<uint32_t *>(p.out_hi + (size_t)row * p.ld_split + col) = hw;
                    *reinterpret_cast<uint32_t *>(p.out_lo + (size_t)row * p.ld_split + col) = lw;
                }
            }
        }
    } else if (p.unit_pool && p.unit_lg == 2) {
        // each 4-row quarter of the warp's 16 rows is one listed unit: two butterfly steps, then lane t owns slots
        // s = i + (BN/8)((t/4) % 4) of rows 4(t/16) .. 4(t/16)+3 of row half (s/2)%2
        quad_rowmax4_transpose<BN / 2>(d, lane);
#pragma unroll
        for (int i = 0; i < BN / 8; i++) {
            const int s = i + (BN / 8) * (rq & 3);
            const int ui = mt * (TC_BM / 4) + 4 * we + 2 * ((s >> 1) & 1) + (rq >> 2);
            const int col = col_t + 8 * (s >> 2) + cq + (s & 1);
            if (ui >= nunits || col >= p.n) continue;
            atomic_max_nonneg(p.out_f32 + (size_t)unit_group((uint32_t)__ldg(p.units + 1 + ui)) * p.ld_f32 + col, d[i]);
        }
    } else if (p.unit_pool) {
        // each 8-row fragment half is one listed unit; its column maxima go to the unit's GROUP row by atomicMax
        frag_pool8<BN>(d, lane);
#pragma unroll
        for (int i = 0; i < BN / 16; i++) {
            const int s = i + (BN / 16) * rq;
            const int ui = mt * (TC_BM / 8) + 2 * we + ((s >> 1) & 1);
            const int col = col_t + 8 * (s >> 2) + cq + (s & 1);
            if (ui >= nunits || col >= p.n) continue;
            atomic_max_nonneg(p.out_f32 + (size_t)unit_group((uint32_t)__ldg(p.units + 1 + ui)) * p.ld_f32 + col, d[i]);
        }
    } else if (p.pool == 8) {
        frag_pool8<BN>(d, lane);
#pragma unroll
        for (int i = 0; i < BN / 16; i++) {
            const int s = i + (BN / 16) * rq;
            const long gg = (long)mt * (TC_BM / 8) + 2 * we + ((s >> 1) & 1);
            if (gg * 8 < p.rows) store_pooled(p, gg, col_t + 8 * (s >> 2) + cq + (s & 1), d[i]);
        }
    } else {
        // pools of 16-128 rows: 16-row maxima per warp, then (32-128) the warps of a group combine through pool_xs
        float u[BN / 4];
        frag_pool16<BN>(d, u, lane);
        const int wpg = p.pool / 16;                                 // warps per pooling group
        if (wpg > 1) {
#pragma unroll
            for (int i = 0; i < BN / 32; i++) {
                const int s = i + (BN / 32) * rq;
                pool_xs[we * BN + 8 * (s >> 1) + cq + (s & 1)] = u[i];
            }
            if (wpg == 8) named_bar_sync(2, 256);
            else named_bar_sync(4 + g, 128);
            if (we % wpg == 0) {
                for (int k = 1; k < wpg; k++) {
#pragma unroll
                    for (int i = 0; i < BN / 32; i++) {
                        const int s = i + (BN / 32) * rq;
                        u[i] = fmaxf(u[i], pool_xs[(we + k) * BN + 8 * (s >> 1) + cq + (s & 1)]);
                    }
                }
            }
            if (wpg == 8) named_bar_sync(2, 256);                     // pool_xs reusable by the next tile
            else named_bar_sync(4 + g, 128);
        }
        if (we % wpg == 0) {
            const long gg = ((long)mt * TC_BM + 16 * we) / p.pool;
#pragma unroll
            for (int i = 0; i < BN / 32; i++) {
                const int s = i + (BN / 32) * rq;
                if (gg * p.pool < p.rows) store_pooled(p, gg, col_t + 8 * (s >> 1) + cq + (s & 1), u[i]);
            }
        }
    }
}

// The consumer side shared by both kernels: the wgmma chain of one tile over the k-blocks of the ring, each stage
// released (release(s, kb)) once the wgmma group that read it has retired.  a_at(s, kb): shared address of this
// warpgroup's 64-row slab of A_hi for k-block kb in ring stage s (A_lo follows TC_A_BYTES later); b_off: B_hi inside a stage.
template <int BN, typename AAt, typename Release>
__device__ __forceinline__ void tc_mma_tile(float (&d)[BN / 2], int &it, int nkb, int kp, int stages, uint32_t ring,
                                            uint32_t stage_bytes, uint32_t b_off, AAt a_at, Release release,
                                            const uint64_t *full_bar)
{
    constexpr uint32_t b_bytes = (uint32_t)BN * TC_BK * 2;
    int prev_s = -1, prev_kb = 0;
    for (int kb = 0; kb < nkb; kb++, it++) {
        const int s = it % stages;
        const uint32_t base = ring + (uint32_t)s * stage_bytes;
        const uint32_t abase = a_at(s, kb, base);
        mbar_wait_cta(smem_u32(&full_bar[s]), (uint32_t)(it / stages) & 1u);
        const int ksteps = min(TC_BK, kp - kb * TC_BK) / 16;
        const uint64_t a_hi = wg_desc(abase, 128), a_lo = wg_desc(abase + TC_A_BYTES, 128);
        const uint64_t b_hi = wg_desc(base + b_off, 128), b_lo = wg_desc(base + b_off + b_bytes, 128);
        wg_fence();
        for (int ks = 0; ks < ksteps; ks++)                          // +2 per k-step: 32 bytes in the address field
            wg_mma3<BN>(d, a_hi + 2 * ks, a_lo + 2 * ks, b_hi + 2 * ks, b_lo + 2 * ks, (kb | ks) ? 1u : 0u);
        wg_commit();
        wg_wait<1>();                                                // the previous k-block's group has retired
        if (prev_s >= 0) release(prev_s, prev_kb);
        prev_s = s; prev_kb = kb;
    }
    wg_wait<0>();
    release(prev_s, prev_kb);
}

// ---- linear_tc_tma_kernel: A from memory ---------------------------------------------------------------------
template <int BN>
__global__ void __launch_bounds__(TC_TMA_THREADS, 1)
linear_tc_tma_kernel(const __grid_constant__ CUtensorMap map_ahi, const __grid_constant__ CUtensorMap map_alo,
                     const __grid_constant__ CUtensorMap map_bhi, const __grid_constant__ CUtensorMap map_blo,
                     const __grid_constant__ CUtensorMap map_ohi, const __grid_constant__ CUtensorMap map_olo,
                     const __grid_constant__ CUtensorMap map_of32, const TcParams p)
{
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // carve: [stages] x { A_hi | A_lo | B_hi | B_lo }, per-warp output blocks (tma_store), scale/shift, pool exchange
    constexpr uint32_t b_bytes = (uint32_t)BN * TC_BK * 2;
    constexpr uint32_t stage_bytes = 2 * TC_A_BYTES + 2 * b_bytes;
    const int nkb = (p.kp + TC_BK - 1) / TC_BK;
    uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int ncov = p.n_tiles * BN + 32;
    uint8_t *out_stage = smem + (size_t)p.stages * stage_bytes;
    float *s_scale = reinterpret_cast<float *>(out_stage + (p.tma_store ? TC_EPI_WARPS * TC_STORE_BLOCK : 0));
    float *s_shift = s_scale + ncov;
    float *pool_xs = s_shift + ncov;                                     // [8 warps][BN] (pools of 16-128 rows)

    __shared__ uint64_t full_bar[TC_MAX_STAGES], empty_bar[TC_MAX_STAGES];

    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;
    // unit-list mode: the row count comes from the list (written earlier on this stream), p.rows is the buffers' capacity
    const int nunits = p.units ? __ldg(p.units) : 0;
    const long rows = p.units ? (long)nunits << p.unit_lg : p.rows;
    const int m_tiles = p.units ? (nunits + (TC_BM >> p.unit_lg) - 1) / (TC_BM >> p.unit_lg) : p.m_tiles;
    const int n_all = m_tiles * p.n_tiles;                               // tiles, n-major round robin over the CTAs

    if (threadIdx.x == 0) {
        // full barrier: the TMA thread's expect_tx arrival; empty: one arrival per consumer warp
        for (int s = 0; s < p.stages; s++) { mbar_init(smem_u32(&full_bar[s]), 1); mbar_init(smem_u32(&empty_bar[s]), TC_EPI_WARPS); }
        fence_mbar_init_cluster();
    }
    for (int i = threadIdx.x; i < ncov; i += TC_TMA_THREADS) {  // columns >= n: scale = shift = 0 -> exact zeros
        s_scale[i] = i < p.n ? __ldg(p.scale + i) : 0.0f;
        s_shift[i] = i < p.n ? __ldg(p.shift + i) : 0.0f;
    }
    __syncthreads();
    if (warp < TC_TMA_EPI_WARP0) {
        // ===== TMA producer: one thread issues every box into the ring
        if (warp == 0 && lane == 0) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(&map_ahi) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(&map_alo) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(&map_bhi) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(&map_blo) : "memory");
            int it = 0;
            TCP_DECL;
            for (int tile = blockIdx.x; tile < n_all; tile += gridDim.x) {
                const int mt = tile / p.n_tiles, nt = tile - mt * p.n_tiles;
                for (int kb = 0; kb < nkb; kb++, it++) {
                    const int s = it % p.stages;
                    mbar_wait_cta(smem_u32(&empty_bar[s]), ((uint32_t)(it / p.stages) & 1u) ^ 1u);
                    TCP(1);
                    const uint32_t base = smem_u32(smem + (size_t)s * stage_bytes);
                    const uint32_t fb = smem_u32(&full_bar[s]);
                    mbar_arrive_expect_tx(fb, stage_bytes);
                    tma_load_2d(base, &map_ahi, kb * TC_BK, mt * TC_BM, fb);
                    tma_load_2d(base + TC_A_BYTES, &map_alo, kb * TC_BK, mt * TC_BM, fb);
                    tma_load_2d(base + 2 * TC_A_BYTES, &map_bhi, kb * TC_BK, nt * BN, fb);
                    tma_load_2d(base + 2 * TC_A_BYTES + b_bytes, &map_blo, kb * TC_BK, nt * BN, fb);
                }
            }
        }
    } else {
        // ===== consumers: warpgroup g = rows 64g..64g+63 of the tile
        const int we = warp - TC_TMA_EPI_WARP0;
        const uint32_t g_off = (uint32_t)(we >> 2) * (64u * 128u);       // this warpgroup's 64 rows (8 swizzle atoms)
        int it = 0;
        TCP_DECL;
        for (int tile = blockIdx.x; tile < n_all; tile += gridDim.x) {
            const int mt = tile / p.n_tiles, nt = tile - mt * p.n_tiles;
            float d[BN / 2];
            tc_mma_tile<BN>(d, it, nkb, p.kp, p.stages, smem_u32(smem), stage_bytes, 2 * TC_A_BYTES,
                            [&](int, int, uint32_t base) { return base + g_off; },
                            [&](int s, int) { if (lane == 0) mbar_arrive(smem_u32(&empty_bar[s])); }, full_bar);
            if (we == 0) TCP(8);
            tc_epilogue<BN>(p, d, mt, nt, rows, nunits, s_scale, s_shift, out_stage, pool_xs, we, lane, &map_ohi, &map_olo,
                            &map_of32);
            if (we == 0) TCP(9);
        }
        if (p.tma_store && lane == 0) tma_store_wait_all();           // global writes complete before the CTA retires
    }
}

// ---- linear_tc_kernel: the gather modes (A built in shared memory by the producer warps) ---------------------------
template <int BN>
__global__ void __launch_bounds__(TC_THREADS, 1)
linear_tc_kernel(const __grid_constant__ CUtensorMap map_bhi, const __grid_constant__ CUtensorMap map_blo,
                 const __grid_constant__ CUtensorMap map_ohi, const __grid_constant__ CUtensorMap map_olo,
                 const __grid_constant__ CUtensorMap map_of32, const TcParams p)
{
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // carve: [resident A tiles] [stages] x { A_hi | A_lo (ring A, without astat) | B_hi | B_lo }, per-warp output blocks,
    // scale/shift, hoisted Wx, pool exchange
    constexpr uint32_t b_bytes = (uint32_t)BN * TC_BK * 2;
    const int nkb = (p.kp + TC_BK - 1) / TC_BK;
    const uint32_t a_region = p.astat ? (uint32_t)nkb * 2u * TC_A_BYTES : 0u;       // resident A tile: [nkb] x { A_hi | A_lo }
    const uint32_t b_off = p.astat ? 0u : 2 * TC_A_BYTES;                           // B_hi inside a stage
    const uint32_t stage_bytes = b_off + 2 * b_bytes;                               // ring stage
    // 1 KiB alignment by pointer arithmetic on the __shared__ array (an integer round-trip would demote every access
    // through these pointers to generic LD/ST with 64-bit address math)
    uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    const int ncov = p.n_tiles * BN + 32;
    uint8_t *ring = smem + a_region;
    uint8_t *out_stage = ring + (size_t)p.stages * stage_bytes;          // [8 warps][4 KiB], 4 KiB aligned
    float *s_scale = reinterpret_cast<float *>(out_stage + (p.tma_store ? TC_EPI_WARPS * TC_STORE_BLOCK : 0));
    float *s_shift = s_scale + ncov;
    float *s_wx = s_shift + ncov;                                        // [3][kp] (hoisted mode only)
    float *pool_xs = s_wx + (p.gather == 2 ? 3 * p.kp : 0);              // [8 warps][BN] (pools of 16-128 rows)

    __shared__ uint64_t full_bar[TC_MAX_STAGES], empty_bar[TC_MAX_STAGES];
    __shared__ uint64_t afull_bar[TC_MAX_AKB], aempty_bar[TC_MAX_AKB];   // per k-block of the resident A tile

    const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // provably warp-uniform
    // unit-list mode: the row count comes from the list (written earlier on this stream), p.rows is the buffers' capacity
    const int nunits = p.units ? __ldg(p.units) : 0;
    const long rows = p.units ? (long)nunits << p.unit_lg : p.rows;
    const int m_tiles = p.units ? (nunits + (TC_BM >> p.unit_lg) - 1) / (TC_BM >> p.unit_lg) : p.m_tiles;
    // local tile i of this CTA -> (mt, nt): n-major round robin over all tiles, or (astat) every n-tile of an m-tile
    auto tile_at = [&](int i, int &mt, int &nt) -> bool {
        if (p.astat) {
            mt = (int)blockIdx.x + (i / p.n_tiles) * (int)gridDim.x;
            nt = i % p.n_tiles;
            return mt < m_tiles;
        }
        const int tile = (int)blockIdx.x + i * (int)gridDim.x;
        mt = tile / p.n_tiles;
        nt = tile - mt * p.n_tiles;
        return tile < m_tiles * p.n_tiles;
    };

    if (threadIdx.x == 0) {
        // full barrier: the TMA thread's expect_tx arrival (+ one arrival per producer warp when A passes through the
        // ring); empty barriers: one arrival per consumer warp once its wgmma group reading the slot has retired
        for (int s = 0; s < p.stages; s++) { mbar_init(smem_u32(&full_bar[s]), p.astat ? 1 : 1 + TC_PROD_WARPS); mbar_init(smem_u32(&empty_bar[s]), TC_EPI_WARPS); }
        for (int k = 0; k < TC_MAX_AKB; k++) { mbar_init(smem_u32(&afull_bar[k]), TC_PROD_WARPS); mbar_init(smem_u32(&aempty_bar[k]), TC_EPI_WARPS); }
        fence_mbar_init_cluster();
    }
    for (int i = threadIdx.x; i < ncov; i += TC_THREADS) {      // columns >= n: scale = shift = 0 -> exact zeros
        s_scale[i] = i < p.n ? __ldg(p.scale + i) : 0.0f;
        s_shift[i] = i < p.n ? __ldg(p.shift + i) : 0.0f;
    }
    if (p.gather == 2)
        for (int i = threadIdx.x; i < 3 * p.kp; i += TC_THREADS) {
            const int a = i / p.kp, k = i - a * p.kp;
            s_wx[i] = k < p.g_c ? __ldg(p.g_wx + a * p.g_c + k) : 0.0f;
        }
    __syncthreads();
    if (warp == 0) {
        // ===== TMA producer of the weights =====
        if (lane == 0) {
            asm volatile("prefetch.tensormap [%0];" ::"l"(&map_bhi) : "memory");
            asm volatile("prefetch.tensormap [%0];" ::"l"(&map_blo) : "memory");
            int it = 0, mt, nt;
            TCP_DECL;
            for (int i = 0; tile_at(i, mt, nt); i++) {
                for (int kb = 0; kb < nkb; kb++, it++) {
                    const int s = it % p.stages;
                    const uint32_t ph = (uint32_t)(it / p.stages) & 1u;
                    TCP(15);
                    mbar_wait_cta(smem_u32(&empty_bar[s]), ph ^ 1u);
                    TCP(1);
                    const uint32_t base = smem_u32(ring + (size_t)s * stage_bytes);
                    const uint32_t fb = smem_u32(&full_bar[s]);
                    mbar_arrive_expect_tx(fb, 2 * b_bytes);
                    tma_load_2d(base + b_off, &map_bhi, kb * TC_BK, nt * BN, fb);
                    tma_load_2d(base + b_off + b_bytes, &map_blo, kb * TC_BK, nt * BN, fb);
                }
            }
        }
    } else if (warp >= TC_PROD_WARP0 && warp < TC_EPI_WARP0) {
        // ===== A-operand producers: 128 threads, one row of the tile each.  A row's source features are one contiguous
        // run (16-byte loads when c % 4 == 0); all loads of a 64-wide k-block are issued before the values are split into
        // bf16 hi/lo and stored as 16-byte chunks in the K-major SWIZZLE_128B layout the wgmma descriptor expects.
        const int pt = threadIdx.x - TC_PROD_WARP0 * 32;
        const int r = pt & (TC_BM - 1);                          // tile row
        const int c16_0 = (pt >> 7) * 4;                         // this thread's 4 chunks of every k-block
        const uint32_t rps = (uint32_t)p.g_m * (uint32_t)p.g_ns;
        const bool hoisted = p.gather == 2;
        const int src_pitch = hoisted ? p.g_ldz : p.g_c;
        const bool vec4 = (p.g_c % 4 == 0) && (src_pitch % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.g_points) & 15u) == 0);
        const int kend = hoisted ? p.g_c : p.g_c + 3;            // operand columns read from the sources
        int it = 0, mi = 0, mt, nt;
        TCP_DECL;
        for (int i = 0; tile_at(i, mt, nt); i++) {
            if (p.astat && nt != 0) continue;                     // A-stationary: the tile built for nt == 0 serves every n-tile
            const uint32_t row = (uint32_t)mt * TC_BM + (uint32_t)r;
            const bool ok = (long)row < rows;
            uint32_t rr = ok ? row : 0u;                          // position of this row's neighbour in idx[]
            if (p.units && ok)
                rr = unit_slot((uint32_t)__ldg(p.units + 1 + (row >> p.unit_lg)), (uint32_t)p.g_ns, (uint32_t)p.unit_lg,
                               row & ((1u << p.unit_lg) - 1u));
            const uint32_t scene = rr / rps, q = rr / (uint32_t)p.g_ns;
            const int a = __ldg(p.g_idx + rr);
            const float *src_f = p.g_points + ((size_t)scene * p.g_n + a) * src_pitch;
            const float *src_x = p.g_xyz + ((size_t)scene * p.g_n + a) * 3;
            const float *ctr = p.g_new_xyz + (size_t)q * 3;
            float dx = 0.0f, dy = 0.0f, dz = 0.0f;
            if (hoisted && ok) {
                dx = __ldg(src_x) - __ldg(ctr); dy = __ldg(src_x + 1) - __ldg(ctr + 1); dz = __ldg(src_x + 2) - __ldg(ctr + 2);
            }
            for (int kb = 0; kb < nkb; kb++, it++) {
                const int s = it % p.stages;
                float f[4][8];
#pragma unroll
                for (int cc = 0; cc < 4; cc++) load_concat8(f[cc], src_f, src_x, ctr, p.g_c, kend, kb * TC_BK + (c16_0 + cc) * 8, vec4, ok);
                // (loads already in flight) wait for the slot: ring stage, or this k-block of the resident A tile
                if (warp == TC_PROD_WARP0) TCP(7);
                if (p.astat) mbar_wait_cta(smem_u32(&aempty_bar[kb]), ((uint32_t)mi & 1u) ^ 1u);
                else mbar_wait_cta(smem_u32(&empty_bar[s]), ((uint32_t)(it / p.stages) & 1u) ^ 1u);
                if (warp == TC_PROD_WARP0) TCP(6);
                uint8_t *blk = p.astat ? smem + (size_t)kb * 2 * TC_A_BYTES : ring + (size_t)s * stage_bytes;
#pragma unroll
                for (int cc = 0; cc < 4; cc++) {
                    const int c16 = c16_0 + cc;
                    const int k0 = kb * TC_BK + c16 * 8;
                    if (k0 >= p.kp) break;
                    if (hoisted) hoisted_row8(f[cc], s_wx + k0, p.kp, dx, dy, dz);   // rows beyond the tensor stay 0
                    const uint32_t off = sw128_chunk((uint32_t)r, (uint32_t)c16);
                    split_store8(blk + off, blk + TC_A_BYTES + off, f[cc]);
                }
                fence_async_smem();                                   // generic-proxy stores -> visible to the tensor core
                __syncwarp();
                if (lane == 0) mbar_arrive(smem_u32(p.astat ? &afull_bar[kb] : &full_bar[s]));
            }
            mi++;
        }
    } else if (warp >= TC_EPI_WARP0) {
        // ===== consumers: warpgroup g = rows 64g..64g+63 of the tile; A from the resident tile (astat) or the ring
        const int we = warp - TC_EPI_WARP0;
        const uint32_t g_off = (uint32_t)(we >> 2) * (64u * 128u);       // this warpgroup's 64 rows (8 swizzle atoms)
        int it = 0, mi = 0, mt, nt;
        TCP_DECL;
        for (int i = 0; tile_at(i, mt, nt); i++) {
            const bool last_nt = nt == p.n_tiles - 1;
            float d[BN / 2];
            // the A slab of k-block kb: a resident k-block is waited for on the m-tile's first n-tile
            auto a_slab = [&](int, int kb, uint32_t base) -> uint32_t {
                if (!p.astat) return base + g_off;
                if (nt == 0) mbar_wait_cta(smem_u32(&afull_bar[kb]), (uint32_t)mi & 1u);
                return smem_u32(smem) + (uint32_t)kb * 2u * TC_A_BYTES + g_off;
            };
            // a ring stage (and, after the last n-tile, a resident A k-block) is free once the wgmma group reading it retired
            auto release = [&](int s, int kb) {
                if (lane == 0) {
                    mbar_arrive(smem_u32(&empty_bar[s]));
                    if (p.astat && last_nt) mbar_arrive(smem_u32(&aempty_bar[kb]));
                }
            };
            tc_mma_tile<BN>(d, it, nkb, p.kp, p.stages, smem_u32(ring), stage_bytes, b_off, a_slab, release, full_bar);
            if (last_nt) mi++;
            if (we == 0) TCP(8);
            tc_epilogue<BN>(p, d, mt, nt, rows, nunits, s_scale, s_shift, out_stage, pool_xs, we, lane, &map_ohi, &map_olo,
                            &map_of32);
            if (we == 0) TCP(9);
        }
        if (p.tma_store && lane == 0) tma_store_wait_all();           // global writes complete before the CTA retires
    }
}

// ---- fp32 -> split bf16 producers -------------------------------------------------------------------------
// hi/lo[row, 0:kp] = split(x[row, 0:c]) zero-padded
__global__ void split_rows_kernel(long rows, int c, const float *__restrict__ x, int ldx, __nv_bfloat16 *__restrict__ hi,
                                  __nv_bfloat16 *__restrict__ lo, int kp)
{
    const long total = rows * kp;
    for (long e = blockIdx.x * (long)blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x) {
        const long row = e / kp;
        const int col = (int)(e - row * kp);
        split_store(col < c ? __ldg(x + (size_t)row * ldx + col) : 0.0f, hi + e, lo + e);
    }
}

// the same, one 8-column chunk per thread and step: two 16-byte loads (when the source rows allow), two 16-byte stores
__global__ void __launch_bounds__(256)
split_rows_v8_kernel(unsigned nchunks, int c, const float *__restrict__ x, int ldx, __nv_bfloat16 *__restrict__ hi,
                     __nv_bfloat16 *__restrict__ lo, int kp, int vec)
{
    const unsigned cpr = (unsigned)kp >> 3;                            // chunks per row
    for (unsigned ch = blockIdx.x * blockDim.x + threadIdx.x; ch < nchunks; ch += gridDim.x * blockDim.x) {
        const unsigned row = ch / cpr;
        const int k0 = (int)(ch - row * cpr) * 8;
        const float *src = x + (size_t)row * ldx + k0;
        float f[8];
        if (vec && k0 + 8 <= c) {
            const float4 a = __ldg(reinterpret_cast<const float4 *>(src)), b2 = __ldg(reinterpret_cast<const float4 *>(src + 4));
            f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w; f[4] = b2.x; f[5] = b2.y; f[6] = b2.z; f[7] = b2.w;
        } else {
#pragma unroll
            for (int e = 0; e < 8; e++) f[e] = k0 + e < c ? __ldg(src + e) : 0.0f;
        }
        const size_t off = (size_t)row * kp + k0;
        split_store8(hi + off, lo + off, f);
    }
}

// fused gather + concat[features, rel-xyz] + split (layers_util.py:160-165), zero-padded to kp columns.
// One warp per output row: the source feature row is one contiguous run (coalesced 16-byte loads when c % 4 == 0),
// the two bf16 rows are written as contiguous 8-byte pieces.
__global__ void __launch_bounds__(256)
group_concat_split_kernel(long rows, int n, int c, int m, int ns, const float *__restrict__ xyz,
                          const float *__restrict__ points, const float *__restrict__ new_xyz,
                          const int *__restrict__ idx, __nv_bfloat16 *__restrict__ hi, __nv_bfloat16 *__restrict__ lo,
                          int kp, int vec4)
{
    constexpr int U = 4;                              // rows in flight per warp (independent load chains)
    extern __shared__ __align__(16) __nv_bfloat16 gcs_stage[];   // [8 warps][U rows][hi kp | lo kp]
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    __nv_bfloat16 *st = gcs_stage + (size_t)wib * U * 2 * kp;
    const long warp0 = (blockIdx.x * (long)blockDim.x + threadIdx.x) >> 5;
    const long nwarps = ((long)gridDim.x * blockDim.x) >> 5;
    const long rows_per_scene = (long)m * ns;
    const int nchunk = kp >> 3;                       // 16-byte chunks per (hi or lo) row
    for (long rbase = warp0 * U; rbase < rows; rbase += nwarps * U) {
        int a[U];
        long scene[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
            const long row = rbase + u;
            a[u] = row < rows ? __ldg(idx + row) : 0;
            scene[u] = row < rows ? row / rows_per_scene : 0;
        }
        int k4 = 0;
        if (vec4) {                                   // c % 4 == 0, 16-byte aligned feature rows
            for (k4 = lane * 4; k4 + 3 < c; k4 += 128) {
                float4 f[U];
#pragma unroll
                for (int u = 0; u < U; u++)
                    f[u] = __ldg(reinterpret_cast<const float4 *>(points + ((size_t)scene[u] * n + a[u]) * c + k4));
#pragma unroll
                for (int u = 0; u < U; u++) {
                    uint32_t h0, l0, h1, l1;
                    split_pair(f[u].x, f[u].y, h0, l0);
                    split_pair(f[u].z, f[u].w, h1, l1);
                    *reinterpret_cast<uint2 *>(st + (size_t)u * 2 * kp + k4) = make_uint2(h0, h1);
                    *reinterpret_cast<uint2 *>(st + (size_t)u * 2 * kp + kp + k4) = make_uint2(l0, l1);
                }
            }
            k4 = c & ~3;
        }
        // tail: remaining feature columns, the 3 relative coordinates, zero padding up to kp
#pragma unroll
        for (int u = 0; u < U; u++) {
            const long row = rbase + u;
            const float *src = points + ((size_t)scene[u] * n + a[u]) * c;
            for (int k = k4 + lane; k < kp; k += 32) {
                float val = 0.0f;
                if (row < rows) {
                    if (k < c) val = __ldg(src + k);
                    else if (k < c + 3) {
                        const long q = row / ns;
                        val = __ldg(xyz + ((size_t)scene[u] * n + a[u]) * 3 + (k - c)) - __ldg(new_xyz + q * 3 + (k - c));
                    }
                }
                split_store(val, st + (size_t)u * 2 * kp + k, st + (size_t)u * 2 * kp + kp + k);
            }
        }
        __syncwarp();
        // whole 16-byte chunks to global: the U rows are consecutive, so hi (and lo) of the warp is one contiguous run
#pragma unroll
        for (int u = 0; u < U; u++) {
            const long row = rbase + u;
            if (row >= rows) break;
            const uint4 *sv = reinterpret_cast<const uint4 *>(st + (size_t)u * 2 * kp);
            uint4 *dh = reinterpret_cast<uint4 *>(hi + (size_t)row * kp);
            uint4 *dl = reinterpret_cast<uint4 *>(lo + (size_t)row * kp);
            for (int ch = lane; ch < 2 * nchunk; ch += 32) {
                if (ch < nchunk) dh[ch] = sv[ch];
                else dl[ch - nchunk] = sv[ch];
            }
        }
        __syncwarp();
    }
}

// The operand of the conv that follows a HOISTED first conv (TcParams::gather == 2), materialised once in split bf16:
//   row (i, j):  relu(z[idx[i,j], :] + (xyz[idx[i,j]] - new_xyz[i]) . wx)        zero-padded to kp columns.
// For wide layers (K >= 256, 3DSSD layer 4) the A-stationary in-kernel producers starve the tensor pipe -- 128 KiB of
// resident operand leave room for two narrow weight stages -- while this elementwise pass runs at memory speed on the whole
// machine and the GEMM then takes the plain TMA-fed path.  One warp per row, one 8-column chunk per lane per step.
// (6 CTAs per SM: without the bound ptxas spends 48 registers on the unrolled chunk and only 5 fit.)
__global__ void __launch_bounds__(256, 6)
hoist_expand_split_kernel(long rows, int n, int n1, int m, int ns, const float *__restrict__ xyz, const float *__restrict__ z,
                          int ldz, const float *__restrict__ wx, const float *__restrict__ new_xyz,
                          const int *__restrict__ idx, const int *__restrict__ units, int lgu,
                          __nv_bfloat16 *__restrict__ hi, __nv_bfloat16 *__restrict__ lo, int kp)
{
    extern __shared__ __align__(16) float hx_wx[];                      // [3][kp] zero padded
    if (units) rows = (long)__ldg(units) << lgu;                        // unit-list mode (TcParams::units): compact rows
    for (int i = threadIdx.x; i < 3 * kp; i += blockDim.x) {
        const int a = i / kp, k = i - a * kp;
        hx_wx[i] = k < n1 ? __ldg(wx + a * n1 + k) : 0.0f;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31;
    const long warp0 = (blockIdx.x * (long)blockDim.x + threadIdx.x) >> 5, nwarps = ((long)gridDim.x * blockDim.x) >> 5;
    const long rps = (long)m * ns;
    const int nchunk = kp >> 3;
    for (long row = warp0; row < rows; row += nwarps) {
        long src = row;                                                  // position of this row's neighbour in idx[]
        if (units) src = unit_slot((uint32_t)__ldg(units + 1 + (row >> lgu)), (uint32_t)ns, (uint32_t)lgu, (uint32_t)row & ((1u << lgu) - 1u));
        const long scene = src / rps, q = src / ns;
        const int a = __ldg(idx + src);
        const float *px = xyz + ((size_t)scene * n + a) * 3, *pc = new_xyz + (size_t)q * 3;
        const float dx = __ldg(px) - __ldg(pc), dy = __ldg(px + 1) - __ldg(pc + 1), dz = __ldg(px + 2) - __ldg(pc + 2);
        const float *zr = z + ((size_t)scene * n + a) * ldz;
        for (int ch = lane; ch < nchunk; ch += 32) {
            const int k0 = ch * 8;
            float f[8];
            if (k0 + 8 <= n1) {
                const float4 u0 = __ldg(reinterpret_cast<const float4 *>(zr + k0)), u1 = __ldg(reinterpret_cast<const float4 *>(zr + k0 + 4));
                f[0] = u0.x; f[1] = u0.y; f[2] = u0.z; f[3] = u0.w; f[4] = u1.x; f[5] = u1.y; f[6] = u1.z; f[7] = u1.w;
            } else {
#pragma unroll
                for (int e = 0; e < 8; e++) f[e] = k0 + e < n1 ? __ldg(zr + k0 + e) : 0.0f;
            }
            hoisted_row8(f, hx_wx + k0, kp, dx, dy, dz);
            split_store8(hi + (size_t)row * kp + k0, lo + (size_t)row * kp + k0, f);
        }
    }
}

// ---- host side ------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn()
{
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
            qres == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    }
    return fn;
}

// bf16 matrix [nrows x kp] row-major -> 2D tensor map, box = 64 columns x box_rows, 128B swizzle, zero OOB fill
static int make_map(CUtensorMap *map, const void *ptr, long nrows, int kp, int box_rows)
{
    EncodeTiledFn enc = get_encode_fn();
    if (!enc) { set_error("cuTensorMapEncodeTiled is not available from the driver"); return SSD3D_ERR_UNSUPPORTED; }
    cuuint64_t dims[2] = {(cuuint64_t)kp, (cuuint64_t)nrows};
    cuuint64_t strides[1] = {(cuuint64_t)kp * 2};
    cuuint32_t box[2] = {(cuuint32_t)TC_BK, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void *>(ptr), dims, strides, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (CUresult %d) for [%ld x %d]", (int)r, nrows, kp); return SSD3D_ERR_INVALID_ARGUMENT; }
    return 0;
}

// output matrix [nrows x ncols] (row pitch ld elements) -> 2D map with a [16 rows x 32 columns] box for the per-warp stores
static int make_out_map(CUtensorMap *map, const void *ptr, long nrows, int ncols, int ld, bool f32)
{
    EncodeTiledFn enc = get_encode_fn();
    if (!enc) { set_error("cuTensorMapEncodeTiled is not available from the driver"); return SSD3D_ERR_UNSUPPORTED; }
    const int esz = f32 ? 4 : 2;
    cuuint64_t dims[2] = {(cuuint64_t)ncols, (cuuint64_t)nrows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * esz};
    cuuint32_t box[2] = {32, 16};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(map, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void *>(ptr),
                     dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     f32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled (output) failed (CUresult %d)", (int)r); return SSD3D_ERR_INVALID_ARGUMENT; }
    return 0;
}

}  // namespace ssd3d

using namespace ssd3d;


struct TcGather { int b, n, c, m, ns; const float *xyz, *points, *new_xyz; const int *idx; int ldz; const float *wx; };

static int linear_tc_launch(long rows, int kp, int n, const void *a_hi, const void *a_lo, const TcGather *g,
                            const void *b_hi, const void *b_lo, const float *scale, const float *shift, int relu, int pool,
                            const int *rowmask, float *out_f32, int ld_f32, void *out_hi, void *out_lo, int ld_split,
                            cudaStream_t stream, const int *units = nullptr, int unit_pool = 0, int unit_rows = 8)
{
    SSD3D_REQUIRE(rows >= 0 && kp > 0 && n > 0, "linear_tc: bad shape rows=%ld kp=%d n=%d", rows, kp, n);
    if (units) {
        SSD3D_REQUIRE(unit_rows == 8 || unit_rows == 4, "linear_tc (unit list): unit_rows=%d must be 8 or 4", unit_rows);
        SSD3D_REQUIRE(rows % unit_rows == 0 && pool == 1 && rowmask == nullptr, "linear_tc (unit list): rows=%ld must be a multiple of %d, no pool / rowmask", rows, unit_rows);
        if (unit_pool) {
            SSD3D_REQUIRE(relu && out_f32 && !out_hi, "linear_tc (unit list): pooling combines post-ReLU values by atomicMax into out_f32 only");
            pool = 8;
        }
    } else {
        SSD3D_REQUIRE(!unit_pool, "linear_tc: unit_pool needs a unit list");
    }
    SSD3D_REQUIRE(kp % 16 == 0, "linear_tc: kp=%d must be a multiple of 16", kp);
    SSD3D_REQUIRE((g || (a_hi && a_lo)) && b_hi && b_lo && scale && shift, "linear_tc: null operand pointer");
    SSD3D_REQUIRE(out_f32 || (out_hi && out_lo), "linear_tc: no output requested");
    SSD3D_REQUIRE(!out_f32 || ld_f32 >= n, "linear_tc: ld_f32=%d < n=%d", ld_f32, n);
    SSD3D_REQUIRE(!out_hi || (out_lo && ld_split >= n && ld_split % 8 == 0), "linear_tc: bad split output (ld_split=%d)", ld_split);
    SSD3D_REQUIRE(pool == 1 || pool == 8 || pool == 16 || pool == 32 || pool == 64 || pool == 128,
                  "linear_tc: pool=%d must be one of 1, 8, 16, 32, 64, 128", pool);
    SSD3D_REQUIRE(rows % pool == 0, "linear_tc: rows=%ld not a multiple of pool=%d", rows, pool);
    SSD3D_REQUIRE(rows < (1L << 31) - 256, "linear_tc: too many rows (%ld)", rows);
    for (const void *ptr : {a_hi, a_lo, b_hi, b_lo, (const void *)out_hi, (const void *)out_lo})
        SSD3D_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15u) == 0, "linear_tc: operand pointers must be 16-byte aligned");
    if (rows == 0) return 0;

    TcParams p = {};
    p.rows = rows; p.kp = kp; p.n = n;
    if (g) {
        p.gather = g->wx ? 2 : 1; p.g_n = g->n; p.g_c = g->c; p.g_m = g->m; p.g_ns = g->ns;
        p.g_xyz = g->xyz; p.g_points = g->points; p.g_new_xyz = g->new_xyz; p.g_idx = g->idx;
        p.g_ldz = g->ldz; p.g_wx = g->wx;
    }
    const int n16 = (n + 15) / 16 * 16;
    // when split outputs are requested the tile must also cover (and zero) the padding columns n..ld_split-1
    const int ncover = out_hi && pool <= 1 ? (ld_split > n16 ? ld_split : n16) : n16;
    // Non-pooled outputs go through TMA tensor stores when exactly one kind is requested and it is 16-byte
    // addressable.
    const bool want_f32 = out_f32 != nullptr, want_split = out_hi != nullptr;
    bool tma_store = pool <= 1 && (want_f32 != want_split);
    if (tma_store && want_f32) tma_store = (ld_f32 % 4 == 0) && ((reinterpret_cast<uintptr_t>(out_f32) & 15u) == 0);
    p.tma_store = tma_store ? 1 : 0;
    const size_t budget = TC_DYN_SMEM - 1024;  // the 1 KiB alignment slack is added back at the launch
    const int nkb = (kp + TC_BK - 1) / TC_BK;
    const bool pool_xs = pool >= 32 && !unit_pool;
    auto misc_bytes = [&](int bn) {            // scale/shift (+ hoisted Wx) + per-warp store blocks + pool exchange
        const int nt = (ncover + bn - 1) / bn;
        return 2 * ((size_t)nt * bn + 32) * sizeof(float) + (tma_store ? TC_EPI_WARPS * TC_STORE_BLOCK : 0) +
               (g && g->wx ? (size_t)3 * kp * sizeof(float) : 0) + (pool_xs ? (size_t)TC_EPI_WARPS * bn * sizeof(float) : 0);
    };
    auto ring_stage = [&](int bn, bool a_in_ring) { return (a_in_ring ? 2 * (size_t)TC_A_BYTES : 0) + 2 * (size_t)bn * TC_BK * 2; };
    // Tile widths are powers of two from 32 (columns beyond the weight rows come in as TMA zero fill and are never
    // stored), widest first but no wider than the columns need: a tile of 128 x BN reads 4 (128 + BN) operand bytes per
    // 6 * 128 * BN FLOP and K element, so a wide tile needs less L2 bandwidth per MMA, and every wgmma re-reads its
    // 64-row A slab from shared memory, so a wide tile also reads A fewer times.
    const int ncover32 = (ncover + 31) / 32 * 32;
    const int widest = g ? TC_GATHER_MAX_BN : TC_MAX_BN;
    int bn = 0, stages = 0;
    p.astat = 0;
    // gather modes keep the produced A tile resident (A-stationary) when all its k-blocks fit next to a >= 2-stage
    // weight ring: the producers then build it once per m-tile, not once per (m, n) tile.
    for (int b = widest; b >= 32 && !bn && g && nkb <= TC_MAX_AKB; b /= 2) {
        if (b > 32 && b / 2 >= ncover32) continue;
        const size_t need = (size_t)nkb * 2 * TC_A_BYTES + misc_bytes(b);
        if (need + 2 * ring_stage(b, false) <= budget) {
            bn = b;
            stages = (int)((budget - need) / ring_stage(b, false));
            p.astat = 1;
        }
    }
    // Tiles wider than 64 columns are taken only where they keep a ring of at least 3 stages (with 2, the stage the
    // producer refills is the one the previous wgmma group still reads, and the loads stop overlapping the MMAs) and
    // still give every SM a tile.
    const long m_tiles = (rows + TC_BM - 1) / TC_BM;
    for (int b = widest; b >= 32 && !bn; b /= 2) {
        if (b > 32 && b / 2 >= ncover32) continue;
        const size_t misc = misc_bytes(b);
        const int st = misc < budget ? (int)((budget - misc) / ring_stage(b, true)) : 0;
        const bool wide_ok = b <= 64 || (st >= 3 && m_tiles * ((ncover + b - 1) / b) >= kNumSMs);
        if (st >= 2 && wide_ok) { bn = b; stages = st; }
    }
    p.bn = bn;
    SSD3D_REQUIRE(bn > 0, "linear_tc: tile does not fit shared memory");
    p.n_tiles = (ncover + p.bn - 1) / p.bn;
    p.m_tiles = (int)((rows + TC_BM - 1) / TC_BM);
    const size_t stage_bytes = ring_stage(p.bn, !p.astat);
    const size_t pool_bytes = misc_bytes(p.bn) + (size_t)p.astat * nkb * 2 * TC_A_BYTES;
    SSD3D_REQUIRE((size_t)p.n_tiles * p.bn <= 4096, "linear_tc: n=%d too wide for the staged scale/shift", n);
    if (stages > TC_MAX_STAGES) stages = TC_MAX_STAGES;
    SSD3D_REQUIRE(stages >= 2, "linear_tc: tile does not fit shared memory");
    p.stages = stages;
    p.scale = scale; p.shift = shift; p.relu = relu; p.pool = pool; p.rowmask = rowmask;
    p.units = units; p.unit_pool = unit_pool; p.unit_lg = unit_rows == 4 ? 2 : 3;
    p.out_f32 = out_f32; p.ld_f32 = ld_f32;
    p.out_hi = (__nv_bfloat16 *)out_hi; p.out_lo = (__nv_bfloat16 *)out_lo; p.ld_split = ld_split;

    CUtensorMap mah, mal, mbh, mbl;
    int rc;
    if ((rc = make_map(&mbh, b_hi, n, kp, p.bn)) != 0) return rc;
    if ((rc = make_map(&mbl, b_lo, n, kp, p.bn)) != 0) return rc;
    if (!g) {
        if ((rc = make_map(&mah, a_hi, rows, kp, TC_BM)) != 0) return rc;
        if ((rc = make_map(&mal, a_lo, rows, kp, TC_BM)) != 0) return rc;
    }
    CUtensorMap moh = mbh, mol = mbh, mof = mbh;   // placeholders when unused
    if (tma_store && want_split) {
        if ((rc = make_out_map(&moh, out_hi, rows, ld_split, ld_split, false)) != 0) return rc;
        if ((rc = make_out_map(&mol, out_lo, rows, ld_split, ld_split, false)) != 0) return rc;
    }
    if (tma_store && want_f32 && (rc = make_out_map(&mof, out_f32, rows, n, ld_f32, true)) != 0) return rc;

    const size_t smem = stages * stage_bytes + pool_bytes + 1024;
    const int total = p.astat ? p.m_tiles : p.m_tiles * p.n_tiles;    // A-stationary CTAs own whole m-tiles
    const int grid = total < kNumSMs ? total : kNumSMs;
    const void *kern = g ? (p.bn == 32 ? (const void *)linear_tc_kernel<32> : (const void *)linear_tc_kernel<64>)
                         : (p.bn == 32 ? (const void *)linear_tc_tma_kernel<32>
                                       : p.bn == 64 ? (const void *)linear_tc_tma_kernel<64> : (const void *)linear_tc_tma_kernel<128>);
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return cuda_status(e, "linear_tc attr");
#ifdef TC_PROFILE
    cudaEvent_t pe0, pe1;
    cudaEventCreate(&pe0); cudaEventCreate(&pe1);
    cudaEventRecord(pe0, stream);
#endif
    if (g) {
        if (p.bn == 32) linear_tc_kernel<32><<<grid, TC_THREADS, smem, stream>>>(mbh, mbl, moh, mol, mof, p);
        else linear_tc_kernel<64><<<grid, TC_THREADS, smem, stream>>>(mbh, mbl, moh, mol, mof, p);
    } else {
        switch (p.bn) {
            case 32: linear_tc_tma_kernel<32><<<grid, TC_TMA_THREADS, smem, stream>>>(mah, mal, mbh, mbl, moh, mol, mof, p); break;
            case 64: linear_tc_tma_kernel<64><<<grid, TC_TMA_THREADS, smem, stream>>>(mah, mal, mbh, mbl, moh, mol, mof, p); break;
            default: linear_tc_tma_kernel<128><<<grid, TC_TMA_THREADS, smem, stream>>>(mah, mal, mbh, mbl, moh, mol, mof, p); break;
        }
    }
#ifdef TC_PROFILE
    {
        cudaEventRecord(pe1, stream);
        cudaDeviceSynchronize();
        float ms = 0.f;
        cudaEventElapsedTime(&ms, pe0, pe1);
        long long h[16];
        cudaMemcpyFromSymbol(h, tc_prof, sizeof(h));
        fprintf(stderr, "tc_prof rows=%ld kp=%d n=%d bn=%d astat=%d stages=%d gather=%d pool=%d tiles/cta=%.1f  %.1f us |"
                " tma_wait %lld | prod: wait %lld work %lld | mma %lld | epi %lld\n",
                rows, kp, n, p.bn, p.astat, p.stages, p.gather, pool, (double)total / grid, ms * 1e3, h[1], h[6], h[7], h[8], h[9]);
        memset(h, 0, sizeof(h));
        cudaMemcpyToSymbol(tc_prof, h, sizeof(h));
        cudaEventDestroy(pe0); cudaEventDestroy(pe1);
    }
#endif
    SSD3D_LAUNCH_CHECK("linear_tc_kernel");
}

static int hoist_expand_split_launch(int b, int n, int n1, int m, int nsample, const float *xyz, const float *z, int ldz,
                                     const float *wx, const float *new_xyz, const int *idx, const int *units, void *hi,
                                     void *lo, int kp, ssd3d_stream_t stream, int unit_rows = 8)
{
    SSD3D_REQUIRE(b >= 0 && n > 0 && m >= 0 && n1 > 0 && nsample > 0 && ldz >= n1, "hoist_expand_split: bad shape");
    SSD3D_REQUIRE(kp % 16 == 0 && kp >= n1 && kp <= 4096, "hoist_expand_split: kp=%d must be a multiple of 16 in [n1, 4096]", kp);
    SSD3D_REQUIRE(ldz % 4 == 0 && (reinterpret_cast<uintptr_t>(z) & 15u) == 0, "hoist_expand_split: z rows must be 16-byte aligned");
    SSD3D_REQUIRE(xyz && z && wx && new_xyz && idx && hi && lo, "hoist_expand_split: null pointer");
    SSD3D_REQUIRE(((reinterpret_cast<uintptr_t>(hi) | reinterpret_cast<uintptr_t>(lo)) & 15u) == 0, "hoist_expand_split: outputs must be 16-byte aligned");
    const long rows = (long)b * m * nsample;
    if (rows == 0) return 0;
    const long blocks_want = (rows + 7) / 8;
    const int blocks = (int)(blocks_want < (long)kNumSMs * 32 ? blocks_want : (long)kNumSMs * 32);
    hoist_expand_split_kernel<<<blocks, 256, (size_t)3 * kp * sizeof(float), (cudaStream_t)stream>>>(
        rows, n, n1, m, nsample, xyz, z, ldz, wx, new_xyz, idx, units, unit_rows == 4 ? 2 : 3, (__nv_bfloat16 *)hi,
        (__nv_bfloat16 *)lo, kp);
    SSD3D_LAUNCH_CHECK("hoist_expand_split_kernel");
}

extern "C" int ssd3d_hoist_expand_split(int b, int n, int n1, int m, int nsample, const float *xyz, const float *z, int ldz,
                                        const float *wx, const float *new_xyz, const int *idx, void *hi, void *lo, int kp,
                                        ssd3d_stream_t stream)
{
    return hoist_expand_split_launch(b, n, n1, m, nsample, xyz, z, ldz, wx, new_xyz, idx, nullptr, hi, lo, kp, stream);
}

extern "C" int ssd3d_hoist_expand_split_units(int b, int n, int n1, int m, int nsample, const float *xyz, const float *z,
                                              int ldz, const float *wx, const float *new_xyz, const int *idx,
                                              const int *units, void *hi, void *lo, int kp, ssd3d_stream_t stream)
{
    return ssd3d_hoist_expand_split_units_ex(b, n, n1, m, nsample, xyz, z, ldz, wx, new_xyz, idx, units, hi, lo, kp, stream, 8);
}

// The unit lists of 8- and 4-row units (include/ssd3d.h): a list names at most 16 units per group, so 4-row units
// cover nsample <= 64 and 8-row units nsample <= 128
static bool unit_rows_ok(int unit_rows, int nsample)
{
    return (unit_rows == 8 || unit_rows == 4) && nsample % unit_rows == 0 && nsample <= 16 * unit_rows;
}

extern "C" int ssd3d_hoist_expand_split_units_ex(int b, int n, int n1, int m, int nsample, const float *xyz, const float *z,
                                                 int ldz, const float *wx, const float *new_xyz, const int *idx,
                                                 const int *units, void *hi, void *lo, int kp, ssd3d_stream_t stream,
                                                 int unit_rows)
{
    SSD3D_REQUIRE(units && unit_rows_ok(unit_rows, nsample),
                  "hoist_expand_split_units: needs a unit list, unit_rows 8 or 4 and nsample a multiple of it, <= 16 * unit_rows (nsample=%d unit_rows=%d)",
                  nsample, unit_rows);
    return hoist_expand_split_launch(b, n, n1, m, nsample, xyz, z, ldz, wx, new_xyz, idx, units, hi, lo, kp, stream, unit_rows);
}

// Unit-list forms of ssd3d_linear_tc / ssd3d_linear_tc_hoisted (TcParams::units): the matrix has units[0] * 8 rows (`rows` /
// b*m*nsample is the capacity of the buffers).  unit_pool != 0: each 8-row unit is max-pooled and combined into
// out_f32[group] by atomicMax (ReLU required, out_f32 zero-filled by the caller, no split output).
extern "C" int ssd3d_linear_tc_units(long rows, int kp, int n, const void *a_hi, const void *a_lo, const void *b_hi,
                                     const void *b_lo, const float *scale, const float *shift, int relu, const int *units,
                                     int unit_pool, float *out_f32, int ld_f32, void *out_hi, void *out_lo, int ld_split,
                                     ssd3d_stream_t stream)
{
    return ssd3d_linear_tc_units_ex(rows, kp, n, a_hi, a_lo, b_hi, b_lo, scale, shift, relu, units, unit_pool, out_f32, ld_f32,
                                    out_hi, out_lo, ld_split, stream, 8);
}

// ... with units of unit_rows (8 or 4) rows: the matrix has units[0] * unit_rows rows
extern "C" int ssd3d_linear_tc_units_ex(long rows, int kp, int n, const void *a_hi, const void *a_lo, const void *b_hi,
                                        const void *b_lo, const float *scale, const float *shift, int relu, const int *units,
                                        int unit_pool, float *out_f32, int ld_f32, void *out_hi, void *out_lo, int ld_split,
                                        ssd3d_stream_t stream, int unit_rows)
{
    SSD3D_REQUIRE(units, "linear_tc_units: null unit list");
    return linear_tc_launch(rows, kp, n, a_hi, a_lo, nullptr, b_hi, b_lo, scale, shift, relu, 1, nullptr, out_f32, ld_f32,
                            out_hi, out_lo, ld_split, (cudaStream_t)stream, units, unit_pool, unit_rows);
}

extern "C" int ssd3d_linear_tc_hoisted_units(int b, int n, int n1, int m, int nsample, const float *xyz, const float *z,
                                             int ldz, const float *wx, const float *new_xyz, const int *idx,
                                             const int *units, int nout, const void *b_hi, const void *b_lo,
                                             const float *scale, const float *shift, int relu, int unit_pool, float *out_f32,
                                             int ld_f32, void *out_hi, void *out_lo, int ld_split, ssd3d_stream_t stream)
{
    return ssd3d_linear_tc_hoisted_units_ex(b, n, n1, m, nsample, xyz, z, ldz, wx, new_xyz, idx, units, nout, b_hi, b_lo, scale,
                                            shift, relu, unit_pool, out_f32, ld_f32, out_hi, out_lo, ld_split, stream, 8);
}

extern "C" int ssd3d_linear_tc_hoisted_units_ex(int b, int n, int n1, int m, int nsample, const float *xyz, const float *z,
                                                int ldz, const float *wx, const float *new_xyz, const int *idx,
                                                const int *units, int nout, const void *b_hi, const void *b_lo,
                                                const float *scale, const float *shift, int relu, int unit_pool, float *out_f32,
                                                int ld_f32, void *out_hi, void *out_lo, int ld_split, ssd3d_stream_t stream,
                                                int unit_rows)
{
    SSD3D_REQUIRE(b >= 0 && n > 0 && m >= 0 && n1 > 0 && nsample > 0 && ldz >= n1, "linear_tc_hoisted_units: bad shape");
    SSD3D_REQUIRE(xyz && new_xyz && idx && z && wx && units, "linear_tc_hoisted_units: null pointer");
    SSD3D_REQUIRE(unit_rows_ok(unit_rows, nsample),
                  "linear_tc_hoisted_units: nsample=%d must be a multiple of unit_rows=%d (8 or 4), <= 16 * unit_rows", nsample, unit_rows);
    TcGather g = {b, n, n1, m, nsample, xyz, z, new_xyz, idx, ldz, wx};
    const int kp = (n1 + 15) / 16 * 16;
    return linear_tc_launch((long)b * m * nsample, kp, nout, nullptr, nullptr, &g, b_hi, b_lo, scale, shift, relu, 1, nullptr,
                            out_f32, ld_f32, out_hi, out_lo, ld_split, (cudaStream_t)stream, units, unit_pool, unit_rows);
}

extern "C" int ssd3d_linear_tc(long rows, int kp, int n, const void *a_hi, const void *a_lo, const void *b_hi,
                               const void *b_lo, const float *scale, const float *shift, int relu, int pool,
                               const int *rowmask, float *out_f32, int ld_f32, void *out_hi, void *out_lo, int ld_split,
                               ssd3d_stream_t stream)
{
    return linear_tc_launch(rows, kp, n, a_hi, a_lo, nullptr, b_hi, b_lo, scale, shift, relu, pool, rowmask, out_f32, ld_f32,
                            out_hi, out_lo, ld_split, (cudaStream_t)stream);
}

// First layer of an SA scale with the gather fused into the operand load: rows = b*m*nsample, K = c+3 (kp = round16).
extern "C" int ssd3d_linear_tc_gather(int b, int n, int c, int m, int nsample, const float *xyz, const float *points,
                                      const float *new_xyz, const int *idx, int nout, const void *b_hi, const void *b_lo,
                                      const float *scale, const float *shift, int relu, int pool, const int *rowmask,
                                      float *out_f32, int ld_f32, void *out_hi, void *out_lo, int ld_split,
                                      ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && n > 0 && m >= 0 && c >= 0 && nsample > 0, "linear_tc_gather: bad shape");
    SSD3D_REQUIRE(xyz && new_xyz && idx && (points || c == 0), "linear_tc_gather: null pointer");
    TcGather g = {b, n, c, m, nsample, xyz, points, new_xyz, idx, 0, nullptr};
    const int kp = (c + 3 + 15) / 16 * 16;
    return linear_tc_launch((long)b * m * nsample, kp, nout, nullptr, nullptr, &g, b_hi, b_lo, scale, shift, relu, pool,
                            rowmask, out_f32, ld_f32, out_hi, out_lo, ld_split, (cudaStream_t)stream);
}

// Second layer of an SA scale fed by the HOISTED first layer (see TcParams): z[b,n,ldz] holds (f . Wf) * s1 + t1 per
// point (this scale's n1 columns start at z), wx = Wx * s1 as [3][n1]; the operand row of grouped element (i,j) is
// relu(z[idx] + (xyz[idx] - new_xyz[i]) . wx), built by the producer warps.  K of this layer = n1 (kp = round16).
extern "C" int ssd3d_linear_tc_hoisted(int b, int n, int n1, int m, int nsample, const float *xyz, const float *z, int ldz,
                                       const float *wx, const float *new_xyz, const int *idx, int nout, const void *b_hi,
                                       const void *b_lo, const float *scale, const float *shift, int relu, int pool,
                                       const int *rowmask, float *out_f32, int ld_f32, void *out_hi, void *out_lo,
                                       int ld_split, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && n > 0 && m >= 0 && n1 > 0 && nsample > 0 && ldz >= n1, "linear_tc_hoisted: bad shape");
    SSD3D_REQUIRE(xyz && new_xyz && idx && z && wx, "linear_tc_hoisted: null pointer");
    TcGather g = {b, n, n1, m, nsample, xyz, z, new_xyz, idx, ldz, wx};
    const int kp = (n1 + 15) / 16 * 16;
    return linear_tc_launch((long)b * m * nsample, kp, nout, nullptr, nullptr, &g, b_hi, b_lo, scale, shift, relu, pool,
                            rowmask, out_f32, ld_f32, out_hi, out_lo, ld_split, (cudaStream_t)stream);
}

extern "C" int ssd3d_split_rows(long rows, int c, const float *x, int ldx, void *hi, void *lo, int kp, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(rows >= 0 && c > 0 && ldx >= c && kp >= c && kp % 8 == 0, "split_rows: bad shape rows=%ld c=%d ldx=%d kp=%d", rows, c, ldx, kp);
    SSD3D_REQUIRE(x && hi && lo, "split_rows: null pointer");
    const long total = rows * kp;
    if (total == 0) return 0;
    const long nchunks = total / 8;
    if (nchunks < (1L << 31) && ((reinterpret_cast<uintptr_t>(hi) | reinterpret_cast<uintptr_t>(lo)) & 15u) == 0) {
        const int vec = (ldx % 4 == 0 && (reinterpret_cast<uintptr_t>(x) & 15u) == 0) ? 1 : 0;
        const long want = (nchunks + 255) / 256;
        const int blocks = (int)(want < (long)kNumSMs * 16 ? want : (long)kNumSMs * 16);
        split_rows_v8_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>((unsigned)nchunks, c, x, ldx, (__nv_bfloat16 *)hi,
                                                                       (__nv_bfloat16 *)lo, kp, vec);
        SSD3D_LAUNCH_CHECK("split_rows_v8_kernel");
    }
    const long want = (total + 255) / 256;
    const int blocks = (int)(want < (long)kNumSMs * 16 ? want : (long)kNumSMs * 16);
    split_rows_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(rows, c, x, ldx, (__nv_bfloat16 *)hi, (__nv_bfloat16 *)lo, kp);
    SSD3D_LAUNCH_CHECK("split_rows_kernel");
}

extern "C" int ssd3d_group_concat_split(int b, int n, int c, int m, int nsample, const float *xyz, const float *points,
                                        const float *new_xyz, const int *idx, void *hi, void *lo, int kp,
                                        ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && n > 0 && m >= 0 && c >= 0 && nsample > 0, "group_concat_split: bad shape");
    SSD3D_REQUIRE(kp >= c + 3 && kp % 8 == 0, "group_concat_split: kp=%d must be >= c+3=%d and a multiple of 8", kp, c + 3);
    SSD3D_REQUIRE(xyz && new_xyz && idx && hi && lo && (points || c == 0), "group_concat_split: null pointer");
    const long rows = (long)b * m * nsample;
    if (rows == 0) return 0;
    const long want = (rows + 31) / 32;                             // 8 warps x 4 rows per block
    const int blocks = (int)(want < (long)kNumSMs * 32 ? want : (long)kNumSMs * 32);
    const int vec4 = (c >= 4 && c % 4 == 0 && (reinterpret_cast<uintptr_t>(points) & 15u) == 0) ? 1 : 0;
    const size_t gsm = (size_t)8 * 4 * 2 * kp * sizeof(__nv_bfloat16);
    SSD3D_REQUIRE(gsm <= 96 * 1024, "group_concat_split: kp=%d too wide", kp);
    const cudaError_t ea = cudaFuncSetAttribute((const void *)group_concat_split_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gsm);
    if (ea != cudaSuccess) return cuda_status(ea, "group_concat_split shared-memory opt-in");
    group_concat_split_kernel<<<blocks, 256, gsm, (cudaStream_t)stream>>>(rows, n, c, m, nsample, xyz, points, new_xyz, idx,
                                                                          (__nv_bfloat16 *)hi, (__nv_bfloat16 *)lo, kp, vec4);
    SSD3D_LAUNCH_CHECK("group_concat_split_kernel");
}
