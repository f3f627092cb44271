// sa_fused.cu -- one SA scale in ONE kernel: gather + concat + (conv+BN+ReLU) x L + max-pool + mask, wgmma.
//
// Fuses lib/utils/layers_util.py:157-180 of the reference (idx masking, 2x group_point, centre subtraction, concat,
// the conv2d/bias/BN/ReLU stack, reduce_max, mask multiply -- ~25 TF kernels per scale, each streaming [B,M,K,C]
// through HBM) for the layers whose weights fit in shared memory (3DSSD layer1/layer2: 93% of the grouped rows).
// Nothing but the neighbour indices, the gathered source rows (L2-resident) and the pooled [B,M,C3] result touches
// global memory; activations go wgmma registers -> fp32 staging in shared memory -> registers -> shared memory (already
// split in bf16 hi/lo and already in the swizzled K-major layout the next layer's wgmma descriptors expect).
//
// Per CTA: S "slots" of 128*WG threads (a slot works on one 128-row tile = 128/K neighbour groups; its WG warpgroups
// split the 16-byte chunks of the gather and the 32-column chunks of every epilogue):
//   weights of all layers (hi+lo images, pre-swizzled on the host) are bulk-copied to shared memory once and shared
//   by the slots; each slot owns ONE operand buffer and one fp32 accumulator staging buffer and loops over tiles:
//   gather+split -> [fence.proxy.async] -> layer-0 MMAs (the slot's warpgroups split the 64-row halves of the tile and
//   the <= 64-column chunks of the layer; each chunk is one wgmma chain into registers, staged row-major) -> epilogue
//   (scale/shift/ReLU, split) written IN PLACE over the operand the finished MMAs no longer need -> ... -> last layer:
//   max-pool.
// Small stacks (layer1) run S=1 with several CTAs per SM; stacks whose weights fill most of shared memory (layer2) run
// one CTA per SM with as many slots as fit, each of two warpgroups -- one slot for the layer-2 stacks, whose staged
// accumulator (128 x 132 fp32) and weights leave no room for a second, so their tiles overlap only across SMs.
// Hoisted mode (SfParams::hoist): the scale's first conv has been moved to a per-point table z (include/ssd3d.h,
// ssd3d_sa_mlp_fused_hoisted); the gather then builds relu(z[idx] + (xyz[idx] - centre) . Wx') and the stack starts at
// the second conv.
// Unit-list mode (SfParams::units, round 2): a neighbour list repeats its first hit beyond pts_cnt
// (grouping/tf_grouping_g.cu:245-248) and the copies cannot change the max-pool, so a tile is made of 16 listed 8-row units
// (the ball query lists ceil(cnt / 8) units per non-empty group) instead of 128 consecutive rows; each unit is pooled by the
// shuffle butterfly and the units of a group meet through atomicMax on the non-negative fp32 result, which the caller
// zero-fills (= the cnt == 0 mask of layers_util.py:180).  Same bits as the dense schedule, 4-8x fewer rows on KITTI-like
// clouds (DESIGN.md section 3.4).
//
// Precision: same bf16 hi/lo split and 3-MMA scheme as mlp_tc.cu.
#include <cuda_bf16.h>
#include <cstdio>
#include <cstring>

#include "common.cuh"
#include "pool.cuh"
#include "wgmma.cuh"

namespace ssd3d {

constexpr int SF_THREADS = 128;
constexpr int SF_MAX_LAYERS = 3;

struct SfParams {
    int n, c, m, ns;                 // points per scene, feature channels, queries per scene, neighbours per query
    long rows;                       // b*m*ns
    int tiles;
    const float *xyz, *points, *new_xyz;
    const int *idx, *cnt;
    // unit list (ssd3d_query_ball_point_multi_ws): when set, a tile is 16 UNITS of 8 rows -- units[1 + u] = (group << 4) | j
    // names rows 8j..8j+7 of neighbour list `group` -- instead of 128 consecutive rows, units[0] is their number, and the
    // pooled result is combined across the units of a group with atomicMax on the (non-negative) fp32 output
    const int *units;
    // hoisted first conv (see ssd3d_linear_tc_hoisted in include/ssd3d.h): `points` is the per-point table z (row pitch
    // ldz, c = its width n1), the operand row is relu(z[idx] + (xyz[idx] - new_xyz) . wx) with wx = [3][c], and the
    // stack starts at the scale's SECOND conv (K = c, no xyz columns appended)
    int hoist, ldz;
    const float *wx;
    int nl;
    int kp[SF_MAX_LAYERS];           // K of layer l padded to 16
    int npad[SF_MAX_LAYERS];         // N of layer l padded to 16
    int nout[SF_MAX_LAYERS];         // true N
    uint32_t w_off[SF_MAX_LAYERS];   // byte offset of the layer's weight image in the packed blob / shared memory
    uint32_t w_half[SF_MAX_LAYERS];  // bytes of the hi half (lo follows)
    uint32_t ss_off[SF_MAX_LAYERS];  // float offset of the layer's scale (shift follows at +npad) in the ss blob
    uint32_t w_total, ss_total;      // bytes / floats
    const uint8_t *w_blob;
    const float *ss_blob;
    int sspad[SF_MAX_LAYERS];        // npad rounded up to 32 (scale/shift arrays are zero padded to this)
    int nfull[SF_MAX_LAYERS];        // layer l's K = nfull 64-wide k-blocks (128-byte rows) + one tail block
    int rbt[SF_MAX_LAYERS];          // bytes per row of the tail block: 0 (none), 32 (16 wide), 64 (32), 128 (48)
    uint32_t abuf_bytes;             // operand buffer of one slot
    uint32_t acc_cols;               // staged accumulator columns of one slot (widest layer, rounded up to 32)
    float *out_f32; int ld_f32;
    __nv_bfloat16 *out_hi, *out_lo; int ld_split;
    int pool_first;                  // caller guarantees scale >= 0 in the LAST layer: pool raw accumulators, affine after
};

__device__ __forceinline__ void sf_fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// x = hi + lo with hi = bf16(x), lo = bf16(x - hi); two values per call, packed {x1 : x0} like two adjacent bf16
__device__ __forceinline__ void sf_split_pair(float x0, float x1, uint32_t &hw, uint32_t &lw)
{
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(hw) : "f"(x1), "f"(x0));
    const float h0 = __uint_as_float(hw << 16), h1 = __uint_as_float(hw & 0xffff0000u);
    asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(lw) : "f"(x1 - h1), "f"(x0 - h0));
}
// Where row r of a 128-row operand tile lives.  An A buffer is laid out as k-blocks of { hi tile | lo tile }
// (128 rows x rb bytes each), each tile in the canonical K-major swizzled layout of span rb: 16-byte chunk j of
// row r sits at chunk j ^ ((r >> log2(128/rb)) & (rb/16 - 1)).  The first nfull blocks are 64 wide (rb = 128),
// the tail block is rbt bytes wide.  Built once per (thread, layer); chunk() is then a handful of integer ops.
struct SfRowMap {
    uint32_t row_f, xor_f;            // full blocks: byte offset of the row inside a tile, swizzle mask
    uint32_t base_t, row_t, xor_t;    // tail block: byte offset of the block, of the row, swizzle mask
    uint32_t lo_t;                    // hi -> lo tile distance in the tail block (full blocks: 16 KiB)
    int full8;                        // nfull * 8: first 16-byte chunk index of the tail block
    __device__ __forceinline__ SfRowMap(int r, int nfull, int rbt)
    {
        row_f = (uint32_t)(r >> 3) * 1024u + (uint32_t)(r & 7) * 128u;
        xor_f = (uint32_t)(r & 7);
        const int sh = rbt == 128 ? 0 : (rbt == 64 ? 1 : 2);
        base_t = (uint32_t)nfull * (2u * 128u * 128u);
        row_t = (uint32_t)(r >> 3) * (uint32_t)(8 * rbt) + (uint32_t)(r & 7) * (uint32_t)rbt;
        xor_t = (uint32_t)((r >> sh) & ((rbt >> 4) - 1));
        lo_t = 128u * (uint32_t)rbt;
        full8 = nfull * 8;
    }
    // byte offset of the 16-byte chunk holding columns [8*c16g, 8*c16g+8); *lo_off = distance to the lo tile
    __device__ __forceinline__ uint32_t chunk(int c16g, uint32_t *lo_off) const
    {
        if (c16g < full8) {
            *lo_off = 128u * 128u;
            return (uint32_t)(c16g >> 3) * (2u * 128u * 128u) + row_f + ((((uint32_t)c16g & 7u) ^ xor_f) << 4);
        }
        *lo_off = lo_t;
        return base_t + row_t + (((uint32_t)(c16g - full8) ^ xor_t) << 4);
    }
};
__device__ __forceinline__ void sf_bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }
__device__ __forceinline__ uint32_t sf_f2ord(float x)
{
    const uint32_t b = __float_as_uint(x);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float sf_ord2f(uint32_t u) { return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u); }

// ---- shape policies -------------------------------------------------------------------------------------------------
// The kernel body is written once against a policy C that answers every shape question (layer count, padded K / N of a
// layer, block layout, blob offsets, neighbours per group).  SfDyn reads the answers from the parameter block at run
// time (any stack the planner accepts); SfStat<...> answers at COMPILE time for the stacks of the shipped 3DSSD
// configuration, so that after unrolling the layer loop every address computation, chunk bound and pooling width is a
// literal (integer / branch / uniform-register bookkeeping of exactly these questions is otherwise a large share of the
// kernel's issued instructions).
__host__ __device__ constexpr int sf_r16(int x) { return (x + 15) / 16 * 16; }
__host__ __device__ constexpr int sf_rbt_of(int kp) { return kp % 64 == 0 ? 0 : (kp % 64 <= 16 ? 32 : (kp % 64 <= 32 ? 64 : 128)); }
__host__ __device__ constexpr uint32_t sf_abuf_of(int kp)
{
    return (uint32_t)(((kp / 64) * 2 * 128 * 128 + 2 * 128 * sf_rbt_of(kp) + 1023) / 1024 * 1024);
}

struct SfDyn {
    static constexpr bool kStatic = false;
    const SfParams &p;
    __device__ __forceinline__ explicit SfDyn(const SfParams &p_) : p(p_) {}
    __device__ __forceinline__ int nl() const { return p.nl; }
    __device__ __forceinline__ int ns() const { return p.ns; }
    __device__ __forceinline__ int c() const { return p.c; }
    __device__ __forceinline__ bool hoist() const { return p.hoist != 0; }
    __device__ __forceinline__ int kp(int l) const { return p.kp[l]; }
    __device__ __forceinline__ int npad(int l) const { return p.npad[l]; }
    __device__ __forceinline__ int nout(int l) const { return p.nout[l]; }
    __device__ __forceinline__ int nfull(int l) const { return p.nfull[l]; }
    __device__ __forceinline__ int rbt(int l) const { return p.rbt[l]; }
    __device__ __forceinline__ uint32_t w_off(int l) const { return p.w_off[l]; }
    __device__ __forceinline__ uint32_t w_half(int l) const { return p.w_half[l]; }
    __device__ __forceinline__ uint32_t ss_off(int l) const { return p.ss_off[l]; }
    __device__ __forceinline__ int sspad(int l) const { return p.sspad[l]; }
    __device__ __forceinline__ uint32_t w_total() const { return p.w_total; }
    __device__ __forceinline__ uint32_t ss_total() const { return p.ss_total; }
    __device__ __forceinline__ uint32_t abuf_bytes() const { return p.abuf_bytes; }
    __device__ __forceinline__ uint32_t acc_cols() const { return p.acc_cols; }
};

// Hoisted stacks of two convs (the shipped configuration): operand width K0 = n1 of the hoisted first conv, then
// K0 -> N0 -> N1, NS neighbours per group.
template <int K0, int N0, int N1, int NS>
struct SfStat {
    static constexpr bool kStatic = true;
    __device__ __forceinline__ explicit SfStat(const SfParams &) {}
    static constexpr int KP0 = sf_r16(K0), NP0 = sf_r16(N0), NP1 = sf_r16(N1);
    __device__ __forceinline__ constexpr int nl() const { return 2; }
    __device__ __forceinline__ constexpr int ns() const { return NS; }
    __device__ __forceinline__ constexpr int c() const { return K0; }
    __device__ __forceinline__ constexpr bool hoist() const { return true; }
    __device__ __forceinline__ constexpr int kp(int l) const { return l == 0 ? KP0 : NP0; }
    __device__ __forceinline__ constexpr int npad(int l) const { return l == 0 ? NP0 : NP1; }
    __device__ __forceinline__ constexpr int nout(int l) const { return l == 0 ? N0 : N1; }
    __device__ __forceinline__ constexpr int nfull(int l) const { return kp(l) / 64; }
    __device__ __forceinline__ constexpr int rbt(int l) const { return sf_rbt_of(kp(l)); }
    __device__ __forceinline__ constexpr uint32_t w_half(int l) const { return (uint32_t)(npad(l) * (nfull(l) * 128 + rbt(l))); }
    __device__ __forceinline__ constexpr uint32_t w_off(int l) const { return l == 0 ? 0u : 2u * w_half(0); }
    __device__ __forceinline__ constexpr int sspad(int l) const { return (npad(l) + 31) / 32 * 32; }
    __device__ __forceinline__ constexpr uint32_t ss_off(int l) const { return l == 0 ? 0u : 2u * (uint32_t)sspad(0); }
    __device__ __forceinline__ constexpr uint32_t w_total() const { return 2u * w_half(0) + 2u * w_half(1); }
    __device__ __forceinline__ constexpr uint32_t ss_total() const { return 2u * (uint32_t)sspad(0) + 2u * (uint32_t)sspad(1); }
    __device__ __forceinline__ constexpr uint32_t abuf_bytes() const { return sf_abuf_of(KP0) > sf_abuf_of(NP0) ? sf_abuf_of(KP0) : sf_abuf_of(NP0); }
    __device__ __forceinline__ constexpr uint32_t acc_cols() const { return (uint32_t)((NP0 > NP1 ? NP0 : NP1) + 31) / 32 * 32; }
};

#ifdef SF_PROFILE
__device__ long long sf_prof[16];
#define SF_T(i) do { if (prof_on) { const long long t_ = clock64(); sf_prof[i] += t_ - t_prev; t_prev = t_; } } while (0)
#else
#define SF_T(i) do { } while (0)
#endif

// Max-pool of one 32-column chunk over runs of POOL rows + mask + store.  AFTER: v holds RAW accumulators and the folded
// affine + ReLU is applied to the pooled values only (valid when the layer's scale is >= 0: fma(x, s, t) is then monotone
// non-decreasing in x, so max_i relu(fma(x_i, s, t)) == relu(fma(max_i x_i, s, t)) exactly) -- 1/POOL of the epilogue math.
template <int POOL, bool AFTER>
__device__ __forceinline__ void sf_pool_store(const SfParams &p, float (&v)[32], int lane, int q, int tile,
                                              int col0, int nout, float *xs, int wg_bar, const float *sc, const float *sh)
{
    constexpr int GP = POOL >= 32 ? 32 : POOL;
    constexpr int KEEP = 32 / GP;
    constexpr int WPG = POOL > 32 ? POOL / 32 : 1;
    warp_colmax_transpose<GP>(v, lane);                   // lane owns columns (lane % GP) * KEEP + k in v[k]
    if (POOL > 32) {                                      // groups spanning 2 or 4 warps: combine through shared memory
        xs[q * 32 + lane] = v[0];
        sf_bar_sync(wg_bar, 128);
        if ((q % WPG) == 0) {
#pragma unroll
            for (int w = 1; w < WPG; w++) v[0] = fmaxf(v[0], xs[(q + w) * 32 + lane]);
        }
        sf_bar_sync(wg_bar, 128);
        if ((q % WPG) != 0) return;
    }
    const int gg = tile * (128 / POOL) + (q * 32 + lane) / POOL;
    if ((long)gg * POOL >= p.rows) return;
    const bool masked = p.cnt && p.cnt[gg] == 0;
#pragma unroll
    for (int k = 0; k < KEEP; k++) {
        const int cc = (lane % GP) * KEEP + k;
        const int col = col0 + cc;
        if (col >= nout) continue;
        float mx = v[k];
        if (AFTER) mx = fmaxf(fmaf(mx, sc[col0 + cc], sh[col0 + cc]), 0.0f);
        mx = masked ? 0.0f : mx;
        if (p.out_f32) asm volatile("st.global.f32 [%0], %1;" ::"l"(p.out_f32 + (size_t)gg * p.ld_f32 + col), "f"(mx) : "memory");
        if (p.out_hi) {
            const __nv_bfloat16 hb = __float2bfloat16_rn(mx);
            const __nv_bfloat16 lb = __float2bfloat16_rn(mx - __bfloat162float(hb));
            asm volatile("st.global.b16 [%0], %1;" ::"l"(p.out_hi + (size_t)gg * p.ld_split + col), "h"(__bfloat16_as_ushort(hb)) : "memory");
            asm volatile("st.global.b16 [%0], %1;" ::"l"(p.out_lo + (size_t)gg * p.ld_split + col), "h"(__bfloat16_as_ushort(lb)) : "memory");
        }
    }
}

// Unit-list mode: a unit is 8 rows = 8 consecutive lanes.  Max over the unit, then atomicMax into out[group]: post-ReLU
// values are >= 0, where the unsigned order of the bit patterns is the float order (a -0.0 is folded to +0.0), and the
// caller zero-fills the output, which is also the result of a group without hits (the mask of layers_util.py:180).
template <bool AFTER>
__device__ __forceinline__ void sf_pool_atomic8(const SfParams &p, float (&v)[32], int lane, int col0, int nout, const float *sc,
                                                const float *sh, int group, bool ok)
{
    warp_colmax_transpose<8>(v, lane);                    // lane owns columns (lane % 8) * 4 + k of its unit in v[k]
    if (!ok) return;
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const int cc = (lane & 7) * 4 + k;
        const int col = col0 + cc;
        if (col >= nout) continue;
        float mx = v[k];
        if (AFTER) mx = fmaxf(fmaf(mx, sc[col0 + cc], sh[col0 + cc]), 0.0f);
        atomicMax(reinterpret_cast<unsigned int *>(p.out_f32 + (size_t)group * p.ld_f32 + col), __float_as_uint(mx) & 0x7fffffffu);
    }
}

// One work item of a layer's MMAs: rows 64*hf .. 64*hf+63 of the slot's tile, output columns n0 .. n0+W-1, over the
// whole K of layer l (full 64-wide blocks + the tail block), issued by one warpgroup as a single wgmma chain; the fp32
// result is staged row-major in acc (pitch floats per row), where the row-per-thread epilogue reads it.
template <int W, class C>
__device__ __forceinline__ void sf_mma_chunk(const C &cfg, int l, uint32_t abase, uint32_t wbase, int hf, int n0, float *acc,
                                             int pitch, int wq, int lane)
{
    float d[W / 2];
    const int nfull = cfg.nfull(l), rbt = cfg.rbt(l);
    const uint32_t npad = (uint32_t)cfg.npad(l), whalf = cfg.w_half(l);
    uint32_t accumulate = 0u;
    // descriptors advance by (bytes >> 4) in their address field; shared memory < 256 KiB: no carry out of it
    wg_fence();
#pragma unroll (C::kStatic ? 4 : 1)
    for (int kb = 0; kb < nfull; kb++) {
        const uint64_t a_hi = wg_desc(abase + (uint32_t)kb * (2u * 128u * 128u) + (uint32_t)hf * (64u * 128u), 128);
        const uint64_t b_hi = wg_desc(wbase + (uint32_t)kb * (npad * 128u) + (uint32_t)n0 * 128u, 128);
        const uint64_t a_lo = a_hi + ((128u * 128u) >> 4), b_lo = b_hi + (whalf >> 4);
#pragma unroll
        for (int kin = 0; kin < 4; kin++) {
            wg_mma3<W>(d, a_hi + 2 * kin, a_lo + 2 * kin, b_hi + 2 * kin, b_lo + 2 * kin, accumulate);
            accumulate = 1u;
        }
    }
    if (rbt) {
        const uint64_t a_hi = wg_desc(abase + (uint32_t)nfull * (2u * 128u * 128u) + (uint32_t)hf * (64u * (uint32_t)rbt), rbt);
        const uint64_t b_hi = wg_desc(wbase + (uint32_t)nfull * (npad * 128u) + (uint32_t)n0 * (uint32_t)rbt, rbt);
        const uint64_t a_lo = a_hi + ((128u * (uint32_t)rbt) >> 4), b_lo = b_hi + (whalf >> 4);
        const int nt = rbt == 128 ? 3 : (rbt >> 5);              // 16-wide k-steps of the tail block
#pragma unroll (C::kStatic ? 3 : 1)
        for (int kin = 0; kin < nt; kin++) {
            wg_mma3<W>(d, a_hi + 2 * kin, a_lo + 2 * kin, b_hi + 2 * kin, b_lo + 2 * kin, accumulate);
            accumulate = 1u;
        }
    }
    wg_commit();
    wg_wait<0>();
    const int r0 = hf * 64 + wq * 16 + (lane >> 2), c = n0 + 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < W / 8; j++) {
        *reinterpret_cast<float2 *>(acc + r0 * pitch + c + 8 * j) = make_float2(d[4 * j], d[4 * j + 1]);
        *reinterpret_cast<float2 *>(acc + (r0 + 8) * pitch + c + 8 * j) = make_float2(d[4 * j + 2], d[4 * j + 3]);
    }
}

// SLOTS tiles in flight per CTA, WG warpgroups (128 threads) working on each: the warpgroups of a slot split the
// 16-byte chunks of the gather and the 32-column chunks of every epilogue between them.  C: shape policy (above).
template <class C, int SLOTS, int WG>
__global__ void __launch_bounds__(SF_THREADS * SLOTS * WG, SLOTS * WG == 1 ? 6 : 1)
sa_fused_kernel(const SfParams p)
{
    const C cfg(p);
    // pointers inside the by-value parameter struct carry no address space: tell the compiler they are global
    __builtin_assume(__isGlobal(p.xyz)); __builtin_assume(__isGlobal(p.new_xyz)); __builtin_assume(__isGlobal(p.idx));
    __builtin_assume(p.points == nullptr || __isGlobal(p.points)); __builtin_assume(p.cnt == nullptr || __isGlobal(p.cnt));
    __builtin_assume(__isGlobal(p.w_blob)); __builtin_assume(__isGlobal(p.ss_blob));
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    // 1 KiB alignment by pointer arithmetic on the __shared__ array (an integer round-trip would demote every access
    // through these pointers to generic LD/ST with 64-bit address math)
    uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
    uint8_t *wsm = smem + (size_t)SLOTS * cfg.abuf_bytes();  // weight images (1024-aligned: buffers are multiples of 1 KiB)
    float *ss = reinterpret_cast<float *>(wsm + cfg.w_total());
    float *wxs = ss + cfg.ss_total();                    // [3][kp0] hoisted mode: Wx * s1, zero beyond c
    const int pitch = (int)cfg.acc_cols() + 4;           // staged accumulator row: +4 floats keep the accesses conflict-free
    float *acc_all = wxs + 3 * cfg.kp(0);                // [SLOTS][128][pitch], 16-byte aligned (kp0 % 16 == 0)

    __shared__ unsigned long long w_bar;
    __shared__ float xs_all[SLOTS * WG][4 * 32];

    constexpr int NT = SF_THREADS * SLOTS * WG, ST = SF_THREADS * WG;     // threads per CTA / per slot
    constexpr int U = WG == 1 ? 4 : (WG == 2 ? 3 : 2);   // gather chunks in flight per thread
    const int tid = threadIdx.x, lane = tid & 31, q = (tid >> 5) & 3;
    const int slot = tid / ST, wg = (tid >> 7) % WG;
    const int r = tid & 127;                             // row of the slot's tile this thread works on
    // warp-uniform copies (shfl) so that descriptors are computed on the uniform datapath
    const int slot_u = __shfl_sync(0xffffffffu, slot, 0), wg_u = __shfl_sync(0xffffffffu, wg, 0);
    const int slot_bar = 1 + slot, wg_bar = 1 + SLOTS + slot * WG + wg;
    uint8_t *buf = smem + (size_t)slot * cfg.abuf_bytes();   // the slot's operand buffer (every layer, in place)
    float *xs = xs_all[slot * WG + wg];
    float *acc = acc_all + (size_t)slot * 128 * pitch;
    const int kp0 = cfg.kp(0);

    if (tid == 0) {
        mbar_init(smem_u32(&w_bar), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        mbar_arrive_expect_tx(smem_u32(&w_bar), cfg.w_total());
        bulk_g2s(smem_u32(wsm), p.w_blob, cfg.w_total(), smem_u32(&w_bar));
    }
    for (uint32_t i = tid; i < cfg.ss_total(); i += NT) ss[i] = __ldg(p.ss_blob + i);
    if (cfg.hoist())
        for (int i = tid; i < 3 * kp0; i += NT) {
            const int a3 = i / kp0, k = i - a3 * kp0;
            wxs[i] = k < cfg.c() ? __ldg(p.wx + a3 * cfg.c() + k) : 0.0f;
        }
    // staged columns a layer narrower than acc_cols leaves unwritten are multiplied by a zero scale: keep them finite
    for (int i = tid; i < SLOTS * 128 * pitch; i += NT) acc_all[i] = 0.0f;
    __syncthreads();
    mbar_wait_cta(smem_u32(&w_bar), 0);                  // weights landed (async proxy writes, read by wgmma only)

#ifdef SF_PROFILE
    const bool prof_on = blockIdx.x == 0 && (tid % ST) == 0 && slot == 0;
    long long t_prev = clock64();
#endif
    const int k0 = cfg.hoist() ? cfg.c() : cfg.c() + 3;  // valid operand columns
    const int src_pitch = cfg.hoist() ? p.ldz : cfg.c();
    const bool vec = (cfg.c() & 3) == 0 && (src_pitch & 3) == 0; // source rows are 16-byte aligned: float4 gathers

    const int tile0 = blockIdx.x * SLOTS + slot, tstep = gridDim.x * SLOTS;
    const int *units = p.units;
    __builtin_assume(units == nullptr || __isGlobal(units));
    const bool compact = units != nullptr;
    const int nunits = compact ? __ldg(units) : 0;
    const int tiles = compact ? (nunits + 15) >> 4 : p.tiles;
    // neighbour index (and, in unit-list mode, unit descriptor) of this thread's row, fetched one tile ahead
    // (rows < 2^31: checked by the launcher)
    auto fetch = [&](int t, int &desc, int &a) {
        desc = -1; a = 0;
        if (t >= tiles) return;
        if (compact) {
            const int ui = t * 16 + (r >> 3);
            if (ui < nunits) {
                desc = __ldg(units + 1 + ui);
                a = __ldg(p.idx + (size_t)(desc >> 4) * (uint32_t)cfg.ns() + (uint32_t)(((desc & 15) << 3) + (r & 7)));
            }
        } else if ((long)t * 128 + r < p.rows) {
            desc = 0;
            a = __ldg(p.idx + (size_t)t * 128u + r);
        }
    };
    int d_next, a_next;
    fetch(tile0, d_next, a_next);
    int my_group = 0;                                                  // unit-list mode: the group this thread's row belongs to
    bool my_ok = false;
    for (int tile = tile0; tile < tiles; tile += tstep) {
        // ---- gather + centre-subtract + concat + split -> buf (layers_util.py:157-165)
        {
            const uint32_t row = (uint32_t)tile * 128u + (uint32_t)r;
            const bool ok = d_next >= 0;
            const uint32_t qi = !ok ? 0u : (compact ? (uint32_t)(d_next >> 4) : row / (uint32_t)cfg.ns());    // == scene*m + query
            const uint32_t scene = qi / (uint32_t)p.m;
            const int a = a_next;
            my_group = (int)qi; my_ok = ok;
            fetch(tile + tstep, d_next, a_next);
            const float *src_f = p.points + ((size_t)scene * p.n + a) * src_pitch;
            const float *src_x = p.xyz + ((size_t)scene * p.n + a) * 3;
            const float *ctr = p.new_xyz + (size_t)qi * 3;
            const int nchunk = kp0 >> 3;
            const SfRowMap map0(r, cfg.nfull(0), cfg.rbt(0));
            float dx = 0.0f, dy = 0.0f, dz = 0.0f;
            if (cfg.hoist() && ok) {
                dx = __ldg(src_x) - __ldg(ctr); dy = __ldg(src_x + 1) - __ldg(ctr + 1); dz = __ldg(src_x + 2) - __ldg(ctr + 2);
            }
#pragma unroll (C::kStatic ? 4 : 1)
            for (int cg0 = wg * U; cg0 < nchunk; cg0 += WG * U) {     // U chunks of 8 columns in flight per thread
                float f[U][8];
#pragma unroll
                for (int u = 0; u < U; u++) {
                    const int kb = (cg0 + u) * 8;
                    if (vec && ok && kb + 8 <= cfg.c()) {
                        const float4 lo4 = __ldg(reinterpret_cast<const float4 *>(src_f + kb));
                        const float4 hi4 = __ldg(reinterpret_cast<const float4 *>(src_f + kb + 4));
                        f[u][0] = lo4.x; f[u][1] = lo4.y; f[u][2] = lo4.z; f[u][3] = lo4.w;
                        f[u][4] = hi4.x; f[u][5] = hi4.y; f[u][6] = hi4.z; f[u][7] = hi4.w;
                    } else {
#pragma unroll
                        for (int e = 0; e < 8; e++) {
                            const int k = kb + e;
                            float val = 0.0f;
                            if (ok) {
                                if (k < cfg.c()) val = __ldg(src_f + k);
                                else if (k < k0) val = __ldg(src_x + (k - cfg.c())) - __ldg(ctr + (k - cfg.c()));   // never in hoisted mode
                            }
                            f[u][e] = val;
                        }
                    }
                }
#pragma unroll
                for (int u = 0; u < U; u++) {
                    if (cg0 + u >= nchunk) break;
                    if (cfg.hoist()) {                                 // relu(z + d . Wx'); padded columns and rows stay 0
                        const float *w = wxs + (cg0 + u) * 8;
#pragma unroll
                        for (int e4 = 0; e4 < 8; e4 += 4) {
                            const float4 w0 = *reinterpret_cast<const float4 *>(w + e4);
                            const float4 w1 = *reinterpret_cast<const float4 *>(w + kp0 + e4);
                            const float4 w2 = *reinterpret_cast<const float4 *>(w + 2 * kp0 + e4);
                            f[u][e4 + 0] = fmaxf(fmaf(dz, w2.x, fmaf(dy, w1.x, fmaf(dx, w0.x, f[u][e4 + 0]))), 0.0f);
                            f[u][e4 + 1] = fmaxf(fmaf(dz, w2.y, fmaf(dy, w1.y, fmaf(dx, w0.y, f[u][e4 + 1]))), 0.0f);
                            f[u][e4 + 2] = fmaxf(fmaf(dz, w2.z, fmaf(dy, w1.z, fmaf(dx, w0.z, f[u][e4 + 2]))), 0.0f);
                            f[u][e4 + 3] = fmaxf(fmaf(dz, w2.w, fmaf(dy, w1.w, fmaf(dx, w0.w, f[u][e4 + 3]))), 0.0f);
                        }
                    }
                    uint32_t hw[4], lw[4], lo_off;
#pragma unroll
                    for (int t = 0; t < 4; t++) sf_split_pair(f[u][2 * t], f[u][2 * t + 1], hw[t], lw[t]);
                    const uint32_t off = map0.chunk(cg0 + u, &lo_off);
                    *reinterpret_cast<uint4 *>(buf + off) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
                    *reinterpret_cast<uint4 *>(buf + off + lo_off) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
                }
            }
        }
        SF_T(0);                                                       // gather
#pragma unroll (C::kStatic ? SF_MAX_LAYERS : 1)
        for (int l = 0; l < cfg.nl(); l++) {
            // operand written with ordinary stores -> make it visible to the tensor-core (async) proxy; the barrier also
            // orders the previous layer's staged-accumulator reads before this layer's MMAs overwrite the staging
            sf_fence_async_smem();
            sf_bar_sync(slot_bar, ST);
            SF_T(1 + 4 * l);                                           // barrier
            {
                // work items (64-row half, <= 64-column chunk) of this layer, round robin over the slot's warpgroups: one
                // wgmma per k-step covers the whole chunk width; chunk widths are 64 but for a 16 / 32 / 48 tail
                const uint32_t abase = smem_u32(smem) + (uint32_t)slot_u * cfg.abuf_bytes();
                const uint32_t wbase = smem_u32(wsm) + cfg.w_off(l);
                const int npad = cfg.npad(l), nch = (npad + 63) / 64;
#pragma unroll (C::kStatic ? 8 : 1)
                for (int item = wg_u; item < 2 * nch; item += WG) {
                    const int hf = item & 1, n0 = (item >> 1) * 64, w = npad - n0 < 64 ? npad - n0 : 64;
                    if (w == 64) sf_mma_chunk<64>(cfg, l, abase, wbase, hf, n0, acc, pitch, q, lane);
                    else if (w == 48) sf_mma_chunk<48>(cfg, l, abase, wbase, hf, n0, acc, pitch, q, lane);
                    else if (w == 32) sf_mma_chunk<32>(cfg, l, abase, wbase, hf, n0, acc, pitch, q, lane);
                    else sf_mma_chunk<16>(cfg, l, abase, wbase, hf, n0, acc, pitch, q, lane);
                }
            }
            SF_T(2 + 4 * l);                                           // MMAs
            sf_bar_sync(slot_bar, ST);                                 // every MMA of the tile done: staging complete, buf free
            SF_T(3 + 4 * l);                                           // MMA wait
            // ---- epilogue of layer l
            const float *sc = ss + cfg.ss_off(l);
            const float *sh = sc + cfg.sspad(l);
            const bool last = l == cfg.nl() - 1;
            const bool pool_first = last && p.pool_first;              // last layer with scale >= 0: pool raw accumulators
            const SfRowMap mapn(r, last ? 0 : cfg.nfull(l + 1), last ? 32 : cfg.rbt(l + 1));
            const int nchunks = (cfg.npad(l) + 31) / 32;
#pragma unroll (C::kStatic ? 4 : 1)
            for (int ci = wg; ci < nchunks; ci += WG) {
                const int c0 = ci * 32;
                float rr[32];
#pragma unroll
                for (int j4 = 0; j4 < 32; j4 += 4) {
                    const float4 a4 = *reinterpret_cast<const float4 *>(acc + r * pitch + c0 + j4);
                    rr[j4] = a4.x; rr[j4 + 1] = a4.y; rr[j4 + 2] = a4.z; rr[j4 + 3] = a4.w;
                }
                float v[32];
                if (pool_first) {
#pragma unroll
                    for (int j = 0; j < 32; j++) v[j] = rr[j];
                } else {
#pragma unroll
                    for (int j4 = 0; j4 < 32; j4 += 4) {              // scale/shift are zero-padded to 32-column chunks
                        const float4 s4 = *reinterpret_cast<const float4 *>(sc + c0 + j4);
                        const float4 h4 = *reinterpret_cast<const float4 *>(sh + c0 + j4);
                        v[j4 + 0] = fmaxf(fmaf(rr[j4 + 0], s4.x, h4.x), 0.0f);   // every conv has a ReLU
                        v[j4 + 1] = fmaxf(fmaf(rr[j4 + 1], s4.y, h4.y), 0.0f);
                        v[j4 + 2] = fmaxf(fmaf(rr[j4 + 2], s4.z, h4.z), 0.0f);
                        v[j4 + 3] = fmaxf(fmaf(rr[j4 + 3], s4.w, h4.w), 0.0f);
                    }
                }
                if (!last) {
#pragma unroll
                    for (int j8 = 0; j8 < 32; j8 += 8) {
                        if (c0 + j8 >= cfg.kp(l + 1)) break;
                        uint32_t hw[4], lw[4], lo_off;
#pragma unroll
                        for (int t = 0; t < 4; t++) sf_split_pair(v[j8 + 2 * t], v[j8 + 2 * t + 1], hw[t], lw[t]);
                        const uint32_t off = mapn.chunk((c0 + j8) >> 3, &lo_off);
                        *reinterpret_cast<uint4 *>(buf + off) = make_uint4(hw[0], hw[1], hw[2], hw[3]);
                        *reinterpret_cast<uint4 *>(buf + off + lo_off) = make_uint4(lw[0], lw[1], lw[2], lw[3]);
                    }
                } else if (compact) {
                    if (pool_first) sf_pool_atomic8<true>(p, v, lane, c0, cfg.nout(l), sc, sh, my_group, my_ok);
                    else sf_pool_atomic8<false>(p, v, lane, c0, cfg.nout(l), sc, sh, my_group, my_ok);
                } else if (pool_first) {
                    switch (cfg.ns()) {
                        case 8: sf_pool_store<8, true>(p, v, lane, q, tile, c0, cfg.nout(l), xs, wg_bar, sc, sh); break;
                        case 16: sf_pool_store<16, true>(p, v, lane, q, tile, c0, cfg.nout(l), xs, wg_bar, sc, sh); break;
                        case 32: sf_pool_store<32, true>(p, v, lane, q, tile, c0, cfg.nout(l), xs, wg_bar, sc, sh); break;
                        case 64: sf_pool_store<64, true>(p, v, lane, q, tile, c0, cfg.nout(l), xs, wg_bar, sc, sh); break;
                        default: sf_pool_store<128, true>(p, v, lane, q, tile, c0, cfg.nout(l), xs, wg_bar, sc, sh); break;
                    }
                } else {
                    switch (cfg.ns()) {
                        case 8: sf_pool_store<8, false>(p, v, lane, q, tile, c0, cfg.nout(l), xs, wg_bar, sc, sh); break;
                        case 16: sf_pool_store<16, false>(p, v, lane, q, tile, c0, cfg.nout(l), xs, wg_bar, sc, sh); break;
                        case 32: sf_pool_store<32, false>(p, v, lane, q, tile, c0, cfg.nout(l), xs, wg_bar, sc, sh); break;
                        case 64: sf_pool_store<64, false>(p, v, lane, q, tile, c0, cfg.nout(l), xs, wg_bar, sc, sh); break;
                        default: sf_pool_store<128, false>(p, v, lane, q, tile, c0, cfg.nout(l), xs, wg_bar, sc, sh); break;
                    }
                }
            }
            SF_T(4 + 4 * l);                                           // epilogue
        }
    }

}

}  // namespace ssd3d

using namespace ssd3d;

// Operand layout of a layer with padded K = kp: nfull 64-wide k-blocks of 128-byte rows + a tail block whose rows
// are 32 / 64 / 128 bytes for a remainder of 16 / 32 / 48 columns (must match params._k_blocks).
static void sf_k_blocks(int kp, int *nfull, int *rbt)
{
    *nfull = kp / 64;
    const int rem = kp % 64;
    *rbt = rem == 0 ? 0 : (rem <= 16 ? 32 : (rem <= 32 ? 64 : 128));
}
static size_t sf_abuf_bytes(int kp)                       // { hi | lo } tiles of 128 rows per block, 1 KiB granular
{
    int nfull, rbt;
    sf_k_blocks(kp, &nfull, &rbt);
    return ((size_t)nfull * 2 * 128 * 128 + (size_t)2 * 128 * rbt + 1023) / 1024 * 1024;
}
static size_t sf_wimg_bytes(int kp, int npad)              // one half (hi or lo) of a layer's weight image
{
    int nfull, rbt;
    sf_k_blocks(kp, &nfull, &rbt);
    return (size_t)npad * (nfull * 128 + rbt);
}

struct SfPlan { size_t abuf, acc, w, ssf; int maxn; };
static bool sf_plan(int k_in, int nl, const int *nout, SfPlan *pl)      // k_in: columns of the first operand
{
    if (nl < 1 || nl > SF_MAX_LAYERS) return false;
    pl->abuf = 0; pl->w = 0; pl->ssf = 0; pl->maxn = 32;
    int kp = (k_in + 15) / 16 * 16;
    pl->ssf = 3 * (size_t)kp;                               // room for the hoisted mode's Wx table
    for (int l = 0; l < nl; l++) {
        const int npad = (nout[l] + 15) / 16 * 16;
        if (npad > 256) return false;
        const size_t a = sf_abuf_bytes(kp);
        if (a > pl->abuf) pl->abuf = a;
        pl->w += 2 * sf_wimg_bytes(kp, npad);
        pl->ssf += (size_t)2 * ((npad + 31) / 32 * 32);
        if (npad > pl->maxn) pl->maxn = npad;
        kp = npad;
    }
    pl->acc = (size_t)128 * ((pl->maxn + 31) / 32 * 32 + 4) * sizeof(float);   // staged accumulator of one slot
    return true;
}
static size_t sf_total(const SfPlan &pl, int slots) { return slots * (pl.abuf + pl.acc) + pl.w + pl.ssf * sizeof(float) + 1024; }
constexpr size_t SF_SMEM_MAX = 226 * 1024;
constexpr size_t SF_SMALL = 72 * 1024;                     // <= this: single-slot, single-warpgroup CTAs, several per SM

// Developer build only (-DSSD3D_DEV_HOOKS, csrc/ssd3d_dev.h): override the slot / warpgroup shape from a probe script.
// The shipped library has no such state.
#ifdef SSD3D_DEV_HOOKS
static int g_sf_slots = 0, g_sf_wg = 0, g_sf_dynamic = 0;
extern "C" void ssd3d_dev_set_fused(int slots, int wg) { g_sf_slots = slots; g_sf_wg = wg; }
extern "C" void ssd3d_dev_set_fused_dynamic(int on) { g_sf_dynamic = on; }   // force the run-time-shape kernel (A/B timing)
#else
constexpr int g_sf_slots = 0, g_sf_wg = 0, g_sf_dynamic = 0;
#endif

// Slots per CTA for a stack: 1 for small stacks (several CTAs per SM), else as many as fit one SM (<= 3).
static int sf_slots(const SfPlan &pl)
{
    if (sf_total(pl, 1) <= SF_SMALL) return 1;
    int s = g_sf_slots > 0 ? (g_sf_slots > 4 ? 4 : g_sf_slots) : 3;
    // the kernel's static shared memory (xs_all: 512 bytes per warpgroup, two per slot) counts against the same limit
    while (s > 1 && sf_total(pl, s) + (size_t)s * 2 * 512 > SF_SMEM_MAX) s--;
    return s;
}

// Shared-memory bytes of the fused kernel for a layer stack, or 0 when it cannot hold it.
extern "C" size_t ssd3d_sa_fused_smem(int c, int nl, const int *nout)
{
    SfPlan pl;
    if (!sf_plan(c + 3, nl, nout, &pl)) return 0;
    const size_t total = sf_total(pl, sf_slots(pl));
    return total <= SF_SMEM_MAX ? total : 0;
}

template <class C, int SLOTS, int WG>
static cudaError_t sf_launch(const SfParams &p, size_t smem, int per_sm, cudaStream_t stream)
{
    cudaError_t e = cudaFuncSetAttribute((const void *)sa_fused_kernel<C, SLOTS, WG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    const int ctas = (p.tiles + SLOTS - 1) / SLOTS;
    int grid = kNumSMs * per_sm;
    if (grid > ctas) grid = ctas;
    sa_fused_kernel<C, SLOTS, WG><<<grid, SF_THREADS * SLOTS * WG, smem, stream>>>(p);
    return cudaSuccess;
}

// The hoisted two-conv stacks of the shipped 3DSSD configuration (configs/kitti/3dssd/3dssd.yaml:47-52) have compile-time
// twins of the kernel: layer 1 [16 -> 16 -> 32] x32 and [32 -> 32 -> 64] x64 neighbours, layer 2 [64 -> 64 -> 128] x32 and
// [64 -> 96 -> 128] x64.  Returns false when (shape, slots, warpgroups) has no twin: the caller takes the dynamic kernel.
static bool sf_launch_static(const SfParams &p, int slots, int wg, size_t smem, int per_sm, cudaStream_t st, cudaError_t *e)
{
    if (!p.hoist || p.nl != 2) return false;
    const int k0 = p.c, n0 = p.nout[0], n1 = p.nout[1], ns = p.ns;
    if (slots == 1 && wg == 1) {
        if (k0 == 16 && n0 == 16 && n1 == 32 && ns == 32) { *e = sf_launch<SfStat<16, 16, 32, 32>, 1, 1>(p, smem, per_sm, st); return true; }
        if (k0 == 32 && n0 == 32 && n1 == 64 && ns == 64) { *e = sf_launch<SfStat<32, 32, 64, 64>, 1, 1>(p, smem, per_sm, st); return true; }
    }
    if (slots == 1 && wg == 2) {
        if (k0 == 64 && n0 == 64 && n1 == 128 && ns == 32) { *e = sf_launch<SfStat<64, 64, 128, 32>, 1, 2>(p, smem, per_sm, st); return true; }
        if (k0 == 64 && n0 == 96 && n1 == 128 && ns == 64) { *e = sf_launch<SfStat<64, 96, 128, 64>, 1, 2>(p, smem, per_sm, st); return true; }
    }
    return false;
}

// w_blob: per layer { hi image | lo image }, each image = k-blocks of [npad x (64 | tail)] bf16 in the canonical
// K-major swizzled layout (built by params.FusedStack); ss_blob: per layer { scale[sspad] | shift[sspad] }.
// wx != NULL selects the hoisted mode: `points` is the per-point table z (pitch ldz), c its width.
static int sa_mlp_fused_impl(int b, int n, int c, int m, int nsample, const float *xyz, const float *points, int ldz,
                             const float *wx, const float *new_xyz, const int *idx, const int *pts_cnt, const int *units, int nl,
                             const int *nout, const void *w_blob, const float *ss_blob, int last_scale_nonneg,
                             float *out_f32, int ld_f32, void *out_hi, void *out_lo, int ld_split, ssd3d_stream_t stream)
{
    const bool hoist = wx != nullptr;
    SSD3D_REQUIRE(b >= 0 && n > 0 && m >= 0 && c >= 0, "sa_mlp_fused: bad shape");
    SSD3D_REQUIRE(nsample == 8 || nsample == 16 || nsample == 32 || nsample == 64 || nsample == 128,
                  "sa_mlp_fused: nsample=%d must be one of 8, 16, 32, 64, 128", nsample);
    SSD3D_REQUIRE(xyz && new_xyz && idx && w_blob && ss_blob && (points || c == 0), "sa_mlp_fused: null pointer");
    SSD3D_REQUIRE(!hoist || (c > 0 && ldz >= c), "sa_mlp_fused_hoisted: bad table shape n1=%d ldz=%d", c, ldz);
    SSD3D_REQUIRE(out_f32 || (out_hi && out_lo), "sa_mlp_fused: no output requested");
    SSD3D_REQUIRE(!units || (out_f32 && !out_hi && !out_lo), "sa_mlp_fused: a unit list combines through atomicMax on the (zero-filled) fp32 output only");
    SSD3D_REQUIRE((reinterpret_cast<uintptr_t>(w_blob) & 15u) == 0, "sa_mlp_fused: weight blob must be 16-byte aligned");
    SSD3D_REQUIRE(!points || (c & 3) || (hoist && (ldz & 3)) || (reinterpret_cast<uintptr_t>(points) & 15u) == 0,
                  "sa_mlp_fused: points must be 16-byte aligned when c is a multiple of 4");
    const int k_in = hoist ? c : c + 3;
    SfPlan pl;
    const bool planned = sf_plan(k_in, nl, nout, &pl);
    const int slots = planned ? sf_slots(pl) : 0;
    const size_t smem = planned ? sf_total(pl, slots) : 0;
    if (!planned || smem > SF_SMEM_MAX) { set_error("sa_mlp_fused: layer stack does not fit shared memory"); return SSD3D_ERR_UNSUPPORTED; }
    SfParams p = {};
    p.n = n; p.c = c; p.m = m; p.ns = nsample;
    p.rows = (long)b * m * nsample;
    if (p.rows == 0) return 0;
    SSD3D_REQUIRE(p.rows < (1L << 31) - 128, "sa_mlp_fused: too many grouped rows (%ld)", p.rows);
    p.tiles = (int)((p.rows + 127) / 128);
    p.xyz = xyz; p.points = points; p.new_xyz = new_xyz; p.idx = idx; p.cnt = pts_cnt; p.units = units;
    p.hoist = hoist ? 1 : 0; p.ldz = ldz; p.wx = wx;
    p.pool_first = last_scale_nonneg ? 1 : 0;
    p.nl = nl;
    int kprev = (k_in + 15) / 16 * 16;
    uint32_t woff = 0, ssoff = 0;
    for (int l = 0; l < nl; l++) {
        p.kp[l] = kprev;
        p.nout[l] = nout[l];
        p.npad[l] = (nout[l] + 15) / 16 * 16;
        sf_k_blocks(p.kp[l], &p.nfull[l], &p.rbt[l]);
        p.w_off[l] = woff;
        p.w_half[l] = (uint32_t)sf_wimg_bytes(p.kp[l], p.npad[l]);
        woff += 2 * p.w_half[l];
        p.ss_off[l] = ssoff;
        p.sspad[l] = (p.npad[l] + 31) / 32 * 32;
        ssoff += 2 * p.sspad[l];
        kprev = p.npad[l];
    }
    p.w_total = woff; p.ss_total = ssoff;
    p.w_blob = (const uint8_t *)w_blob; p.ss_blob = ss_blob;
    p.abuf_bytes = (uint32_t)pl.abuf;
    p.acc_cols = (uint32_t)(pl.maxn + 31) / 32 * 32;
    p.out_f32 = out_f32; p.ld_f32 = ld_f32;
    p.out_hi = (__nv_bfloat16 *)out_hi; p.out_lo = (__nv_bfloat16 *)out_lo; p.ld_split = ld_split;

    // one warpgroup per slot for small stacks (several CTAs per SM), two when a slot needs most of an SM's shared memory
    const bool small = slots == 1 && smem <= SF_SMALL;
    const int wg = g_sf_wg > 0 ? g_sf_wg : (small ? 1 : 2);
    // resident CTAs per SM: bounded by shared memory and, for single-warpgroup CTAs, registers
    int per_sm = 1;
    if (slots == 1 && wg == 1) {
        per_sm = (int)((227 * 1024) / (smem + 1024));
        if (per_sm < 1) per_sm = 1;
        if (per_sm > 6) per_sm = 6;                                   // 6 x 128 threads x 80 registers
    }
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaSuccess;
    if (g_sf_dynamic || !sf_launch_static(p, slots, wg, smem, per_sm, st, &e))
        e = slots == 1 ? (wg == 1 ? sf_launch<SfDyn, 1, 1>(p, smem, per_sm, st) : sf_launch<SfDyn, 1, 2>(p, smem, per_sm, st))
          : slots == 2 ? (wg == 4 ? sf_launch<SfDyn, 2, 4>(p, smem, per_sm, st) : wg == 1 ? sf_launch<SfDyn, 2, 1>(p, smem, per_sm, st)
                                                                                           : sf_launch<SfDyn, 2, 2>(p, smem, per_sm, st))
          : slots == 3 ? (wg == 1 ? sf_launch<SfDyn, 3, 1>(p, smem, per_sm, st) : sf_launch<SfDyn, 3, 2>(p, smem, per_sm, st))
                       : sf_launch<SfDyn, 4, 1>(p, smem, per_sm, st);
    if (e != cudaSuccess) return cuda_status(e, "sa_mlp_fused attr");
#ifdef SF_PROFILE
    {
        long long h[16];
        cudaDeviceSynchronize();
        cudaMemcpyFromSymbol(h, sf_prof, sizeof(h));
        fprintf(stderr, "sf_prof slots=%d tiles=%d:", slots, p.tiles);
        for (int i = 0; i < 13; i++) fprintf(stderr, " %lld", h[i]);
        fprintf(stderr, "\n");
        memset(h, 0, sizeof(h));
        cudaMemcpyToSymbol(sf_prof, h, sizeof(h));
    }
#endif
    SSD3D_LAUNCH_CHECK("sa_fused_kernel");
}

extern "C" int ssd3d_sa_mlp_fused(int b, int n, int c, int m, int nsample, const float *xyz, const float *points,
                                  const float *new_xyz, const int *idx, const int *pts_cnt, const int *units, int nl,
                                  const int *nout, const void *w_blob, const float *ss_blob, int last_scale_nonneg,
                                  float *out_f32, int ld_f32, void *out_hi, void *out_lo, int ld_split, ssd3d_stream_t stream)
{
    return sa_mlp_fused_impl(b, n, c, m, nsample, xyz, points, c, nullptr, new_xyz, idx, pts_cnt, units, nl, nout, w_blob, ss_blob,
                             last_scale_nonneg, out_f32, ld_f32, out_hi, out_lo, ld_split, stream);
}

// The fused SA scale with its first conv hoisted (see ssd3d_linear_tc_hoisted): z[b,n,ldz] per-point table (this scale's
// n1 columns start at z), wx = Wx*s1 as [3][n1]; the stack (w_blob / ss_blob / nout) starts at the scale's SECOND conv.
extern "C" int ssd3d_sa_mlp_fused_hoisted(int b, int n, int n1, int m, int nsample, const float *xyz, const float *z, int ldz,
                                          const float *wx, const float *new_xyz, const int *idx, const int *pts_cnt,
                                          const int *units, int nl, const int *nout, const void *w_blob, const float *ss_blob,
                                          int last_scale_nonneg, float *out_f32, int ld_f32, void *out_hi, void *out_lo,
                                          int ld_split, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(z && wx, "sa_mlp_fused_hoisted: null table pointer");
    return sa_mlp_fused_impl(b, n, n1, m, nsample, xyz, z, ldz, wx, new_xyz, idx, pts_cnt, units, nl, nout, w_blob, ss_blob,
                             last_scale_nonneg, out_f32, ld_f32, out_hi, out_lo, ld_split, stream);
}
