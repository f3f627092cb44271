// sa_fused.cu -- one SA scale in ONE kernel: gather + concat + (conv+BN+ReLU) x L + max-pool + mask, wgmma.
//
// Fuses lib/utils/layers_util.py:157-180 of the reference (idx masking, 2x group_point, centre subtraction, concat,
// the conv2d/bias/BN/ReLU stack, reduce_max, mask multiply -- ~25 TF kernels per scale, each streaming [B,M,K,C]
// through HBM) for the layers whose weights fit in shared memory (3DSSD layer1/layer2: 93% of the grouped rows).
// Nothing but the neighbour indices, the gathered source rows (L2-resident) and the pooled [B,M,C3] result touches
// global memory; activations go wgmma registers -> epilogue on the accumulator fragments -> shared memory (already split
// in bf16 hi/lo and already in the swizzled K-major layout the next layer's wgmma descriptors expect).
//
// Per CTA: S "slots" of 128*WG threads, each working on one 128-row tile (= 128/K neighbour groups) at a time:
//   weights of all layers (hi+lo images, pre-swizzled on the host) are bulk-copied to shared memory once and shared
//   by the slots; each slot owns ONE operand buffer and loops over tiles.  The buffer keeps the two 64-row halves of the
//   tile in separate byte ranges for every layer (SfRowMap), so a row half is a pipeline of its own:
//   gather+split of the half -> [fence.proxy.async + warpgroup barrier] -> the layer's MMAs for the half (one wgmma chain
//   per <= 64-column chunk, all chunks held in registers) -> epilogue on the fragments (scale/shift/ReLU, split) written
//   IN PLACE over the half's operand, which its retired MMAs no longer need -> ... -> last layer: one chunk at a time,
//   max-pooled on the fragment (8-row units by a shuffle butterfly; wider groups meet in a 4 KiB per-slot exchange).
// Small stacks (layer1) run S=1 with one warpgroup that takes the two halves in turn, several CTAs per SM; larger
// stacks (layer2) run one CTA per SM with two slots of two warpgroups, each warpgroup owning one row half, so that no
// barrier wider than a warpgroup separates the layers (only a pool of 128 rows meets the other half).
// Hoisted mode (SfParams::hoist): the scale's first conv has been moved to a per-point table z (include/ssd3d.h,
// ssd3d_sa_mlp_fused_hoisted); the gather then builds relu(z[idx] + (xyz[idx] - centre) . Wx') and the stack starts at
// the second conv.
// Unit-list mode (SfParams::units, round 2): a neighbour list repeats its first hit beyond pts_cnt
// (grouping/tf_grouping_g.cu:245-248) and the copies cannot change the max-pool, so a tile is made of 16 listed 8-row units
// (the ball query lists ceil(cnt / 8) units per non-empty group) instead of 128 consecutive rows; each unit is pooled by the
// shuffle butterfly and the units of a group meet through atomicMax on the non-negative fp32 result, which the caller
// zero-fills (= the cnt == 0 mask of layers_util.py:180).  Same bits as the dense schedule, 4-8x fewer rows on KITTI-like
// clouds (DESIGN.md section 3.4).  Lists of 4-row units (SfParams::unit_lg == 2, nsample <= 64) put 32 units in a tile and
// pool each with one butterfly step fewer; groups of 1-4 hits then convolve 4 rows instead of 8.
//
// Precision: same bf16 hi/lo split and 3-MMA scheme as mlp_tc.cu.
#include <cuda_bf16.h>
#include <cstdio>
#include <cstring>
#include <type_traits>

#include "common.cuh"
#include "operand.cuh"
#include "pool.cuh"
#include "wgmma.cuh"

namespace ssd3d {

constexpr int SF_THREADS = 128;
constexpr int SF_MAX_LAYERS = 3;
constexpr int SF_MAX_NCH = 4;                // <= 64-column chunks of a layer (npad <= 256)
constexpr int SF_XS_FLOATS = 16 * 64;        // pooled-value exchange of a slot: [8-row slab][chunk column]

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
    int unit_lg;                     // log2 of the rows per unit: 3 (8-row units) or 2 (4-row units)
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
    float *out_f32; int ld_f32;
    __nv_bfloat16 *out_hi, *out_lo; int ld_split;
    int pool_first;                  // caller guarantees scale >= 0 in the LAST layer: pool raw accumulators, affine after
};

// Where row r of a 128-row operand tile lives.  The buffer holds the two 64-row halves of the tile one after the other,
// half_bytes (half the buffer of the widest layer) apart, so that rows 64h .. 64h+63 of EVERY layer stay inside half h's
// bytes and the warpgroup running a half can overwrite them with the next layer's operand as soon as its own MMAs have
// retired.  A half is laid out as k-blocks of { hi tile | lo tile } (64 rows x rb bytes each), each tile in the canonical
// K-major swizzled layout of span rb: 16-byte chunk j of row r sits at chunk j ^ ((r >> log2(128/rb)) & (rb/16 - 1)).
// The first nfull blocks are 64 wide (rb = 128, sw128_chunk), the tail block is rbt bytes wide.  Built once per
// (thread, row, layer); chunk() is then a handful of integer ops.
struct SfRowMap {
    uint32_t half, row;               // byte offset of the row's half, row within the half
    uint32_t base_t, row_t, xor_t;    // tail block: byte offset of the block, of the row, swizzle mask
    uint32_t lo_t;                    // hi -> lo tile distance in the tail block (full blocks: 8 KiB)
    int full8;                        // nfull * 8: first 16-byte chunk index of the tail block
    __device__ __forceinline__ SfRowMap(int r, int nfull, int rbt, uint32_t half_bytes)
    {
        half = (uint32_t)(r >> 6) * half_bytes;
        row = (uint32_t)r & 63u;
        const int sh = rbt == 128 ? 0 : (rbt == 64 ? 1 : 2);
        base_t = half + (uint32_t)nfull * (2u * 64u * 128u);
        row_t = row * (uint32_t)rbt;
        xor_t = (uint32_t)((r >> sh) & ((rbt >> 4) - 1));
        lo_t = 64u * (uint32_t)rbt;
        full8 = nfull * 8;
    }
    // byte offset of the 16-byte chunk holding columns [8*c16g, 8*c16g+8); *lo_off = distance to the lo tile
    __device__ __forceinline__ uint32_t chunk(int c16g, uint32_t *lo_off) const
    {
        if (c16g < full8) {
            *lo_off = 64u * 128u;
            return half + (uint32_t)(c16g >> 3) * (2u * 64u * 128u) + sw128_chunk(row, (uint32_t)c16g & 7u);
        }
        *lo_off = lo_t;
        return base_t + row_t + (((uint32_t)(c16g - full8) ^ xor_t) << 4);
    }
};

// ---- shape policies -------------------------------------------------------------------------------------------------
// The kernel body is written once against a policy C that answers every shape question (layer count, padded K / N of a
// layer, block layout, blob offsets, neighbours per group).  SfDyn reads the answers from the parameter block at run
// time (any stack the planner accepts); SfStat<...> answers at COMPILE time for the stacks of the shipped 3DSSD
// configuration, so that after unrolling the layer loop every address computation, chunk bound and pooling width is a
// literal (integer / branch / uniform-register bookkeeping of exactly these questions is otherwise a large share of the
// kernel's issued instructions) and every accumulator fragment index is resolved at compile time.
__host__ __device__ constexpr int sf_r16(int x) { return (x + 15) / 16 * 16; }
// Operand layout of a layer with padded K = kp: nfull 64-wide k-blocks of 128-byte rows + a tail block whose rows are
// 32 / 64 / 128 bytes for a remainder of 16 / 32 / 48 columns (must match params._k_blocks)
__host__ __device__ constexpr int sf_nfull(int kp) { return kp / 64; }
__host__ __device__ constexpr int sf_rbt(int kp) { return kp % 64 == 0 ? 0 : (kp % 64 <= 16 ? 32 : (kp % 64 <= 32 ? 64 : 128)); }
// operand buffer: { hi | lo } tiles of 128 rows per block (a multiple of 8 KiB, so each row half is 1 KiB aligned)
__host__ __device__ constexpr uint32_t sf_abuf_bytes(int kp) { return (uint32_t)(sf_nfull(kp) * 2 * 128 * 128 + 2 * 128 * sf_rbt(kp)); }
// one half (hi or lo) of a layer's weight image
__host__ __device__ constexpr uint32_t sf_wimg_bytes(int kp, int npad) { return (uint32_t)(npad * (sf_nfull(kp) * 128 + sf_rbt(kp))); }

struct SfDyn {
    static constexpr bool kStatic = false;
    const SfParams &p;
    __device__ __forceinline__ explicit SfDyn(const SfParams &p_) : p(p_) {}
    __device__ __forceinline__ int nl() const { return p.nl; }
    __device__ __forceinline__ int ns() const { return p.ns; }
    __device__ __forceinline__ int c() const { return p.c; }
    __device__ __forceinline__ bool hoist() const { return p.hoist != 0; }
    __device__ __forceinline__ int lgu() const { return p.unit_lg; }
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
};

// Hoisted stacks of two convs (the shipped configuration): operand width K0 = n1 of the hoisted first conv, then
// K0 -> N0 -> N1, NS neighbours per group, unit lists (if any) of 1 << LGU rows per unit.
template <int K0, int N0, int N1, int NS, int LGU = 3>
struct SfStat {
    static constexpr bool kStatic = true;
    __device__ __forceinline__ explicit SfStat(const SfParams &) {}
    static constexpr int KP0 = sf_r16(K0), NP0 = sf_r16(N0), NP1 = sf_r16(N1);
    __device__ __forceinline__ constexpr int nl() const { return 2; }
    __device__ __forceinline__ constexpr int ns() const { return NS; }
    __device__ __forceinline__ constexpr int c() const { return K0; }
    __device__ __forceinline__ constexpr bool hoist() const { return true; }
    __device__ __forceinline__ constexpr int lgu() const { return LGU; }
    __device__ __forceinline__ constexpr int kp(int l) const { return l == 0 ? KP0 : NP0; }
    __device__ __forceinline__ constexpr int npad(int l) const { return l == 0 ? NP0 : NP1; }
    __device__ __forceinline__ constexpr int nout(int l) const { return l == 0 ? N0 : N1; }
    __device__ __forceinline__ constexpr int nfull(int l) const { return sf_nfull(kp(l)); }
    __device__ __forceinline__ constexpr int rbt(int l) const { return sf_rbt(kp(l)); }
    __device__ __forceinline__ constexpr uint32_t w_half(int l) const { return sf_wimg_bytes(kp(l), npad(l)); }
    __device__ __forceinline__ constexpr uint32_t w_off(int l) const { return l == 0 ? 0u : 2u * w_half(0); }
    __device__ __forceinline__ constexpr int sspad(int l) const { return (npad(l) + 31) / 32 * 32; }
    __device__ __forceinline__ constexpr uint32_t ss_off(int l) const { return l == 0 ? 0u : 2u * (uint32_t)sspad(0); }
    __device__ __forceinline__ constexpr uint32_t w_total() const { return 2u * w_half(0) + 2u * w_half(1); }
    __device__ __forceinline__ constexpr uint32_t ss_total() const { return 2u * (uint32_t)sspad(0) + 2u * (uint32_t)sspad(1); }
    __device__ __forceinline__ constexpr uint32_t abuf_bytes() const { return sf_abuf_bytes(KP0) > sf_abuf_bytes(NP0) ? sf_abuf_bytes(KP0) : sf_abuf_bytes(NP0); }
};

#ifdef SF_PROFILE
__device__ long long sf_prof[16];
#define SF_T(i) do { if (prof_on) { const long long t_ = clock64(); sf_prof[i] += t_ - t_prev; t_prev = t_; } } while (0)
#else
#define SF_T(i) do { } while (0)
#endif

// Calls f(std::integral_constant<int, W>()) for the width w of a column chunk: 64, or the 16 / 32 / 48 remainder of a layer
// (the wgmma width is part of the instruction)
template <class F>
__device__ __forceinline__ void sf_with_width(int w, F &&f)
{
    if (w == 64) f(std::integral_constant<int, 64>());
    else if (w == 48) f(std::integral_constant<int, 48>());
    else if (w == 32) f(std::integral_constant<int, 32>());
    else f(std::integral_constant<int, 16>());
}

// The MMAs of one column chunk: rows of the row half at abase (64 rows), output columns n0 .. n0+W-1, over the whole K of
// layer l (full 64-wide blocks + the tail block), issued by one warpgroup as a single wgmma chain into d and committed;
// the caller waits.  Thread t of warp w holds rows 16w + t/4 (d[4j], d[4j+1]) and +8 (d[4j+2], d[4j+3]) of columns
// n0 + 8j + 2(t%4) + {0, 1} (wgmma.cuh).
template <int W, class C>
__device__ __forceinline__ void sf_mma_chain(const C &cfg, int l, uint32_t abase, uint32_t wbase, int n0, float (&d)[W / 2])
{
    const int nfull = cfg.nfull(l), rbt = cfg.rbt(l);
    const uint32_t npad = (uint32_t)cfg.npad(l), whalf = cfg.w_half(l);
    uint32_t accumulate = 0u;
    // descriptors advance by (bytes >> 4) in their address field; shared memory < 256 KiB: no carry out of it
    wg_fence();
#pragma unroll (C::kStatic ? 4 : 1)
    for (int kb = 0; kb < nfull; kb++) {
        const uint64_t a_hi = wg_desc(abase + (uint32_t)kb * (2u * 64u * 128u), 128);
        const uint64_t b_hi = wg_desc(wbase + (uint32_t)kb * (npad * 128u) + (uint32_t)n0 * 128u, 128);
        const uint64_t a_lo = a_hi + ((64u * 128u) >> 4), b_lo = b_hi + (whalf >> 4);
#pragma unroll
        for (int kin = 0; kin < 4; kin++) {
            wg_mma3<W>(d, a_hi + 2 * kin, a_lo + 2 * kin, b_hi + 2 * kin, b_lo + 2 * kin, accumulate);
            accumulate = 1u;
        }
    }
    if (rbt) {
        const uint64_t a_hi = wg_desc(abase + (uint32_t)nfull * (2u * 64u * 128u), rbt);
        const uint64_t b_hi = wg_desc(wbase + (uint32_t)nfull * (npad * 128u) + (uint32_t)n0 * (uint32_t)rbt, rbt);
        const uint64_t a_lo = a_hi + ((64u * (uint32_t)rbt) >> 4), b_lo = b_hi + (whalf >> 4);
        const int nt = rbt == 128 ? 3 : (rbt >> 5);              // 16-wide k-steps of the tail block
#pragma unroll (C::kStatic ? 3 : 1)
        for (int kin = 0; kin < nt; kin++) {
            wg_mma3<W>(d, a_hi + 2 * kin, a_lo + 2 * kin, b_hi + 2 * kin, b_lo + 2 * kin, accumulate);
            accumulate = 1u;
        }
    }
    wg_commit();
}

// Calls f(std::integral_constant<int, c>()) for c = 0 .. n-1 (n <= SF_MAX_NCH): the chunk index is a literal before any
// loop unrolling, so the accumulator arrays it selects stay in registers
template <int C0 = 0, class F>
__device__ __forceinline__ void sf_for_chunks(int n, F &&f)
{
    if constexpr (C0 < SF_MAX_NCH) {
        if (C0 < n) {
            f(std::integral_constant<int, C0>());
            sf_for_chunks<C0 + 1>(n, f);
        }
    }
}

// Width of column chunk c of a layer with npad columns
__device__ __forceinline__ int sf_chunk_w(int npad, int c) { return npad - 64 * c < 64 ? npad - 64 * c : 64; }

// SLOTS tiles in flight per CTA, WG warpgroups (128 threads) working on each: WG == 1 runs the two row halves of its tile
// in turn, WG == 2 gives each warpgroup one row half for the whole tile (gather, every layer, pool).  C: shape policy.
template <class C, int SLOTS, int WG>
__global__ void __launch_bounds__(SF_THREADS * SLOTS * WG, SLOTS * WG == 1 ? 6 : 1)
sa_fused_kernel(const SfParams p)
{
    static_assert(WG == 1 || WG == 2, "sa_fused: one warpgroup per slot or one per row half");
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
    float *xs_all = wxs + 3 * cfg.kp(0);                 // [SLOTS][SF_XS_FLOATS] pooled-value exchange

    __shared__ unsigned long long w_bar;

    constexpr int NT = SF_THREADS * SLOTS * WG, ST = SF_THREADS * WG;     // threads per CTA / per slot
    constexpr int U = WG == 1 ? 4 : 3;                   // gather chunks in flight per thread
    const int tid = threadIdx.x, lane = tid & 31, q = (tid >> 5) & 3, t = tid & 127;
    const int slot = tid / ST, wg = (tid >> 7) % WG;
    // gather: WG == 1: thread t builds row t; WG == 2: warpgroup wg builds row half wg, two threads per row (`phase`)
    const int r = WG == 1 ? t : 64 * wg + (t & 63);
    const int phase = WG == 1 ? 0 : t >> 6;
    const int cq = 2 * (lane & 3);                       // this thread's column pair inside each 8 columns of a fragment
    // warp-uniform copies (shfl) so that descriptors are computed on the uniform datapath
    const int slot_u = __shfl_sync(0xffffffffu, slot, 0), wg_u = __shfl_sync(0xffffffffu, wg, 0);
    const int slot_bar = 1 + slot, wg_bar = 1 + SLOTS + slot * WG + wg;
    uint8_t *buf = smem + (size_t)slot * cfg.abuf_bytes();   // the slot's operand buffer (every layer, in place)
    float *xs = xs_all + (size_t)slot * SF_XS_FLOATS;
    const uint32_t half_bytes = cfg.abuf_bytes() / 2;
    const uint32_t abuf_u = smem_u32(smem) + (uint32_t)slot_u * cfg.abuf_bytes();
    const int kp0 = cfg.kp(0);

    if (tid == 0) {
        mbar_init(smem_u32(&w_bar), 1);
        fence_mbar_init_cluster();
        mbar_arrive_expect_tx(smem_u32(&w_bar), cfg.w_total());
        bulk_g2s(smem_u32(wsm), p.w_blob, cfg.w_total(), smem_u32(&w_bar));
    }
    for (uint32_t i = tid; i < cfg.ss_total(); i += NT) ss[i] = __ldg(p.ss_blob + i);
    if (cfg.hoist())
        for (int i = tid; i < 3 * kp0; i += NT) {
            const int a3 = i / kp0, k = i - a3 * kp0;
            wxs[i] = k < cfg.c() ? __ldg(p.wx + a3 * cfg.c() + k) : 0.0f;
        }
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
    // (a compile-time twin of 4-row units is launched with a unit list only: its dense schedule is never compiled)
    const bool compact = (C::kStatic && cfg.lgu() == 2) || units != nullptr;
    const int nunits = compact ? __ldg(units) : 0;
    const int lgu = cfg.lgu(), upt = 128 >> lgu;        // rows per unit (log2), units per tile
    const int tiles = compact ? (nunits + upt - 1) / upt : p.tiles;
    // neighbour index (and, in unit-list mode, unit descriptor) of this thread's row, fetched one tile ahead
    // (rows < 2^31: checked by the launcher)
    auto fetch = [&](int tl, int &desc, int &a) {
        desc = -1; a = 0;
        if (tl >= tiles) return;
        if (compact) {
            const int ui = tl * upt + (r >> lgu);
            if (ui < nunits) {
                desc = __ldg(units + 1 + ui);
                a = __ldg(p.idx + unit_slot((uint32_t)desc, (uint32_t)cfg.ns(), (uint32_t)lgu, (uint32_t)r & ((1u << lgu) - 1u)));
            }
        } else if ((long)tl * 128 + r < p.rows) {
            desc = 0;
            a = __ldg(p.idx + (size_t)tl * 128u + r);
        }
    };
    int d_next, a_next;
    fetch(tile0, d_next, a_next);
    for (int tile = tile0; tile < tiles; tile += tstep) {
        // ---- gather + centre-subtract + concat + split -> buf (layers_util.py:157-165)
        {
            const uint32_t row = (uint32_t)tile * 128u + (uint32_t)r;
            const bool ok = d_next >= 0;
            const uint32_t qi = !ok ? 0u : (compact ? unit_group((uint32_t)d_next) : row / (uint32_t)cfg.ns());    // == scene*m + query
            const uint32_t scene = qi / (uint32_t)p.m;
            const int a = a_next;
            fetch(tile + tstep, d_next, a_next);
            const float *src_f = p.points + ((size_t)scene * p.n + a) * src_pitch;
            const float *src_x = p.xyz + ((size_t)scene * p.n + a) * 3;
            const float *ctr = p.new_xyz + (size_t)qi * 3;
            const int nchunk = kp0 >> 3;
            const SfRowMap map0(r, cfg.nfull(0), cfg.rbt(0), half_bytes);
            float dx = 0.0f, dy = 0.0f, dz = 0.0f;
            if (cfg.hoist() && ok) {
                dx = __ldg(src_x) - __ldg(ctr); dy = __ldg(src_x + 1) - __ldg(ctr + 1); dz = __ldg(src_x + 2) - __ldg(ctr + 2);
            }
#pragma unroll (C::kStatic ? 4 : 1)
            for (int cg0 = phase * U; cg0 < nchunk; cg0 += WG * U) {  // U chunks of 8 columns in flight per thread
                float f[U][8];
#pragma unroll
                for (int u = 0; u < U; u++) load_concat8(f[u], src_f, src_x, ctr, cfg.c(), k0, (cg0 + u) * 8, vec, ok);
#pragma unroll
                for (int u = 0; u < U; u++) {
                    if (cg0 + u >= nchunk) break;
                    if (cfg.hoist()) hoisted_row8(f[u], wxs + (cg0 + u) * 8, kp0, dx, dy, dz);   // padded columns and rows stay 0
                    uint4 h, l;
                    uint32_t lo_off;
                    split8(f[u], 0, h, l);
                    const uint32_t off = map0.chunk(cg0 + u, &lo_off);
                    *reinterpret_cast<uint4 *>(buf + off) = h;
                    *reinterpret_cast<uint4 *>(buf + off + lo_off) = l;
                }
            }
        }
        SF_T(0);                                                       // gather
#pragma unroll (C::kStatic ? SF_MAX_LAYERS : 1)
        for (int l = 0; l < cfg.nl(); l++) {
            // the half's operand was written with ordinary stores by this warpgroup -> visible to the tensor-core (async) proxy
            fence_async_smem();
            named_bar_sync(wg_bar, 128);
            const uint32_t wbase = smem_u32(wsm) + cfg.w_off(l);
            const int npad = cfg.npad(l), nch = (npad + 63) / 64;
            const float *sc = ss + cfg.ss_off(l);
            const float *sh = sc + cfg.sspad(l);                       // scale/shift are zero-padded to 32-column chunks
            if (l < cfg.nl() - 1) {
                // ---- a hidden layer: every chunk of the half into registers, then scale/shift/ReLU/split IN PLACE
#pragma unroll
                for (int hi = 0; hi < 2 / WG; hi++) {
                    const int hf = WG == 1 ? hi : wg_u;
                    const uint32_t abase = abuf_u + (uint32_t)hf * half_bytes;
                    float d[SF_MAX_NCH][32];
                    sf_for_chunks(nch, [&](auto cc) {
                        constexpr int c = decltype(cc)::value;
                        sf_with_width(sf_chunk_w(npad, c), [&](auto wc) {
                            constexpr int W = decltype(wc)::value;
                            sf_mma_chain<W>(cfg, l, abase, wbase, 64 * c, *reinterpret_cast<float(*)[W / 2]>(&d[c][0]));
                        });
                    });
                    wg_wait<0>();                                      // the half's operand is free from here on
                    const int r0 = 64 * hf + 16 * q + (lane >> 2);
                    const SfRowMap m0(r0, cfg.nfull(l + 1), cfg.rbt(l + 1), half_bytes);
                    const SfRowMap m1(r0 + 8, cfg.nfull(l + 1), cfg.rbt(l + 1), half_bytes);
                    sf_for_chunks(nch, [&](auto cc) {
                        constexpr int c = decltype(cc)::value;
                        sf_with_width(sf_chunk_w(npad, c), [&](auto wc) {
                            constexpr int W = decltype(wc)::value;
#pragma unroll
                            for (int j = 0; j < W / 8; j++) {
                                const int col = 64 * c + 8 * j + cq;
                                const float2 s2 = *reinterpret_cast<const float2 *>(sc + col);
                                const float2 h2 = *reinterpret_cast<const float2 *>(sh + col);
                                // every conv has a ReLU; a column pair is 4 bytes of one 16-byte chunk of the next operand
                                uint32_t hw, lw, lo_off;
                                split_pair(fmaxf(fmaf(d[c][4 * j], s2.x, h2.x), 0.0f), fmaxf(fmaf(d[c][4 * j + 1], s2.y, h2.y), 0.0f), hw, lw);
                                uint32_t off = m0.chunk(8 * c + j, &lo_off) + 2u * (uint32_t)cq;
                                *reinterpret_cast<uint32_t *>(buf + off) = hw;
                                *reinterpret_cast<uint32_t *>(buf + off + lo_off) = lw;
                                split_pair(fmaxf(fmaf(d[c][4 * j + 2], s2.x, h2.x), 0.0f), fmaxf(fmaf(d[c][4 * j + 3], s2.y, h2.y), 0.0f), hw, lw);
                                off = m1.chunk(8 * c + j, &lo_off) + 2u * (uint32_t)cq;
                                *reinterpret_cast<uint32_t *>(buf + off) = hw;
                                *reinterpret_cast<uint32_t *>(buf + off + lo_off) = lw;
                            }
                        });
                    });
                }
            } else {
                // ---- the last layer: one chunk at a time (nothing is written in place), max-pooled on the fragment.
                // pool_first (scale >= 0): fma(x, s, t) is then monotone non-decreasing in x, so max_i relu(fma(x_i, s, t))
                // == relu(fma(max_i x_i, s, t)) exactly -- the affine + ReLU runs on the pooled values only.
                const bool pool_first = p.pool_first != 0;
                const int ns = cfg.ns(), nout = cfg.nout(l);
                auto finish = [&](float mx, int col) { return pool_first ? fmaxf(fmaf(mx, sc[col], sh[col]), 0.0f) : mx; };
#pragma unroll (C::kStatic ? SF_MAX_NCH : 1)
                for (int c = 0; c < nch; c++)
                    sf_with_width(sf_chunk_w(npad, c), [&](auto wc) {
                        constexpr int W = decltype(wc)::value;
#pragma unroll
                        for (int hi = 0; hi < 2 / WG; hi++) {
                            const int hf = WG == 1 ? hi : wg_u;
                            float d[W / 2];
                            sf_mma_chain<W>(cfg, l, abuf_u + (uint32_t)hf * half_bytes, wbase, 64 * c, d);
                            wg_wait<0>();
                            if (!pool_first) {
#pragma unroll
                                for (int j = 0; j < W / 8; j++) {
                                    const float2 s2 = *reinterpret_cast<const float2 *>(sc + 64 * c + 8 * j + cq);
                                    const float2 h2 = *reinterpret_cast<const float2 *>(sh + 64 * c + 8 * j + cq);
                                    d[4 * j] = fmaxf(fmaf(d[4 * j], s2.x, h2.x), 0.0f);
                                    d[4 * j + 1] = fmaxf(fmaf(d[4 * j + 1], s2.y, h2.y), 0.0f);
                                    d[4 * j + 2] = fmaxf(fmaf(d[4 * j + 2], s2.x, h2.x), 0.0f);
                                    d[4 * j + 3] = fmaxf(fmaf(d[4 * j + 3], s2.y, h2.y), 0.0f);
                                }
                            }
                            if (compact && lgu == 2) {
                                // 4-row maxima: lane owns slots s = i + (W/8)((lane/4) % 4) of d, column 8(s/4) + cq + (s%2)
                                // of rows 4(lane/16) .. +3 of the 8-row slab (s/2)%2 of its warp's 16 rows: one listed unit,
                                // combined into its group by atomicMax
                                quad_rowmax4_transpose<W / 2>(d, lane);
#pragma unroll
                                for (int i = 0; i < W / 8; i++) {
                                    const int s = i + (W / 8) * ((lane >> 2) & 3);
                                    const int ui = tile * 32 + 16 * hf + 4 * q + 2 * ((s >> 1) & 1) + (lane >> 4);
                                    const int col = 64 * c + 8 * (s >> 2) + cq + (s & 1);
                                    if (ui < nunits && col < nout)
                                        atomic_max_nonneg(p.out_f32 + (size_t)unit_group((uint32_t)__ldg(units + 1 + ui)) * p.ld_f32 + col,
                                                          finish(d[i], col));
                                }
                                continue;                              // (the row half's last step)
                            }
                            // 8-row maxima: lane owns slots s = i + (W/16)(lane/4) of d, column 8(s/4) + cq + (s%2) of the
                            // 8-row slab (s/2)%2 of its warp's 16 rows
                            quad_rowmax_transpose<W / 2>(d, lane);
#pragma unroll
                            for (int i = 0; i < W / 16; i++) {
                                const int s = i + (W / 16) * (lane >> 2);
                                const int slab = 8 * hf + 2 * q + ((s >> 1) & 1);      // 8-row slab of the tile
                                const int cl = 8 * (s >> 2) + cq + (s & 1), col = 64 * c + cl;
                                if (compact) {                         // a slab is one listed unit: atomicMax into its group
                                    const int ui = tile * 16 + slab;
                                    if (ui < nunits && col < nout)
                                        atomic_max_nonneg(p.out_f32 + (size_t)unit_group((uint32_t)__ldg(units + 1 + ui)) * p.ld_f32 + col,
                                                          finish(d[i], col));
                                } else if (ns == 8) {
                                    const long gg = (long)tile * 16 + slab;
                                    if (gg * 8 < p.rows && col < nout)
                                        store_pooled_value(finish(d[i], col), p.cnt && p.cnt[gg] == 0, (size_t)gg, col, p.out_f32,
                                                           p.ld_f32, p.out_hi, p.out_lo, p.ld_split);
                                } else {
                                    xs[slab * 64 + cl] = d[i];
                                }
                            }
                        }
                        if (!compact && ns > 8) {
                            // groups of 16-128 rows: the slabs of a group meet in xs.  A team is the threads whose slabs
                            // they are: the slot's warpgroup (WG == 1), the half's warpgroup, or both halves (128 rows, WG == 2)
                            const bool both = WG == 2 && ns == 128;
                            const int bar = both ? slot_bar : wg_bar, nthr = both ? ST : 128, tt = both ? tid % ST : t;
                            const int slab0 = WG == 2 && !both ? 8 * wg : 0, per = ns / 8;
                            const int outs = ((WG == 1 || both ? 16 : 8) / per) * W;
                            named_bar_sync(bar, nthr);
                            for (int o = tt; o < outs; o += nthr) {
                                const int gl = o / W, cl = o - gl * W, col = 64 * c + cl;
                                const float *x = xs + (slab0 + gl * per) * 64 + cl;
                                float mx = x[0];
                                for (int k = 1; k < per; k++) mx = fmaxf(mx, x[k * 64]);
                                const long gg = (long)tile * (128 / ns) + slab0 * 8 / ns + gl;
                                if (gg * ns < p.rows && col < nout)
                                    store_pooled_value(finish(mx, col), p.cnt && p.cnt[gg] == 0, (size_t)gg, col, p.out_f32,
                                                       p.ld_f32, p.out_hi, p.out_lo, p.ld_split);
                            }
                            named_bar_sync(bar, nthr);                         // xs reusable by the next chunk
                        }
                    });
            }
            SF_T(1 + l);                                               // layer l
        }
    }
}

}  // namespace ssd3d

using namespace ssd3d;

struct SfPlan { size_t abuf, w, ssf; };
static bool sf_plan(int k_in, int nl, const int *nout, SfPlan *pl)      // k_in: columns of the first operand
{
    if (nl < 1 || nl > SF_MAX_LAYERS) return false;
    pl->abuf = 0; pl->w = 0; pl->ssf = 0;
    int kp = (k_in + 15) / 16 * 16;
    pl->ssf = 3 * (size_t)kp;                               // room for the hoisted mode's Wx table
    for (int l = 0; l < nl; l++) {
        const int npad = (nout[l] + 15) / 16 * 16;
        if (npad > 64 * SF_MAX_NCH) return false;
        const size_t a = sf_abuf_bytes(kp);
        if (a > pl->abuf) pl->abuf = a;
        pl->w += 2 * sf_wimg_bytes(kp, npad);
        pl->ssf += (size_t)2 * ((npad + 31) / 32 * 32);
        kp = npad;
    }
    return true;
}
// per slot: the operand buffer and the pooled-value exchange; per CTA: weights, scale/shift, Wx table, alignment slack
static size_t sf_total(const SfPlan &pl, int slots) { return slots * (pl.abuf + SF_XS_FLOATS * sizeof(float)) + pl.w + pl.ssf * sizeof(float) + 1024; }
constexpr size_t SF_SMEM_MAX = 226 * 1024;
constexpr size_t SF_SMALL = 72 * 1024;                     // <= this: single-slot, single-warpgroup CTAs, several per SM
// Slots of larger stacks: two slots of two warpgroups (512 threads) leave 128 registers per thread, which hold a hidden
// layer's accumulators (up to 48 per thread in the shipped stacks) and the fragment epilogue without spills; a third slot
// would cut that to 80.
constexpr int SF_MAX_SLOTS = 2;

// Developer build only (-DSSD3D_DEV_HOOKS, csrc/ssd3d_dev.h): override the slot / warpgroup shape from a probe script.
// The shipped library has no such state.
#ifdef SSD3D_DEV_HOOKS
static int g_sf_slots = 0, g_sf_wg = 0, g_sf_dynamic = 0;
extern "C" void ssd3d_dev_set_fused(int slots, int wg) { g_sf_slots = slots; g_sf_wg = wg; }
extern "C" void ssd3d_dev_set_fused_dynamic(int on) { g_sf_dynamic = on; }   // force the run-time-shape kernel (A/B timing)
#else
constexpr int g_sf_slots = 0, g_sf_wg = 0, g_sf_dynamic = 0;
#endif

// Slots per CTA for a stack: 1 for small stacks (several CTAs per SM), else as many as fit one SM (<= SF_MAX_SLOTS).
static int sf_slots(const SfPlan &pl)
{
    if (sf_total(pl, 1) <= SF_SMALL) return 1;
    int s = g_sf_slots > 0 && g_sf_slots < SF_MAX_SLOTS ? g_sf_slots : SF_MAX_SLOTS;
    while (s > 1 && sf_total(pl, s) > SF_SMEM_MAX) s--;
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
// [64 -> 96 -> 128] x64, each for 8-row units (and the dense schedule) and for lists of 4-row units.  Returns false when
// (shape, slots, warpgroups) has no twin: the caller takes the dynamic kernel.
template <int LGU>
static bool sf_launch_static_lg(const SfParams &p, int slots, int wg, size_t smem, int per_sm, cudaStream_t st, cudaError_t *e)
{
    const int k0 = p.c, n0 = p.nout[0], n1 = p.nout[1], ns = p.ns;
    if (slots == 1 && wg == 1) {
        if (k0 == 16 && n0 == 16 && n1 == 32 && ns == 32) { *e = sf_launch<SfStat<16, 16, 32, 32, LGU>, 1, 1>(p, smem, per_sm, st); return true; }
        if (k0 == 32 && n0 == 32 && n1 == 64 && ns == 64) { *e = sf_launch<SfStat<32, 32, 64, 64, LGU>, 1, 1>(p, smem, per_sm, st); return true; }
    }
    if (slots == 2 && wg == 2) {
        if (k0 == 64 && n0 == 64 && n1 == 128 && ns == 32) { *e = sf_launch<SfStat<64, 64, 128, 32, LGU>, 2, 2>(p, smem, per_sm, st); return true; }
        if (k0 == 64 && n0 == 96 && n1 == 128 && ns == 64) { *e = sf_launch<SfStat<64, 96, 128, 64, LGU>, 2, 2>(p, smem, per_sm, st); return true; }
    }
    return false;
}
static bool sf_launch_static(const SfParams &p, int slots, int wg, size_t smem, int per_sm, cudaStream_t st, cudaError_t *e)
{
    if (!p.hoist || p.nl != 2) return false;
    return p.units && p.unit_lg == 2 ? sf_launch_static_lg<2>(p, slots, wg, smem, per_sm, st, e)
                                     : sf_launch_static_lg<3>(p, slots, wg, smem, per_sm, st, e);
}

// w_blob: per layer { hi image | lo image }, each image = k-blocks of [npad x (64 | tail)] bf16 in the canonical
// K-major swizzled layout (built by params.FusedStack); ss_blob: per layer { scale[sspad] | shift[sspad] }.
// wx != NULL selects the hoisted mode: `points` is the per-point table z (pitch ldz), c its width.
static int sa_mlp_fused_impl(int b, int n, int c, int m, int nsample, const float *xyz, const float *points, int ldz,
                             const float *wx, const float *new_xyz, const int *idx, const int *pts_cnt, const int *units, int nl,
                             const int *nout, const void *w_blob, const float *ss_blob, int last_scale_nonneg,
                             float *out_f32, int ld_f32, void *out_hi, void *out_lo, int ld_split, ssd3d_stream_t stream,
                             int unit_rows)
{
    const bool hoist = wx != nullptr;
    SSD3D_REQUIRE(b >= 0 && n > 0 && m >= 0 && c >= 0, "sa_mlp_fused: bad shape");
    SSD3D_REQUIRE(nsample == 8 || nsample == 16 || nsample == 32 || nsample == 64 || nsample == 128,
                  "sa_mlp_fused: nsample=%d must be one of 8, 16, 32, 64, 128", nsample);
    SSD3D_REQUIRE(xyz && new_xyz && idx && w_blob && ss_blob && (points || c == 0), "sa_mlp_fused: null pointer");
    SSD3D_REQUIRE(!hoist || (c > 0 && ldz >= c), "sa_mlp_fused_hoisted: bad table shape n1=%d ldz=%d", c, ldz);
    SSD3D_REQUIRE(out_f32 || (out_hi && out_lo), "sa_mlp_fused: no output requested");
    SSD3D_REQUIRE(!units || (out_f32 && !out_hi && !out_lo), "sa_mlp_fused: a unit list combines through atomicMax on the (zero-filled) fp32 output only");
    SSD3D_REQUIRE(!units || unit_rows == 8 || (unit_rows == 4 && nsample <= 64),
                  "sa_mlp_fused: unit_rows=%d must be 8, or 4 with nsample <= 64 (nsample=%d)", unit_rows, nsample);
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
    p.unit_lg = units && unit_rows == 4 ? 2 : 3;
    p.hoist = hoist ? 1 : 0; p.ldz = ldz; p.wx = wx;
    p.pool_first = last_scale_nonneg ? 1 : 0;
    p.nl = nl;
    int kprev = (k_in + 15) / 16 * 16;
    uint32_t woff = 0, ssoff = 0;
    for (int l = 0; l < nl; l++) {
        p.kp[l] = kprev;
        p.nout[l] = nout[l];
        p.npad[l] = (nout[l] + 15) / 16 * 16;
        p.nfull[l] = sf_nfull(p.kp[l]);
        p.rbt[l] = sf_rbt(p.kp[l]);
        p.w_off[l] = woff;
        p.w_half[l] = sf_wimg_bytes(p.kp[l], p.npad[l]);
        woff += 2 * p.w_half[l];
        p.ss_off[l] = ssoff;
        p.sspad[l] = (p.npad[l] + 31) / 32 * 32;
        ssoff += 2 * p.sspad[l];
        kprev = p.npad[l];
    }
    p.w_total = woff; p.ss_total = ssoff;
    p.w_blob = (const uint8_t *)w_blob; p.ss_blob = ss_blob;
    p.abuf_bytes = (uint32_t)pl.abuf;
    p.out_f32 = out_f32; p.ld_f32 = ld_f32;
    p.out_hi = (__nv_bfloat16 *)out_hi; p.out_lo = (__nv_bfloat16 *)out_lo; p.ld_split = ld_split;

    // one warpgroup per slot for small stacks (several CTAs per SM), else one per row half
    const bool small = slots == 1 && smem <= SF_SMALL;
    const int wg = slots == 1 && g_sf_wg > 0 ? (g_sf_wg == 1 ? 1 : 2) : (small ? 1 : 2);
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
        e = slots == 2 ? sf_launch<SfDyn, 2, 2>(p, smem, per_sm, st)
          : wg == 1 ? sf_launch<SfDyn, 1, 1>(p, smem, per_sm, st) : sf_launch<SfDyn, 1, 2>(p, smem, per_sm, st);
    if (e != cudaSuccess) return cuda_status(e, "sa_mlp_fused attr");
#ifdef SF_PROFILE
    {
        long long h[16];
        cudaDeviceSynchronize();
        cudaMemcpyFromSymbol(h, sf_prof, sizeof(h));
        fprintf(stderr, "sf_prof slots=%d tiles=%d:", slots, p.tiles);
        for (int i = 0; i < 1 + SF_MAX_LAYERS; i++) fprintf(stderr, " %lld", h[i]);
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
                             last_scale_nonneg, out_f32, ld_f32, out_hi, out_lo, ld_split, stream, 8);
}

extern "C" int ssd3d_sa_mlp_fused_ex(int b, int n, int c, int m, int nsample, const float *xyz, const float *points,
                                     const float *new_xyz, const int *idx, const int *pts_cnt, const int *units, int nl,
                                     const int *nout, const void *w_blob, const float *ss_blob, int last_scale_nonneg,
                                     float *out_f32, int ld_f32, void *out_hi, void *out_lo, int ld_split, ssd3d_stream_t stream,
                                     int unit_rows)
{
    return sa_mlp_fused_impl(b, n, c, m, nsample, xyz, points, c, nullptr, new_xyz, idx, pts_cnt, units, nl, nout, w_blob, ss_blob,
                             last_scale_nonneg, out_f32, ld_f32, out_hi, out_lo, ld_split, stream, unit_rows);
}

// The fused SA scale with its first conv hoisted (see ssd3d_linear_tc_hoisted): z[b,n,ldz] per-point table (this scale's
// n1 columns start at z), wx = Wx*s1 as [3][n1]; the stack (w_blob / ss_blob / nout) starts at the scale's SECOND conv.
extern "C" int ssd3d_sa_mlp_fused_hoisted(int b, int n, int n1, int m, int nsample, const float *xyz, const float *z, int ldz,
                                          const float *wx, const float *new_xyz, const int *idx, const int *pts_cnt,
                                          const int *units, int nl, const int *nout, const void *w_blob, const float *ss_blob,
                                          int last_scale_nonneg, float *out_f32, int ld_f32, void *out_hi, void *out_lo,
                                          int ld_split, ssd3d_stream_t stream)
{
    return ssd3d_sa_mlp_fused_hoisted_ex(b, n, n1, m, nsample, xyz, z, ldz, wx, new_xyz, idx, pts_cnt, units, nl, nout, w_blob,
                                         ss_blob, last_scale_nonneg, out_f32, ld_f32, out_hi, out_lo, ld_split, stream, 8);
}

extern "C" int ssd3d_sa_mlp_fused_hoisted_ex(int b, int n, int n1, int m, int nsample, const float *xyz, const float *z, int ldz,
                                             const float *wx, const float *new_xyz, const int *idx, const int *pts_cnt,
                                             const int *units, int nl, const int *nout, const void *w_blob, const float *ss_blob,
                                             int last_scale_nonneg, float *out_f32, int ld_f32, void *out_hi, void *out_lo,
                                             int ld_split, ssd3d_stream_t stream, int unit_rows)
{
    SSD3D_REQUIRE(z && wx, "sa_mlp_fused_hoisted: null table pointer");
    return sa_mlp_fused_impl(b, n, n1, m, nsample, xyz, z, ldz, wx, new_xyz, idx, pts_cnt, units, nl, nout, w_blob, ss_blob,
                             last_scale_nonneg, out_f32, ld_f32, out_hi, out_lo, ld_split, stream, unit_rows);
}
