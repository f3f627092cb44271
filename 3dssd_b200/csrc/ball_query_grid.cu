// ball_query_grid.cu -- the radius search of ball_query.cu with spatial culling, for large candidate sets.
//
// Same operator, same bits (query_ball_point_gpu / query_ball_point_dilated_gpu,
// /root/reference/lib/utils/tf_ops/grouping/tf_grouping_g.cu:215-255, :308-357): per query the FIRST nsample hits in
// ascending candidate index, first hit back-filled, pts_cnt = min(hits, nsample).  The brute-force kernel tests every
// query against all n candidates (5.4e8 tests for 3DSSD layer 1); network inputs arrive in random order (the loader
// shuffles, lib/dataset/dataloader/kitti_dataloader.py:143-147), so candidate-index tiles have no spatial locality to
// cull by.  Instead:
//   1. bq_grid_build_kernel (one CTA per scene): bounding box -> a 2-D uniform grid over the two widest axes with cell
//      size >= 1.01 * r_max (<= 8192 cells), counting sort of the points by cell into (x, y, z, index) records.
//      A candidate within r_max of a query lies in the 3x3 cell neighbourhood of the query's cell; in the row-major
//      cell order these are three CONTIGUOUS ranges of the sorted array.
//   2. ball_query_grid_kernel: a warp takes one query at a time, streams the three ranges (32 candidates per step,
//      coalesced 16-byte records), evaluates the reference's distance recipe, and marks every hit in a per-shell BITMAP
//      over candidate indices in shared memory (n <= 16384 bits).  Scanning the bitmap in word order then yields the hits
//      in ascending index, whatever order the cells delivered them in -- first-K semantics without any sort.
//      A query whose neighbourhood holds more than n/8 candidates takes the index-order scan with early exit instead: a
//      dense ball is full after a few hundred candidates, where culling would still visit (and mark) thousands.
// Non-finite coordinates keep the reference's behaviour (NaN distances hit in the plain query, never in the dilated one):
// a scene containing any collapses to a single cell, i.e. the exhaustive scan.
#include <math.h>

#include "common.cuh"

namespace ssd3d {

constexpr int BQG_MAX_N = 16384;              // bitmap width (bits) the query kernel keeps per shell
constexpr int BQG_WORDS = BQG_MAX_N / 32;
constexpr int BQG_MAX_CELLS = 8192;
constexpr int BQG_BUILD_T = 1024;
constexpr int BQG_THREADS = 256;
constexpr int BQG_WARPS = BQG_THREADS / 32;
constexpr int BQG_QPW = 4;                    // queries per warp (sequential)
constexpr int BQG_MAX_SHELLS = 4;

// per-scene header at the start of the scene's workspace slice
struct BqgHeader {
    float min_a, min_b, inv_c;
    int na, nb, axis_a, axis_b, pad;
};
static_assert(sizeof(BqgHeader) == 32, "header is two 16-byte pieces");
struct BqgCounters { int *ptr[BQG_MAX_SHELLS]; };   // unit-list counters the build kernel resets (see BqgParams::units)

__host__ __device__ inline size_t bqg_scene_bytes(int n)
{
    // header | cell_start[BQG_MAX_CELLS + 1] (padded to 16 bytes) | records[n] float4
    return sizeof(BqgHeader) + ((size_t)(BQG_MAX_CELLS + 1) * 4 + 15) / 16 * 16 + (size_t)n * 16;
}

__device__ __forceinline__ int bqg_cell_coord(float v, float mn, float inv_c, int nc)
{
    const float u = (v - mn) * inv_c;
    int i = (int)floorf(u);                    // NaN -> 0 after the clamps below (only reached in 1-cell grids)
    i = i < 0 ? 0 : i;
    return i > nc - 1 ? nc - 1 : i;
}

__global__ void __launch_bounds__(BQG_BUILD_T, 1)
bq_grid_build_kernel(int n, float r_max, const float *__restrict__ xyz, uint8_t *__restrict__ ws, const BqgCounters zero)
{
    if (blockIdx.x == 0 && threadIdx.x < BQG_MAX_SHELLS && zero.ptr[threadIdx.x] != nullptr) *zero.ptr[threadIdx.x] = 0;
    __shared__ int counts[BQG_MAX_CELLS + 1];
    __shared__ float red[6][32];
    __shared__ int s_bad, s_scan[32];
    __shared__ BqgHeader hdr;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int scene = blockIdx.x;
    const float *pts = xyz + (size_t)scene * n * 3;
    uint8_t *base = ws + (size_t)scene * bqg_scene_bytes(n);
    int *cell_start = reinterpret_cast<int *>(base + sizeof(BqgHeader));
    float4 *rec = reinterpret_cast<float4 *>(base + sizeof(BqgHeader) + ((size_t)(BQG_MAX_CELLS + 1) * 4 + 15) / 16 * 16);

    // ---- bounding box (finite points) + non-finite flag
    float mn[3] = {INFINITY, INFINITY, INFINITY}, mx[3] = {-INFINITY, -INFINITY, -INFINITY};
    int bad = 0;
    for (int k = tid; k < n; k += BQG_BUILD_T) {
#pragma unroll
        for (int a = 0; a < 3; a++) {
            const float v = pts[3 * k + a];
            if (!(fabsf(v) <= 3.0e38f)) bad = 1;            // NaN or +-Inf
            mn[a] = fminf(mn[a], v); mx[a] = fmaxf(mx[a], v);
        }
    }
    if (tid == 0) s_bad = 0;
    __syncthreads();
#pragma unroll
    for (int a = 0; a < 3; a++) {
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            mn[a] = fminf(mn[a], __shfl_xor_sync(0xffffffffu, mn[a], o));
            mx[a] = fmaxf(mx[a], __shfl_xor_sync(0xffffffffu, mx[a], o));
        }
        if (lane == 0) { red[a][warp] = mn[a]; red[3 + a][warp] = mx[a]; }
    }
    if (bad) atomicOr(&s_bad, 1);
    __syncthreads();
    if (tid == 0) {
        float lo[3], ext[3];
        for (int a = 0; a < 3; a++) {
            float l = INFINITY, h = -INFINITY;
            for (int w = 0; w < BQG_BUILD_T / 32; w++) { l = fminf(l, red[a][w]); h = fmaxf(h, red[3 + a][w]); }
            lo[a] = l; ext[a] = h - l;
        }
        // the two widest axes span the grid
        int a0 = 0, a1 = 1, a2 = 2;
        if (ext[a1] > ext[a0]) { int t = a0; a0 = a1; a1 = t; }
        if (ext[a2] > ext[a0]) { int t = a0; a0 = a2; a2 = t; }
        if (ext[a2] > ext[a1]) { int t = a1; a1 = a2; a2 = t; }
        BqgHeader h;
        h.axis_a = a0; h.axis_b = a1; h.pad = 0;
        const bool one_cell = s_bad || !(ext[a0] >= 0.0f) || !(ext[a0] <= 1.0e30f) || !(r_max > 0.0f) || !(r_max <= 1.0e30f);
        if (one_cell) {
            h.min_a = 0.0f; h.min_b = 0.0f; h.inv_c = 0.0f; h.na = 1; h.nb = 1;
        } else {
            float c = r_max * 1.01f;                         // margin: cell arithmetic rounds (u up to 8192), the 3x3 stencil must still cover r_max
            for (;;) {
                const float fa = floorf(ext[a0] / c) + 1.0f, fb = floorf(ext[a1] / c) + 1.0f;
                if (fa * fb <= (float)BQG_MAX_CELLS) { h.na = (int)fa; h.nb = (int)fb; break; }
                c *= 1.25f;
            }
            h.min_a = lo[a0]; h.min_b = lo[a1]; h.inv_c = 1.0f / c;
        }
        hdr = h;
        *reinterpret_cast<BqgHeader *>(base) = h;
    }
    for (int i = tid; i <= BQG_MAX_CELLS; i += BQG_BUILD_T) counts[i] = 0;
    __syncthreads();
    const BqgHeader h = hdr;
    const int ncell = h.na * h.nb;

    // ---- histogram
    for (int k = tid; k < n; k += BQG_BUILD_T) {
        const int ia = bqg_cell_coord(pts[3 * k + h.axis_a], h.min_a, h.inv_c, h.na);
        const int ib = bqg_cell_coord(pts[3 * k + h.axis_b], h.min_b, h.inv_c, h.nb);
        atomicAdd(&counts[ib * h.na + ia], 1);
    }
    __syncthreads();
    // ---- exclusive scan over the cells (8 per thread)
    constexpr int PER = BQG_MAX_CELLS / BQG_BUILD_T;
    int v[PER], sum = 0;
#pragma unroll
    for (int i = 0; i < PER; i++) { v[i] = counts[tid * PER + i]; sum += v[i]; }
    int incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) s_scan[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        int w = s_scan[lane], wi = w;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int t = __shfl_up_sync(0xffffffffu, wi, o);
            if (lane >= o) wi += t;
        }
        s_scan[lane] = wi - w;                               // exclusive prefix of the warp totals
    }
    __syncthreads();
    int run = s_scan[warp] + incl - sum;
#pragma unroll
    for (int i = 0; i < PER; i++) { counts[tid * PER + i] = run; run += v[i]; }
    if (tid == BQG_BUILD_T - 1) counts[BQG_MAX_CELLS] = run;  // == n
    __syncthreads();
    for (int i = tid; i <= ncell; i += BQG_BUILD_T) cell_start[i] = counts[i < ncell ? i : BQG_MAX_CELLS];
    __syncthreads();
    // ---- scatter (order inside a cell is irrelevant: the query kernel restores index order through its bitmap)
    for (int k = tid; k < n; k += BQG_BUILD_T) {
        const float x = pts[3 * k], y = pts[3 * k + 1], z = pts[3 * k + 2];
        const float c3[3] = {x, y, z};
        const int ia = bqg_cell_coord(c3[h.axis_a], h.min_a, h.inv_c, h.na);
        const int ib = bqg_cell_coord(c3[h.axis_b], h.min_b, h.inv_c, h.nb);
        const int pos = atomicAdd(&counts[ib * h.na + ia], 1);
        rec[pos] = make_float4(x, y, z, __int_as_float(k));
    }
}

struct BqgParams {
    int n, m, nshell;
    int nsample[BQG_MAX_SHELLS];
    float t_lo[BQG_MAX_SHELLS], t_hi[BQG_MAX_SHELLS];
    float t_max;
    int *idx[BQG_MAX_SHELLS];
    int *cnt[BQG_MAX_SHELLS];
    // optional per-shell UNIT LISTS for the grouped MLP (include/ssd3d.h, ssd3d_query_ball_point_multi_ws_ex): units[s][0]
    // counts the units, units[s][1 + u] = (group << 4) | j names rows Wj .. Wj+W-1 of that group's neighbour list, W =
    // 1 << lgu[s] (8 or 4).  A group with cnt hits gets ceil(cnt / W) units: the slots beyond cnt repeat the first hit and
    // cannot change a max-pool.
    int *units[BQG_MAX_SHELLS];
    int lgu[BQG_MAX_SHELLS];
};

// Bitmap word wi of a shell lives at wi + (wi >> lg): one pad word per lane chunk of 2^lg words, so that the chunks of
// consecutive lanes start an ODD number of words apart and the per-lane sequential reads of the read-back are free of
// bank conflicts (unpadded, 16-word chunks collide 16 ways: that alone was ~90% of the first version's run time).
constexpr int BQG_WORDS_P = BQG_WORDS + 32;

__device__ __forceinline__ void bqg_emit_units(int *units, int group, int cnt, int lgu)
{
    if (units == nullptr || cnt <= 0) return;
    const int nu = (cnt + (1 << lgu) - 1) >> lgu;
    const int base = atomicAdd(units, nu);                 // order of the list is irrelevant: the consumer max-pools
    for (int j = 0; j < nu; j++) units[1 + base + j] = (group << 4) | j;
}

template <int NS, bool DILATED>
__global__ void __launch_bounds__(BQG_THREADS)
ball_query_grid_kernel(const float *__restrict__ xyz1, const float *__restrict__ xyz2, const uint8_t *__restrict__ ws,
                       const BqgParams p)
{
    extern __shared__ uint4 dyn_smem4[];
    uint32_t *bitmaps = reinterpret_cast<uint32_t *>(dyn_smem4);       // [BQG_WARPS][NS][BQG_WORDS_P]
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int scene = blockIdx.y;
    const int n = p.n, m = p.m;
    const uint8_t *base = ws + (size_t)scene * bqg_scene_bytes(n);
    const BqgHeader h = *reinterpret_cast<const BqgHeader *>(base);
    const int *cell_start = reinterpret_cast<const int *>(base + sizeof(BqgHeader));
    const float4 *rec = reinterpret_cast<const float4 *>(base + sizeof(BqgHeader) + ((size_t)(BQG_MAX_CELLS + 1) * 4 + 15) / 16 * 16);
    const float *cand = xyz1 + (size_t)scene * n * 3;
    uint32_t *bm = bitmaps + (size_t)warp * NS * BQG_WORDS_P;
    const int words = (n + 31) >> 5;                                   // bitmap words in use
    int lg = 1;                                                        // words per lane chunk = 2^lg >= ceil(words / 32), >= 2
    while ((32 << lg) < words) lg++;
    const int wpl = 1 << lg;
    const int words_p = 32 * (wpl + 1);                                // padded words in use (<= BQG_WORDS_P)

    for (int qq = 0; qq < BQG_QPW; qq++) {
        const int qi = (blockIdx.x * BQG_WARPS + warp) * BQG_QPW + qq;
        if (qi >= m) break;                                            // warp-uniform
        const float *qsrc = xyz2 + ((size_t)scene * m + qi) * 3;
        const float qx = qsrc[0], qy = qsrc[1], qz = qsrc[2];
        const float q3[3] = {qx, qy, qz};
        const bool qfin = fabsf(qx) <= 3.0e38f && fabsf(qy) <= 3.0e38f && fabsf(qz) <= 3.0e38f;
        const int ca = bqg_cell_coord(q3[h.axis_a], h.min_a, h.inv_c, h.na);
        const int cb = bqg_cell_coord(q3[h.axis_b], h.min_b, h.inv_c, h.nb);
        const int a_lo = ca > 0 ? ca - 1 : 0, a_hi = ca + 1 < h.na ? ca + 1 : h.na - 1;
        const int b_lo = cb > 0 ? cb - 1 : 0, b_hi = cb + 1 < h.nb ? cb + 1 : h.nb - 1;
        // population of the 3x3 cell neighbourhood (three contiguous record ranges)
        int j0r[3], j1r[3], ncand = 0;
#pragma unroll
        for (int rr = 0; rr < 3; rr++) {
            const int rb = b_lo + rr;
            j0r[rr] = rb <= b_hi ? cell_start[rb * h.na + a_lo] : 0;
            j1r[rr] = rb <= b_hi ? cell_start[rb * h.na + a_hi + 1] : 0;
            ncand += j1r[rr] - j0r[rr];
        }
        if (!qfin || ncand * 8 > n) {
            // ---- DENSE neighbourhood (or a query with a non-finite coordinate, whose NaN distances hit everywhere in the
            // plain query): culling buys nothing, and a dense ball fills its nsample slots within the first few hundred
            // candidates -- scan in index order and stop as soon as every shell is full, like the reference does.
            int cnt[NS], first[NS];
#pragma unroll
            for (int s = 0; s < NS; s++) { cnt[s] = 0; first[s] = 0; }
            for (int k0 = 0; k0 < n; k0 += 32) {
                bool all_full = true;
#pragma unroll
                for (int s = 0; s < NS; s++) all_full = all_full && cnt[s] >= p.nsample[s];
                if (all_full) break;
                const int k = k0 + lane;
                const bool in = k < n;
                const float cx = in ? __ldg(cand + 3 * k) : 0.0f, cy = in ? __ldg(cand + 3 * k + 1) : 0.0f, cz = in ? __ldg(cand + 3 * k + 2) : 0.0f;
                const float dx = qx - cx, dy = qy - cy, dz = qz - cz;
                float t = __fmul_rn(dy, dy);
                t = __fmaf_rn(dx, dx, t);
                t = __fmaf_rn(dz, dz, t);
#pragma unroll
                for (int s = 0; s < NS; s++) {
                    const bool hit = in && (DILATED ? (t == 0.0f || (t >= p.t_lo[s] && t < p.t_hi[s])) : !(t >= p.t_hi[s]));
                    const uint32_t hs = __ballot_sync(0xffffffffu, hit);
                    const int ns = p.nsample[s], c0 = cnt[s];
                    if (hs != 0u && c0 < ns) {
                        int *dst = p.idx[s] + ((size_t)scene * m + qi) * ns;
                        const int pos = c0 + __popc(hs & ((1u << lane) - 1u));
                        if (hit && pos < ns) dst[pos] = k;
                        if (c0 == 0) first[s] = k0 + __ffs(hs) - 1;
                        cnt[s] = min(ns, c0 + __popc(hs));
                    }
                }
            }
#pragma unroll
            for (int s = 0; s < NS; s++) {
                const int ns = p.nsample[s], c = cnt[s];
                int *dst = p.idx[s] + ((size_t)scene * m + qi) * ns;
                for (int l = c + lane; l < ns; l += 32) dst[l] = first[s];   // back-fill (zeros for an empty ball)
                if (lane == 0) {
                    p.cnt[s][(size_t)scene * m + qi] = c;
                    bqg_emit_units(p.units[s], scene * m + qi, c, p.lgu[s]);
                }
            }
            continue;
        }
        // ---- SPARSE neighbourhood: mark the hits of the three record ranges in the per-shell index bitmaps
        for (int w = lane; w * 4 < NS * BQG_WORDS_P; w += 32) {
            const int s = (w * 4) / BQG_WORDS_P, j = w * 4 - s * BQG_WORDS_P;
            if (j < words_p) reinterpret_cast<uint4 *>(bm)[w] = make_uint4(0u, 0u, 0u, 0u);
        }
        __syncwarp();
#pragma unroll
        for (int rr = 0; rr < 3; rr++) {
            for (int j = j0r[rr] + lane; j < j1r[rr]; j += 32) {
                const float4 c = __ldg(rec + j);
                // the reference's contracted recipe: t = dy*dy ; t = fma(dx,dx,t) ; t = fma(dz,dz,t)   (query - candidate)
                const float dx = qx - c.x, dy = qy - c.y, dz = qz - c.z;
                float t = __fmul_rn(dy, dy);
                t = __fmaf_rn(dx, dx, t);
                t = __fmaf_rn(dz, dz, t);
                const bool near = DILATED ? (t < p.t_max) : !(t >= p.t_max);
                if (near) {
                    const int k = __float_as_int(c.w);
                    const int wi = k >> 5;
#pragma unroll
                    for (int s = 0; s < NS; s++) {
                        const bool hit = DILATED ? (t == 0.0f || (t >= p.t_lo[s] && t < p.t_hi[s])) : !(t >= p.t_hi[s]);
                        if (hit) atomicOr(bm + s * BQG_WORDS_P + wi + (wi >> lg), 1u << (k & 31));
                    }
                }
            }
        }
        __syncwarp();
        // ---- read the bitmaps back in index order: lane L owns words [L*wpl, (L+1)*wpl), stored from L*(wpl+1)
#pragma unroll
        for (int s = 0; s < NS; s++) {
            const uint32_t *b = bm + s * BQG_WORDS_P + lane * (wpl + 1);
            const int ns = p.nsample[s];
            int mine = 0;
            uint32_t nz = 0u;                                              // which of this lane's words hold hits
            for (int w = 0; w < wpl; w++) {
                const uint32_t bits = b[w];                                // words beyond `words` were cleared and never set
                mine += __popc(bits);
                nz |= (bits != 0u ? 1u : 0u) << w;
            }
            int incl = mine;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int t = __shfl_up_sync(0xffffffffu, incl, o);
                if (lane >= o) incl += t;
            }
            const int total = __shfl_sync(0xffffffffu, incl, 31);
            const int c = total < ns ? total : ns;
            int pos = incl - mine;                                         // hits before this lane's words
            int *dst = p.idx[s] + ((size_t)scene * m + qi) * ns;
            int first = 0x7fffffff;                                        // lowest set bit of the whole bitmap (back-fill)
            // only the lanes that hold hits walk, and only over their non-empty words (the first version walked all 16
            // words of a lane: 70% of the kernel's instructions)
            while (nz != 0u && pos < ns) {
                const int w = __ffs(nz) - 1;
                nz &= nz - 1u;
                uint32_t bits = b[w];
                while (bits != 0u && pos < ns) {
                    const int bit = __ffs(bits) - 1;
                    bits &= bits - 1u;
                    const int k = (lane * wpl + w) * 32 + bit;
                    if (pos == 0) first = k;
                    dst[pos++] = k;
                }
            }
            first = __reduce_min_sync(0xffffffffu, first);
            if (c > 0) for (int l = c + lane; l < ns; l += 32) dst[l] = first;      // tf_grouping_g.cu:245-248 back-fill
            else for (int l = lane; l < ns; l += 32) dst[l] = 0;                     // empty ball: the caller's idx * (cnt > 0)
            if (lane == 0) {
                p.cnt[s][(size_t)scene * m + qi] = c;
                bqg_emit_units(p.units[s], scene * m + qi, c, p.lgu[s]);
            }
        }
        __syncwarp();
    }
}

float bq_sq_threshold(float r);   // ball_query.cu

// Unit lists from finished neighbour counts (the exhaustive kernel's route: small candidate sets): one CTA per shell scans
// the groups in order -- a group with cnt hits owns ceil(cnt / W) units of W = 1 << lgu rows -- so this list is in group order.
constexpr int GU_THREADS = 1024;
struct GuParams { const int *cnt[BQG_MAX_SHELLS]; int *units[BQG_MAX_SHELLS]; int nsample[BQG_MAX_SHELLS]; int lgu[BQG_MAX_SHELLS]; };

__global__ void __launch_bounds__(GU_THREADS)
group_units_kernel(int groups, const GuParams p)
{
    const int s = blockIdx.x;
    int *units = p.units[s];
    if (units == nullptr) return;
    const int *cnt = p.cnt[s];
    const int ns = p.nsample[s], lgu = p.lgu[s], w1 = (1 << lgu) - 1;
    __shared__ int warp_tot[GU_THREADS / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int per = (groups + GU_THREADS - 1) / GU_THREADS;
    const int g0 = min(groups, tid * per), g1 = min(groups, g0 + per);
    int mine = 0;
    for (int g = g0; g < g1; g++) mine += (min(__ldg(cnt + g), ns) + w1) >> lgu;
    int incl = mine;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const int o = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += o;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        int t = warp_tot[lane];
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const int o = __shfl_up_sync(0xffffffffu, t, d);
            if (lane >= d) t += o;
        }
        warp_tot[lane] = t;                                   // inclusive totals of the warps
    }
    __syncthreads();
    int pos = incl - mine + (warp > 0 ? warp_tot[warp - 1] : 0);
    if (tid == GU_THREADS - 1) units[0] = pos + mine;
    for (int g = g0; g < g1; g++) {
        const int nu = (min(__ldg(cnt + g), ns) + w1) >> lgu;
        for (int j = 0; j < nu; j++) units[1 + pos + j] = (g << 4) | j;
        pos += nu;
    }
}

template <int NS>
static cudaError_t launch_bqg(bool dilated, dim3 grid, size_t smem, cudaStream_t st, const float *xyz1, const float *xyz2,
                              const uint8_t *ws, const BqgParams &p)
{
    cudaError_t e;
    if (dilated) {
        e = cudaFuncSetAttribute((const void *)ball_query_grid_kernel<NS, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e == cudaSuccess) ball_query_grid_kernel<NS, true><<<grid, BQG_THREADS, smem, st>>>(xyz1, xyz2, ws, p);
    } else {
        e = cudaFuncSetAttribute((const void *)ball_query_grid_kernel<NS, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e == cudaSuccess) ball_query_grid_kernel<NS, false><<<grid, BQG_THREADS, smem, st>>>(xyz1, xyz2, ws, p);
    }
    return e;
}

}  // namespace ssd3d

using namespace ssd3d;

extern "C" size_t ssd3d_query_ball_point_workspace(int b, int n)
{
    if (b <= 0 || n <= 0 || n > BQG_MAX_N) return 0;      // 0: this size takes the exhaustive kernel
    return (size_t)b * bqg_scene_bytes(n);
}

extern "C" int ssd3d_query_ball_point_multi_ws(int b, int n, int m, int nqueries, int dilated, const float *min_radius,
                                               const float *max_radius, const int *nsample, const float *xyz1,
                                               const float *xyz2, int *const *idx, int *const *pts_cnt, int *const *units,
                                               void *workspace, size_t workspace_bytes, ssd3d_stream_t stream)
{
    return ssd3d_query_ball_point_multi_ws_ex(b, n, m, nqueries, dilated, min_radius, max_radius, nsample, xyz1, xyz2, idx, pts_cnt,
                                              units, workspace, workspace_bytes, stream, nullptr);
}

// rows per unit of shell s's list: 8 (no unit_rows array) or unit_rows[s], 8 or 4; a list names at most 16 units per group
static int bq_unit_lg(const int *unit_rows, int s) { return unit_rows == nullptr || unit_rows[s] == 8 ? 3 : 2; }
static int bq_check_units(int *const *units, const int *unit_rows, const int *nsample, int nqueries, int b, int m)
{
    if (!units) return 0;
    SSD3D_REQUIRE(nqueries >= 1 && nqueries <= BQG_MAX_SHELLS, "query_ball_point: unit lists for 1..%d radius shells per call, got %d", BQG_MAX_SHELLS, nqueries);
    for (int s = 0; s < nqueries; s++) {
        if (!units[s]) continue;
        const int w = unit_rows ? unit_rows[s] : 8;
        SSD3D_REQUIRE(w == 8 || w == 4, "query_ball_point: unit_rows[%d]=%d must be 8 or 4", s, w);
        SSD3D_REQUIRE(nsample[s] <= 16 * w, "query_ball_point: unit lists of %d-row units cover nsample <= %d, got %d", w, 16 * w, nsample[s]);
        SSD3D_REQUIRE((long)b * m < (1L << 27), "query_ball_point: too many groups for a unit list");
    }
    return 0;
}

extern "C" int ssd3d_query_ball_point_multi_ws_ex(int b, int n, int m, int nqueries, int dilated, const float *min_radius,
                                                  const float *max_radius, const int *nsample, const float *xyz1,
                                                  const float *xyz2, int *const *idx, int *const *pts_cnt, int *const *units,
                                                  void *workspace, size_t workspace_bytes, ssd3d_stream_t stream,
                                                  const int *unit_rows)
{
    if (int rc = bq_check_units(units, unit_rows, nsample, nqueries, b, m)) return rc;
    if (workspace == nullptr || workspace_bytes == 0) {
        const int rc = ssd3d_query_ball_point_multi(b, n, m, nqueries, dilated, min_radius, max_radius, nsample, xyz1, xyz2, idx,
                                                    pts_cnt, stream);
        if (rc || units == nullptr || b == 0 || m == 0) return rc;
        GuParams gp = {};
        for (int s = 0; s < nqueries; s++) {
            gp.cnt[s] = pts_cnt[s]; gp.units[s] = units[s]; gp.nsample[s] = nsample[s]; gp.lgu[s] = bq_unit_lg(unit_rows, s);
        }
        group_units_kernel<<<nqueries, GU_THREADS, 0, (cudaStream_t)stream>>>(b * m, gp);
        SSD3D_LAUNCH_CHECK("group_units_kernel");
    }
    SSD3D_REQUIRE(b >= 0 && n > 0 && m >= 0, "query_ball_point: bad shape b=%d n=%d m=%d", b, n, m);
    SSD3D_REQUIRE(n <= BQG_MAX_N, "query_ball_point (grid): n=%d exceeds %d; pass no workspace", n, BQG_MAX_N);
    SSD3D_REQUIRE(nqueries >= 1 && nqueries <= BQG_MAX_SHELLS, "query_ball_point: 1..%d radius shells per call, got %d", BQG_MAX_SHELLS, nqueries);
    SSD3D_REQUIRE(workspace_bytes >= (size_t)b * bqg_scene_bytes(n), "query_ball_point: workspace of %zu bytes, need %zu (ssd3d_query_ball_point_workspace)",
                  workspace_bytes, (size_t)b * bqg_scene_bytes(n));
    SSD3D_REQUIRE((reinterpret_cast<uintptr_t>(workspace) & 15u) == 0, "query_ball_point: workspace must be 16-byte aligned");
    SSD3D_REQUIRE(xyz1 && xyz2, "query_ball_point: null pointer");
    BqgParams p = {};
    p.n = n; p.m = m; p.nshell = nqueries;
    float tmax = 0.0f, rmax = 0.0f;
    for (int s = 0; s < nqueries; s++) {
        SSD3D_REQUIRE(max_radius[s] > 0.0f, "query_ball_point expects positive radius");     // tf_grouping.cpp:275-279 / :368-374
        SSD3D_REQUIRE(nsample[s] > 0, "query_ball_point expects positive nsample");
        SSD3D_REQUIRE(idx[s] && pts_cnt[s], "query_ball_point: null output pointer");
        p.nsample[s] = nsample[s];
        p.t_hi[s] = bq_sq_threshold(max_radius[s]);
        p.t_lo[s] = dilated ? bq_sq_threshold(min_radius[s]) : 0.0f;
        if (!dilated && !(max_radius[s] > 1e-20f)) p.t_hi[s] = -1.0f;
        tmax = fmaxf(tmax, p.t_hi[s]);
        rmax = fmaxf(rmax, max_radius[s]);
        p.idx[s] = idx[s];
        p.cnt[s] = pts_cnt[s];
        p.units[s] = units ? units[s] : nullptr;
        p.lgu[s] = bq_unit_lg(unit_rows, s);
    }
    p.t_max = tmax;
    if (b == 0 || m == 0) return 0;
    cudaStream_t st = (cudaStream_t)stream;
    BqgCounters zero = {};
    for (int s = 0; s < nqueries; s++) zero.ptr[s] = p.units[s];
    bq_grid_build_kernel<<<b, BQG_BUILD_T, 0, st>>>(n, rmax, xyz1, (uint8_t *)workspace, zero);
    int rc = cuda_status(cudaGetLastError(), "bq_grid_build_kernel");
    if (rc) return rc;
    const size_t smem = (size_t)BQG_WARPS * nqueries * BQG_WORDS_P * 4;
    dim3 grid((unsigned)ceil_div(m, BQG_WARPS * BQG_QPW), (unsigned)b);
    cudaError_t e;
    switch (nqueries) {
        case 1: e = launch_bqg<1>(dilated != 0, grid, smem, st, xyz1, xyz2, (const uint8_t *)workspace, p); break;
        case 2: e = launch_bqg<2>(dilated != 0, grid, smem, st, xyz1, xyz2, (const uint8_t *)workspace, p); break;
        case 3: e = launch_bqg<3>(dilated != 0, grid, smem, st, xyz1, xyz2, (const uint8_t *)workspace, p); break;
        default: e = launch_bqg<4>(dilated != 0, grid, smem, st, xyz1, xyz2, (const uint8_t *)workspace, p); break;
    }
    if (e != cudaSuccess) return cuda_status(e, "ball_query_grid_kernel shared-memory opt-in");
    SSD3D_LAUNCH_CHECK("ball_query_grid_kernel");
}
