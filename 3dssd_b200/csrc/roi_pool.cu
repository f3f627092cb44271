// roi_pool.cu -- PointRCNN's region pool (the 'RegionPool' of POINTS_POOLER, lib/builder/points_pooler.py:40-61,
// :119-170), the bridge between the RPN's proposals and the stage-2 network (DESIGN.md section 3.16):
//   * query_boxes_3d_points   tf_grouping_g.cu:27-94: the first nsample points (in index order) inside each bottom-centred
//                             box (x, y_bottom, z, l, h, w, ry), the list padded with the first hit, plus the hit count.
//   * region_pool             one launch from (xyz, RPN features, per-point RPN score, proposal block, count) to the
//                             stage-2 input: expand each proposal by the context range, collect its points as above,
//                             gather xyz / features, build the info channels [canonical xyz | mask | dist], run the
//                             5 -> c_info roi_pool/conv0 (folded BN, ReLU) on the CUDA cores and write
//                             xyz [b*p, nsample, 3] (canonical) and features [b*p, nsample, c_info + c_feat].
//
// The membership test is point_inside_box_3d with the reference build's arithmetic, read off its SASS (nvcc -O2,
// default -fmad=true): the max_distance is sqrtf of the double fma(l/2, l/2, (w/2)^2) rounded to float, the rotated
// coordinates are fma(dx, cos, -(dz * sin)) and fma(dz, cos, dx * sin) in float with cosf / sinf of ry, and the face
// tests compare in double against +-l/2.0 and +-w/2.0.  Written with _rn intrinsics so that no compiler contracts it
// differently.  Both kernels use the one device function, so the fused pool collects exactly the reference's points.
//
// Scan: one warp per proposal walks the points 32 at a time; a ballot + popc compaction keeps index order and the walk
// stops after nsample hits.  The fused kernel first stages its scene's xyz in shared memory (192 KiB at n = 16384) and
// then runs one warp per proposal of a group of RP_WARPS.
#include "common.cuh"

namespace ssd3d {

constexpr int RP_WARPS = 8;
constexpr int RP_THREADS = RP_WARPS * 32;
constexpr int RP_MAX_NSAMPLE = 1024;
constexpr int RP_MAX_INFO = 256;           // roi_pool/conv0 output channels
constexpr int RP_INFO_IN = 5;              // [canonical xyz | mask | dist]
constexpr size_t RP_SMEM_MAX = 227 * 1024;

struct RoiBox {
    float cx, by, cz, h, cos_ry, sin_ry, max_distance;
    double half_l, half_w;
};

// point_inside_box_3d's per-box constants (tf_grouping_g.cu:27-40, :65-72)
__device__ __forceinline__ RoiBox roi_box(float cx, float by, float cz, float l, float h, float w, float ry)
{
    RoiBox b;
    b.cx = cx; b.by = by; b.cz = cz; b.h = h;
    b.half_l = __dmul_rn((double)l, 0.5);
    b.half_w = __dmul_rn((double)w, 0.5);
    b.max_distance = fmaxf(sqrtf((float)__fma_rn(b.half_l, b.half_l, __dmul_rn(b.half_w, b.half_w))), 1e-20f);
    b.cos_ry = cosf(ry);
    b.sin_ry = sinf(ry);
    return b;
}

__device__ __forceinline__ bool roi_inside(float x, float y, float z, const RoiBox &b)
{
    const float dx = __fsub_rn(x, b.cx), dz = __fsub_rn(z, b.cz);
    if (fabsf(dx) > b.max_distance || y > b.by || __fsub_rn(b.by, y) > b.h || fabsf(dz) > b.max_distance) return false;
    const double u = (double)__fmaf_rn(dx, b.cos_ry, -__fmul_rn(dz, b.sin_ry));
    const double v = (double)__fmaf_rn(dz, b.cos_ry, __fmul_rn(dx, b.sin_ry));
    return u >= -b.half_l && u <= b.half_l && v >= -b.half_w && v <= b.half_w;
}

// One warp: the first ns points of xyz[0..n) inside b, in index order, into idx[0..ns); the rest of idx is the first
// hit (0 when there is none).  Returns the hit count (<= ns).  idx may be shared or global memory.
__device__ __forceinline__ int roi_scan_warp(const float *xyz, int n, const RoiBox &b, int ns, int *idx, int lane)
{
    int cnt = 0;
    for (int base = 0; base < n && cnt < ns; base += 32) {
        const int k = base + lane;
        const bool in = k < n && roi_inside(xyz[3 * k], xyz[3 * k + 1], xyz[3 * k + 2], b);
        const uint32_t bal = __ballot_sync(0xffffffffu, in);
        const int pos = cnt + __popc(bal & ((1u << lane) - 1u));
        if (in && pos < ns) idx[pos] = k;
        cnt += __popc(bal);
    }
    cnt = min(cnt, ns);
    __syncwarp();
    const int first = cnt > 0 ? idx[0] : 0;
    for (int q = cnt + lane; q < ns; q += 32) idx[q] = first;
    __syncwarp();
    return cnt;
}

__global__ void __launch_bounds__(RP_THREADS)
query_boxes_3d_points_kernel(int b, int n, int m, int ns, const float *__restrict__ xyz, const float *__restrict__ boxes,
                             int *__restrict__ idx, int *__restrict__ cnt)
{
    const int row = (int)((blockIdx.x * (long)RP_THREADS + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (row >= b * m) return;                  // whole warps leave together
    const float *p = boxes + (size_t)row * 7;
    const RoiBox bx = roi_box(p[0], p[1], p[2], p[3], p[4], p[5], p[6]);
    const int c = roi_scan_warp(xyz + (size_t)(row / m) * n * 3, n, bx, ns, idx + (size_t)row * ns, lane);
    if (lane == 0) cnt[row] = c;
}

struct RegionPoolArgs {
    int n, p, ns, cf, co, ldbox;
    float context, mask_thresh;
    const float *xyz, *feat, *score, *boxes;
    const int *count;
    const float *w, *scale, *shift;
    int *idx, *cnt;
    float *oxyz, *ofeat;
};

// grid (ceil(p / RP_WARPS), b); shared: xyz [n*3] | conv0 weights [5*co] | scale [co] | shift [co] | idx [RP_WARPS][ns]
__global__ void __launch_bounds__(RP_THREADS)
region_pool_kernel(const RegionPoolArgs a)
{
    extern __shared__ __align__(16) float rp_smem[];
    float *sx = rp_smem;
    float *sw = sx + (size_t)a.n * 3;
    float *ssc = sw + RP_INFO_IN * a.co, *ssh = ssc + a.co;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, s = blockIdx.y;
    int *sidx = reinterpret_cast<int *>(ssh + a.co) + warp * a.ns;

    const float *gx = a.xyz + (size_t)s * a.n * 3;
    for (int e = tid; e < a.n * 3; e += RP_THREADS) sx[e] = gx[e];
    for (int e = tid; e < RP_INFO_IN * a.co; e += RP_THREADS) sw[e] = a.w[e];
    for (int e = tid; e < a.co; e += RP_THREADS) { ssc[e] = a.scale[e]; ssh[e] = a.shift[e]; }
    __syncthreads();

    const int r = blockIdx.x * RP_WARPS + warp;
    if (r >= a.p) return;                      // no block-wide barrier follows
    const size_t row = (size_t)s * a.p + r;
    const float *pb = a.boxes + row * a.ldbox;
    const float cx = pb[0], by = pb[1], cz = pb[2], ry = pb[6];
    const bool valid = a.count == nullptr || r < a.count[s];
    int c = 0;
    if (valid) {                               // expand_proposals_context: l, h, w + context, the bottom centre kept
        const RoiBox bx = roi_box(cx, by, cz, __fadd_rn(pb[3], a.context), __fadd_rn(pb[4], a.context),
                                  __fadd_rn(pb[5], a.context), ry);
        c = roi_scan_warp(sx, a.n, bx, a.ns, sidx, lane);
    } else {
        for (int q = lane; q < a.ns; q += 32) sidx[q] = 0;
        __syncwarp();
    }
    for (int q = lane; q < a.ns; q += 32) a.idx[row * a.ns + q] = sidx[q];
    if (lane == 0) a.cnt[row] = c;

    // canonical_xyz (points_pooler.py:157-170): rotate_points(xyz - box[:3], -ry), R = [[c,0,s],[0,1,0],[-s,0,c]]
    const float cr = cosf(-ry), sr = sinf(-ry);
    float *ox = a.oxyz + row * a.ns * 3;
    for (int q = lane; q < a.ns; q += 32) {
        const int k = sidx[q];
        const float nx = __fsub_rn(sx[3 * k], cx), ny = __fsub_rn(sx[3 * k + 1], by), nz = __fsub_rn(sx[3 * k + 2], cz);
        ox[3 * q] = __fadd_rn(__fmul_rn(cr, nx), __fmul_rn(sr, nz));
        ox[3 * q + 1] = ny;
        ox[3 * q + 2] = __fadd_rn(__fmul_rn(-sr, nx), __fmul_rn(cr, nz));
    }
    // [conv0([canonical xyz | mask | dist]) | features] per pooled point, one float4 of each part per lane
    const int cw = a.co + a.cf;
    const float *gf = a.feat + (size_t)s * a.n * a.cf;
    const float *gs = a.score + (size_t)s * a.n;
#pragma unroll 2
    for (int q = 0; q < a.ns; q++) {
        const int k = sidx[q];
        const float x = sx[3 * k], y = sx[3 * k + 1], z = sx[3 * k + 2];
        const float nx = __fsub_rn(x, cx), ny = __fsub_rn(y, by), nz = __fsub_rn(z, cz);
        float in[RP_INFO_IN];
        in[0] = __fadd_rn(__fmul_rn(cr, nx), __fmul_rn(sr, nz));
        in[1] = ny;
        in[2] = __fadd_rn(__fmul_rn(-sr, nx), __fmul_rn(cr, nz));
        in[3] = gs[k] >= a.mask_thresh ? 1.0f : 0.0f;                                  // POOLER_MASK_THRESHOLD
        in[4] = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(y, y)), __fmul_rn(z, z)));   // ||raw xyz||
        float *o = a.ofeat + (row * a.ns + q) * cw;
        for (int c4 = lane; c4 < a.co / 4; c4 += 32) {
            float v[4];
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const int oc = 4 * c4 + j;
                float acc = 0.0f;
#pragma unroll
                for (int t = 0; t < RP_INFO_IN; t++) acc = __fmaf_rn(in[t], sw[t * a.co + oc], acc);
                v[j] = fmaxf(__fmaf_rn(acc, ssc[oc], ssh[oc]), 0.0f);
            }
            reinterpret_cast<float4 *>(o)[c4] = make_float4(v[0], v[1], v[2], v[3]);
        }
        const float4 *fk = reinterpret_cast<const float4 *>(gf + (size_t)k * a.cf);
        for (int c4 = lane; c4 < a.cf / 4; c4 += 32) reinterpret_cast<float4 *>(o + a.co)[c4] = __ldg(fk + c4);
    }
}

static size_t region_pool_smem(int n, int ns, int co)
{
    return ((size_t)n * 3 + (size_t)(RP_INFO_IN + 2) * co) * 4 + (size_t)RP_WARPS * ns * 4;
}

}  // namespace ssd3d

using namespace ssd3d;

extern "C" int ssd3d_query_boxes_3d_points(int b, int n, int m, int nsample, const float *xyz, const float *proposals,
                                           int *idx, int *pts_cnt, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && n >= 0 && m >= 0 && nsample > 0, "query_boxes_3d_points: bad shape b=%d n=%d m=%d nsample=%d",
                  b, n, m, nsample);
    if (b == 0 || m == 0) return 0;
    SSD3D_REQUIRE((xyz || n == 0) && proposals && idx && pts_cnt, "query_boxes_3d_points: null pointer");
    const long warps = (long)b * m;
    query_boxes_3d_points_kernel<<<ceil_div(warps * 32, RP_THREADS), RP_THREADS, 0, (cudaStream_t)stream>>>(
        b, n, m, nsample, xyz, proposals, idx, pts_cnt);
    SSD3D_LAUNCH_CHECK("query_boxes_3d_points_kernel");
}

extern "C" size_t ssd3d_region_pool_smem(int n, int nsample, int c_info)
{
    if (n < 0 || nsample <= 0 || c_info <= 0) return 0;
    return region_pool_smem(n, nsample, c_info);
}

extern "C" int ssd3d_region_pool(int b, int n, int p, int nsample, int c_feat, int c_info, const float *xyz,
                                 const float *features, const float *point_score, const float *proposals, int ld_proposals,
                                 const int *count, float context, float mask_thresh, const float *info_w,
                                 const float *info_scale, const float *info_shift, int *idx, int *pts_cnt, float *out_xyz,
                                 float *out_features, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && n >= 1 && p >= 0 && nsample > 0 && nsample <= RP_MAX_NSAMPLE && ld_proposals >= 7,
                  "region_pool: bad shape b=%d n=%d p=%d nsample=%d ld_proposals=%d", b, n, p, nsample, ld_proposals);
    SSD3D_REQUIRE(c_feat >= 0 && c_feat % 4 == 0 && c_info > 0 && c_info % 4 == 0 && c_info <= RP_MAX_INFO,
                  "region_pool: c_feat=%d and c_info=%d must be multiples of 4 (c_info <= %d)", c_feat, c_info, RP_MAX_INFO);
    const size_t smem = region_pool_smem(n, nsample, c_info);
    SSD3D_REQUIRE(smem <= RP_SMEM_MAX, "region_pool: n=%d points need %zu bytes of shared memory (at most %zu)", n, smem,
                  RP_SMEM_MAX);
    if (b == 0 || p == 0) return 0;
    SSD3D_REQUIRE(xyz && (features || c_feat == 0) && point_score && proposals && info_w && info_scale && info_shift && idx &&
                  pts_cnt && out_xyz && out_features, "region_pool: null pointer");
    SSD3D_REQUIRE((reinterpret_cast<uintptr_t>(features) & 15u) == 0 && (reinterpret_cast<uintptr_t>(out_features) & 15u) == 0,
                  "region_pool: features and out_features must be 16-byte aligned");
    const int e = cuda_status(cudaFuncSetAttribute(region_pool_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                              "region_pool_kernel shared memory");
    if (e) return e;
    RegionPoolArgs a;
    a.n = n; a.p = p; a.ns = nsample; a.cf = c_feat; a.co = c_info; a.ldbox = ld_proposals;
    a.context = context; a.mask_thresh = mask_thresh;
    a.xyz = xyz; a.feat = features; a.score = point_score; a.boxes = proposals; a.count = count;
    a.w = info_w; a.scale = info_scale; a.shift = info_shift;
    a.idx = idx; a.cnt = pts_cnt; a.oxyz = out_xyz; a.ofeat = out_features;
    region_pool_kernel<<<dim3(ceil_div(p, RP_WARPS), b), RP_THREADS, smem, (cudaStream_t)stream>>>(a);
    SSD3D_LAUNCH_CHECK("region_pool_kernel");
}
