// misc.cu -- the small elementwise stages of the SA path and of the detection head, one kernel each, so that a
// captured step contains no framework (at::) kernels:
//   * split_points        points[:, :, 0:3] / points[:, :, 3:]   (single_stage_detector.py:116-117)
//   * iota_idx            tf.tile(tf.range(npoint)) identity sampling (layers_util.py:91-92, :100-101)
//   * concat_cols         tf.concat([xyz, points], -1) feeding calc_square_dist (layers_util.py:94, :102)
//   * vote_translate      clamp of the vote offsets + add to the seed xyz (layers_util.py:20-23)
//   * decode_dist_anchor_free  anchor_decoder.py:86-112 + decode_class2angle :6-14 + the sigmoid of
//                         single_stage_detector.py:210-211: raw head outputs -> (x,y,z,l,h,w,ry) + score, the
//                         inputs of bev_nms.
//   * decode_bin_anchor   the same for PointRCNN's 'Bin-Anchor' regression: anchor_decoder.py:115-164 on the anchors of
//                         generate_anchors.py:33-65 (one anchor size per point) + the sigmoid.
//   * decode_bin_anchor_rows  the same decode against per-row anchors (PointRCNN's stage 2: the bottom-centred
//                         proposals, double_stage_detector.py:298-337) + the 2-way softmax score times the pool mask.
// All HBM-bound copies / a few flops per element; sized far below one wave, so launch latency is the cost.
#include "common.cuh"

namespace ssd3d {

__global__ void split_points_kernel(long rows, int c, const float *__restrict__ pts, float *__restrict__ xyz,
                                    float *__restrict__ feat)
{
    const long total = rows * c;
    const int cf = c - 3;
    for (long e = blockIdx.x * (long)blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x) {
        const long r = e / c;
        const int l = (int)(e - r * c);
        const float v = pts[e];
        if (l < 3) xyz[r * 3 + l] = v;
        else feat[r * cf + (l - 3)] = v;
    }
}

__global__ void fill_zero_kernel(float4 *__restrict__ x4, long n4, float *__restrict__ tail, int ntail)
{
    for (long e = blockIdx.x * (long)blockDim.x + threadIdx.x; e < n4; e += (long)gridDim.x * blockDim.x)
        x4[e] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (blockIdx.x == 0 && (int)threadIdx.x < ntail) tail[threadIdx.x] = 0.0f;
}

__global__ void iota_idx_kernel(int b, int m, int start, int *__restrict__ out, int ldo)
{
    const int total = b * m;
    for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < total; e += gridDim.x * blockDim.x) {
        const int s = e / m, j = e - s * m;
        out[(size_t)s * ldo + j] = start + j;
    }
}

__global__ void concat_cols_kernel(int b, int n, int ca, int cb, const float *__restrict__ a, long long sa,
                                   const float *__restrict__ bsrc, long long sb, float *__restrict__ out)
{
    const int c = ca + cb;
    const long total = (long)b * n * c;
    for (long e = blockIdx.x * (long)blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x) {
        const long row = e / c;
        const int l = (int)(e - row * c);
        const long s = row / n, k = row - s * n;
        out[e] = l < ca ? a[s * sa + k * ca + l] : bsrc[s * sb + k * cb + (l - ca)];
    }
}

__global__ void vote_translate_kernel(long rows, const float *__restrict__ xyz, const float *__restrict__ off, int ldoff,
                                      float lx, float ly, float lz, float *__restrict__ out)
{
    const long total = rows * 3;
    for (long e = blockIdx.x * (long)blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x) {
        const long r = e / 3;
        const int l = (int)(e - r * 3);
        const float lo = l == 0 ? lx : (l == 1 ? ly : lz);               // negative bound; upper bound is -lo
        const float v = fminf(fmaxf(off[r * ldoff + l], lo), -lo);       // tf.minimum(tf.maximum(off, min), -min)
        out[e] = xyz[e] + v;
    }
}

// one thread per candidate point
__global__ void decode_kernel(long rows, int nbins, int ncls, const float *__restrict__ ctr, const float *__restrict__ reg,
                              int ldreg, const float *__restrict__ cls, int ldcls, float bin_interval, float *__restrict__ boxes,
                              float *__restrict__ scores)
{
    const long r = blockIdx.x * (long)blockDim.x + threadIdx.x;
    if (r >= rows) return;
    const float *g = reg + r * ldreg;                  // [6 distances | nbins angle logits | nbins angle residuals]
    int bin = 0;
    float bv = g[6];
    for (int k = 1; k < nbins; k++) {                  // tf.argmax: first maximum
        const float v = g[6 + k];
        if (v > bv) { bv = v; bin = k; }
    }
    const float res = g[6 + nbins + bin];
    const float angle = __fmul_rn(__fadd_rn((float)bin, res), bin_interval);     // (bin + res + 0) * interval
    const float hx = g[3], hy = g[4], hz = g[5];
    float *o = boxes + r * 7;
    o[0] = __fadd_rn(ctr[r * 3 + 0], g[0]);
    o[1] = __fadd_rn(__fadd_rn(ctr[r * 3 + 1], g[1]), hy);                       // centre moved down by half the height (:103-106)
    o[2] = __fadd_rn(ctr[r * 3 + 2], g[2]);
    o[3] = fmaxf(__fmul_rn(hx, 2.0f), 0.1f);
    o[4] = fmaxf(__fmul_rn(hy, 2.0f), 0.1f);
    o[5] = fmaxf(__fmul_rn(hz, 2.0f), 0.1f);
    o[6] = angle;
    // the sigmoid in double, rounded once: in float, expf's own 2-ulp error plus the rounding of the add and the divide
    // put some scores more than 2 ulp away from the exact sigmoid
    for (int c = 0; c < ncls; c++) scores[r * ncls + c] = (float)(1.0 / (1.0 + exp(-(double)cls[r * ldcls + c])));
}

// argmax over nb logits, ties to the first index (tf.argmax)
__device__ __forceinline__ int first_argmax(const float *g, int nb)
{
    int bin = 0;
    float bv = g[0];
    for (int k = 1; k < nb; k++)
        if (g[k] > bv) { bv = g[k]; bin = k; }
    return bin;
}

// one thread per candidate point; reg row = [x_bin nb | x_res nb | z_bin nb | z_res nb | y_res | size_res 3 |
// angle_cls na | angle_res na].  TF's fp32 order, one rounding per operation:
//   x = (ax - half_range) + ((bin + res) + 0.5) * interval,  z likewise
//   y = (ay + h / 2) + y_res,  lhw = max(anchor_lhw + res, 0.1),  ry = 0 + (bin + res) * (2 pi / na)
__global__ void decode_bin_kernel(long rows, int nb, int na, const float *__restrict__ ctr, const float *__restrict__ reg,
                                  int ldreg, const float *__restrict__ cls, int ldcls, float half_range, float bin_interval,
                                  float angle_interval, float al, float ah, float aw, float *__restrict__ boxes,
                                  float *__restrict__ scores)
{
    const long r = blockIdx.x * (long)blockDim.x + threadIdx.x;
    if (r >= rows) return;
    const float *g = reg + r * ldreg;
    const float *c = ctr + r * 3;
    float *o = boxes + r * 7;
    const int xb = first_argmax(g, nb), zb = first_argmax(g + 2 * nb, nb);
    const float dx = __fmul_rn(__fadd_rn(__fadd_rn((float)xb, g[nb + xb]), 0.5f), bin_interval);
    const float dz = __fmul_rn(__fadd_rn(__fadd_rn((float)zb, g[3 * nb + zb]), 0.5f), bin_interval);
    const float *off = g + 4 * nb;
    o[0] = __fadd_rn(__fsub_rn(c[0], half_range), dx);
    o[1] = __fadd_rn(__fadd_rn(c[1], __fmul_rn(ah, 0.5f)), off[0]);
    o[2] = __fadd_rn(__fsub_rn(c[2], half_range), dz);
    o[3] = fmaxf(__fadd_rn(al, off[1]), 0.1f);
    o[4] = fmaxf(__fadd_rn(ah, off[2]), 0.1f);
    o[5] = fmaxf(__fadd_rn(aw, off[3]), 0.1f);
    const float *ang = off + 4;
    const int ab = first_argmax(ang, na);
    o[6] = __fadd_rn(0.0f, __fmul_rn(__fadd_rn(__fadd_rn((float)ab, ang[na + ab]), 0.0f), angle_interval));
    scores[r] = (float)(1.0 / (1.0 + exp(-(double)cls[r * ldcls])));    // as decode_kernel
}

// one thread per proposal; anchors[r] = (x, y_bottom, z, l, h, w, ry).  As decode_bin_kernel with the anchor's own
// centre, size and angle: x = (ax - half_range) + ((bin + res) + 0.5) * interval (camera x / z, not the anchor's axes),
// y = ay + y_res, lhw = max(anchor_lhw + res, 0.1), ry = ary + ((bin + res) + 0) * (2 pi / na).  score = softmax(cls)[1]
// in double, rounded once, times (pool_cnt > 0) (double_stage_detector.py:317-328)
__global__ void decode_bin_rows_kernel(long rows, int nb, int na, const float *__restrict__ anchors, int ldanc,
                                       const float *__restrict__ reg, int ldreg, const float *__restrict__ cls, int ldcls,
                                       const int *__restrict__ pool_cnt, float half_range, float bin_interval,
                                       float angle_interval, float *__restrict__ boxes, float *__restrict__ scores)
{
    const long r = blockIdx.x * (long)blockDim.x + threadIdx.x;
    if (r >= rows) return;
    const float *g = reg + r * ldreg;
    const float *an = anchors + r * ldanc;
    float *o = boxes + r * 7;
    const int xb = first_argmax(g, nb), zb = first_argmax(g + 2 * nb, nb);
    const float dx = __fmul_rn(__fadd_rn(__fadd_rn((float)xb, g[nb + xb]), 0.5f), bin_interval);
    const float dz = __fmul_rn(__fadd_rn(__fadd_rn((float)zb, g[3 * nb + zb]), 0.5f), bin_interval);
    const float *off = g + 4 * nb;
    o[0] = __fadd_rn(__fsub_rn(an[0], half_range), dx);
    o[1] = __fadd_rn(an[1], off[0]);
    o[2] = __fadd_rn(__fsub_rn(an[2], half_range), dz);
    o[3] = fmaxf(__fadd_rn(an[3], off[1]), 0.1f);
    o[4] = fmaxf(__fadd_rn(an[4], off[2]), 0.1f);
    o[5] = fmaxf(__fadd_rn(an[5], off[3]), 0.1f);
    const float *ang = off + 4;
    const int ab = first_argmax(ang, na);
    o[6] = __fadd_rn(an[6], __fmul_rn(__fadd_rn(__fadd_rn((float)ab, ang[na + ab]), 0.0f), angle_interval));
    const float *c = cls + r * ldcls;
    const float p1 = (float)(1.0 / (1.0 + exp((double)c[0] - (double)c[1])));
    scores[r] = pool_cnt == nullptr ? p1 : __fmul_rn(p1, pool_cnt[r] > 0 ? 1.0f : 0.0f);
}

// out[s, off_i + q, :] = src_i[s, q, :] for the (up to 8) row blocks of a scene: tf.concat(axis=1) of per-part results
struct ConcatRowsArgs {
    const float *src[8];
    int m[8];       // rows per scene of part i
    int start[8];   // first output row of part i
    int parts, mtot, c;
};
__global__ void concat_rows_kernel(int b, const ConcatRowsArgs a, float *__restrict__ out)
{
    const long total = (long)b * a.mtot * a.c;
    for (long e = blockIdx.x * (long)blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x) {
        const long row = e / a.c;
        const int l = (int)(e - row * a.c);
        const long s = row / a.mtot;
        const int q = (int)(row - s * a.mtot);
        int i = 0;
#pragma unroll
        for (int t = 1; t < 8; t++)
            if (t < a.parts && q >= a.start[t]) i = t;
        out[e] = a.src[i][((size_t)s * a.m[i] + (q - a.start[i])) * a.c + l];
    }
}

static int grid_for(long total, int threads) { return (int)((total + threads - 1) / threads < 1184 ? (total + threads - 1) / threads : 1184); }

}  // namespace ssd3d

using namespace ssd3d;

extern "C" int ssd3d_split_points(long rows, int c, const float *points, float *xyz, float *feat, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(rows >= 0 && c >= 3, "split_points: bad shape rows=%ld c=%d", rows, c);
    if (rows == 0) return 0;
    SSD3D_REQUIRE(points && xyz && (feat || c == 3), "split_points: null pointer");
    split_points_kernel<<<grid_for(rows * c, 256), 256, 0, (cudaStream_t)stream>>>(rows, c, points, xyz, feat);
    SSD3D_LAUNCH_CHECK("split_points_kernel");
}

extern "C" int ssd3d_iota_idx(int b, int m, int start, int *out, int ldo, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && m >= 0 && ldo >= m, "iota_idx: bad shape b=%d m=%d ldo=%d", b, m, ldo);
    if (b == 0 || m == 0) return 0;
    SSD3D_REQUIRE(out != nullptr, "iota_idx: null pointer");
    iota_idx_kernel<<<grid_for((long)b * m, 256), 256, 0, (cudaStream_t)stream>>>(b, m, start, out, ldo);
    SSD3D_LAUNCH_CHECK("iota_idx_kernel");
}

extern "C" int ssd3d_concat_cols(int b, int n, int ca, int cb, const float *a, long long a_stride, const float *bsrc,
                                 long long b_stride, float *out, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && n >= 0 && ca >= 0 && cb >= 0 && ca + cb > 0, "concat_cols: bad shape b=%d n=%d c=%d+%d", b, n, ca, cb);
    SSD3D_REQUIRE(a_stride >= (long long)n * ca && b_stride >= (long long)n * cb, "concat_cols: strides smaller than a scene");
    if (b == 0 || n == 0) return 0;
    SSD3D_REQUIRE((a || ca == 0) && (bsrc || cb == 0) && out, "concat_cols: null pointer");
    concat_cols_kernel<<<grid_for((long)b * n * (ca + cb), 256), 256, 0, (cudaStream_t)stream>>>(b, n, ca, cb, a, a_stride, bsrc,
                                                                                                 b_stride, out);
    SSD3D_LAUNCH_CHECK("concat_cols_kernel");
}

extern "C" int ssd3d_vote_translate(long rows, const float *xyz, const float *offsets, int ld_offsets, float min_x, float min_y,
                                    float min_z, float *out, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(rows >= 0 && ld_offsets >= 3, "vote_translate: bad shape rows=%ld ld=%d", rows, ld_offsets);
    if (rows == 0) return 0;
    SSD3D_REQUIRE(xyz && offsets && out, "vote_translate: null pointer");
    vote_translate_kernel<<<grid_for(rows * 3, 256), 256, 0, (cudaStream_t)stream>>>(rows, xyz, offsets, ld_offsets, min_x, min_y,
                                                                                     min_z, out);
    SSD3D_LAUNCH_CHECK("vote_translate_kernel");
}

static int decode_dist_anchor_free(const char *op, long rows, int angle_bins, int cls_num, const float *center_xyz,
                                   const float *pred_reg, int ld_reg, const float *pred_cls, int ld_cls, float *boxes, float *scores,
                                   ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(rows >= 0 && angle_bins >= 1 && ld_reg >= 6 + 2 * angle_bins && cls_num >= 1 && cls_num <= SSD3D_MAX_CLASSES &&
                  ld_cls >= cls_num, "%s: bad shape rows=%ld bins=%d ld_reg=%d ld_cls=%d cls_num=%d", op, rows, angle_bins, ld_reg,
                  ld_cls, cls_num);
    if (rows == 0) return 0;
    SSD3D_REQUIRE(center_xyz && pred_reg && pred_cls && boxes && scores, "%s: null pointer", op);
    const float interval = (float)(2.0 * 3.14159265358979323846 / angle_bins);
    decode_kernel<<<(int)((rows + 127) / 128), 128, 0, (cudaStream_t)stream>>>(rows, angle_bins, cls_num, center_xyz, pred_reg,
                                                                              ld_reg, pred_cls, ld_cls, interval, boxes, scores);
    SSD3D_LAUNCH_CHECK("decode_kernel");
}

extern "C" int ssd3d_decode_dist_anchor_free(long rows, int angle_bins, const float *center_xyz, const float *pred_reg,
                                             int ld_reg, const float *pred_cls, int ld_cls, float *boxes, float *scores,
                                             ssd3d_stream_t stream)
{
    return decode_dist_anchor_free("decode_dist_anchor_free", rows, angle_bins, 1, center_xyz, pred_reg, ld_reg, pred_cls, ld_cls,
                                   boxes, scores, stream);
}

extern "C" int ssd3d_decode_dist_anchor_free_classes(long rows, int angle_bins, int cls_num, const float *center_xyz,
                                                     const float *pred_reg, int ld_reg, const float *pred_cls, int ld_cls,
                                                     float *boxes, float *scores, ssd3d_stream_t stream)
{
    return decode_dist_anchor_free("decode_dist_anchor_free_classes", rows, angle_bins, cls_num, center_xyz, pred_reg, ld_reg,
                                   pred_cls, ld_cls, boxes, scores, stream);
}

extern "C" int ssd3d_decode_bin_anchor(long rows, int bin_num, float half_bin_search_range, int angle_bins,
                                       const float *center_xyz, const float *pred_reg, int ld_reg, const float *pred_cls,
                                       int ld_cls, const float *anchor_lhw, float *boxes, float *scores, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(rows >= 0 && bin_num >= 1 && angle_bins >= 1 && ld_reg >= 4 * bin_num + 4 + 2 * angle_bins && ld_cls >= 1,
                  "decode_bin_anchor: bad shape rows=%ld bins=%d angle_bins=%d ld_reg=%d ld_cls=%d", rows, bin_num, angle_bins,
                  ld_reg, ld_cls);
    SSD3D_REQUIRE(anchor_lhw != nullptr, "decode_bin_anchor: null anchor size");
    if (rows == 0) return 0;
    SSD3D_REQUIRE(center_xyz && pred_reg && pred_cls && boxes && scores, "decode_bin_anchor: null pointer");
    // the Python constants of anchor_decoder.py:137-145 / :160, rounded once to the float32 TF computes in
    const float bin_interval = (float)((double)half_bin_search_range * 2.0 / bin_num);
    const float angle_interval = (float)(2.0 * 3.14159265358979323846 / angle_bins);
    decode_bin_kernel<<<(int)((rows + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
        rows, bin_num, angle_bins, center_xyz, pred_reg, ld_reg, pred_cls, ld_cls, half_bin_search_range, bin_interval,
        angle_interval, anchor_lhw[0], anchor_lhw[1], anchor_lhw[2], boxes, scores);
    SSD3D_LAUNCH_CHECK("decode_bin_kernel");
}

extern "C" int ssd3d_decode_bin_anchor_rows(long rows, int bin_num, float half_bin_search_range, int angle_bins,
                                            const float *anchors, int ld_anchors, const float *pred_reg, int ld_reg,
                                            const float *pred_cls, int ld_cls, const int *pool_cnt, float *boxes, float *scores,
                                            ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(rows >= 0 && bin_num >= 1 && angle_bins >= 1 && ld_anchors >= 7 &&
                  ld_reg >= 4 * bin_num + 4 + 2 * angle_bins && ld_cls >= 2,
                  "decode_bin_anchor_rows: bad shape rows=%ld bins=%d angle_bins=%d ld_anchors=%d ld_reg=%d ld_cls=%d", rows,
                  bin_num, angle_bins, ld_anchors, ld_reg, ld_cls);
    if (rows == 0) return 0;
    SSD3D_REQUIRE(anchors && pred_reg && pred_cls && boxes && scores, "decode_bin_anchor_rows: null pointer");
    const float bin_interval = (float)((double)half_bin_search_range * 2.0 / bin_num);     // as ssd3d_decode_bin_anchor
    const float angle_interval = (float)(2.0 * 3.14159265358979323846 / angle_bins);
    decode_bin_rows_kernel<<<(int)((rows + 127) / 128), 128, 0, (cudaStream_t)stream>>>(
        rows, bin_num, angle_bins, anchors, ld_anchors, pred_reg, ld_reg, pred_cls, ld_cls, pool_cnt, half_bin_search_range,
        bin_interval, angle_interval, boxes, scores);
    SSD3D_LAUNCH_CHECK("decode_bin_rows_kernel");
}

extern "C" int ssd3d_concat_rows(int b, int parts, const float *const *src, const int *m, int c, float *out,
                                 ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && parts >= 1 && parts <= 8 && c >= 1, "concat_rows: bad shape b=%d parts=%d c=%d", b, parts, c);
    SSD3D_REQUIRE(src && m && out, "concat_rows: null pointer");
    ConcatRowsArgs a = {};
    a.parts = parts; a.c = c;
    int tot = 0;
    for (int i = 0; i < parts; i++) {
        SSD3D_REQUIRE(src[i] != nullptr && m[i] >= 0, "concat_rows: part %d is null or negative", i);
        a.src[i] = src[i]; a.m[i] = m[i]; a.start[i] = tot;
        tot += m[i];
    }
    a.mtot = tot;
    if (b == 0 || tot == 0) return 0;
    concat_rows_kernel<<<grid_for((long)b * tot * c, 256), 256, 0, (cudaStream_t)stream>>>(b, a, out);
    SSD3D_LAUNCH_CHECK("concat_rows_kernel");
}

extern "C" int ssd3d_fill_zero(float *x, long count, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(count >= 0, "fill_zero: negative count");
    if (count == 0) return 0;
    SSD3D_REQUIRE(x != nullptr && (reinterpret_cast<uintptr_t>(x) & 15u) == 0, "fill_zero: pointer must be non-null and 16-byte aligned");
    const long n4 = count / 4;
    fill_zero_kernel<<<grid_for(n4 > 0 ? n4 : 1, 256), 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<float4 *>(x), n4, x + n4 * 4,
                                                                                       (int)(count - n4 * 4));
    SSD3D_LAUNCH_CHECK("fill_zero_kernel");
}
