// gather_group.cu -- index-driven copies: gather_point, group_point, group_concat, three_interpolate.
//
// Replaces gatherpointKernel (/root/reference/lib/utils/tf_ops/sampling/tf_sampling_g.cu:320-331),
// group_point_gpu (grouping/tf_grouping_g.cu:362-379) and three_interpolate_gpu
// (interpolation/tf_interpolate_g.cu:87-113).  The reference launches a fixed <<<512,64>>> grid-stride
// grid whatever the size; here the grid covers the output with 16-byte vector accesses when the channel
// count allows it, so a warp moves whole contiguous rows.
#include "three_nn.cuh"

namespace ssd3d {

// out[row, :] = src[scene(row), idx[row], :]   rows = b*rows_per_scene, c % 4 == 0, 16-byte aligned
__global__ void gather_rows_v4_kernel(long rows, long rows_per_scene, int n, int c4, const float4 *__restrict__ src,
                                      const int *__restrict__ idx, float4 *__restrict__ out, int neg_is_zero,
                                      long idx_scene_stride)
{
    const long total = rows * c4;
    for (long e = blockIdx.x * (long)blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x) {
        const long row = e / c4;
        const int v = (int)(e - row * c4);
        const long scene = row / rows_per_scene;
        const int a = __ldg(idx + scene * idx_scene_stride + (row - scene * rows_per_scene));
        float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
        if (!(neg_is_zero && a == -1)) val = __ldg(src + ((size_t)scene * n + a) * c4 + v);
        out[e] = val;
    }
}

__global__ void gather_rows_kernel(long rows, long rows_per_scene, int n, int c, const float *__restrict__ src,
                                   const int *__restrict__ idx, float *__restrict__ out, int neg_is_zero,
                                   long idx_scene_stride)
{
    const long total = rows * c;
    for (long e = blockIdx.x * (long)blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x) {
        const long row = e / c;
        const int ch = (int)(e - row * c);
        const long scene = row / rows_per_scene;
        const int a = __ldg(idx + scene * idx_scene_stride + (row - scene * rows_per_scene));
        float val = 0.0f;
        if (!(neg_is_zero && a == -1)) val = __ldg(src + ((size_t)scene * n + a) * c + ch);
        out[e] = val;
    }
}

static int launch_gather(long rows, long rows_per_scene, int n, int c, const float *src, const int *idx, float *out,
                         int neg_is_zero, cudaStream_t st, const char *what, long idx_scene_stride = -1)
{
    if (idx_scene_stride < 0) idx_scene_stride = rows_per_scene;
    if (rows == 0 || c == 0) return 0;
    const bool vec = (c % 4 == 0) && ((reinterpret_cast<uintptr_t>(src) & 15u) == 0) &&
                     ((reinterpret_cast<uintptr_t>(out) & 15u) == 0);
    const long total = vec ? rows * (c / 4) : rows * c;
    const int threads = 256;
    const int blocks = (int)((total + threads - 1) / threads < (long)kNumSMs * 16 ? (total + threads - 1) / threads
                                                                                  : (long)kNumSMs * 16);
    if (vec)
        gather_rows_v4_kernel<<<blocks, threads, 0, st>>>(rows, rows_per_scene, n, c / 4, (const float4 *)src, idx,
                                                          (float4 *)out, neg_is_zero, idx_scene_stride);
    else
        gather_rows_kernel<<<blocks, threads, 0, st>>>(rows, rows_per_scene, n, c, src, idx, out, neg_is_zero, idx_scene_stride);
    SSD3D_LAUNCH_CHECK(what);
}

// x[row, 0:c] = points[scene, idx[row], :], x[row, c:c+3] = xyz[scene, idx[row], :] - new_xyz[scene, row/ns, :],
// x[row, c+3:ldx] = 0        (lib/utils/layers_util.py:160-165: features first, then relative xyz)
__global__ void group_concat_kernel(long rows, int n, int c, int m, int ns, const float *__restrict__ xyz,
                                    const float *__restrict__ points, const float *__restrict__ new_xyz,
                                    const int *__restrict__ idx, float *__restrict__ x, int ldx)
{
    const long total = rows * ldx;
    const long rows_per_scene = (long)m * ns;
    for (long e = blockIdx.x * (long)blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x) {
        const long row = e / ldx;
        const int col = (int)(e - row * ldx);
        const long scene = row / rows_per_scene;
        const int a = __ldg(idx + row);
        float val = 0.0f;
        if (col < c) val = __ldg(points + ((size_t)scene * n + a) * c + col);
        else if (col < c + 3) {
            const long q = row / ns;  // == scene*m + query
            val = __ldg(xyz + ((size_t)scene * n + a) * 3 + (col - c)) - __ldg(new_xyz + q * 3 + (col - c));
        }
        x[e] = val;
    }
}

// out[b,i,ch] = fma(w3,c3, fma(w1,c1, w2*c2))   -- three_interp_value, the reference's contraction
__global__ void three_interpolate_kernel(long total, int m, int c, int n, const float *__restrict__ points,
                                         const int *__restrict__ idx, const float *__restrict__ weight,
                                         float *__restrict__ out)
{
    for (long e = blockIdx.x * (long)blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x) {
        const long pt = e / c;
        const int ch = (int)(e - pt * c);
        const long scene = pt / n;
        const float *pts = points + (size_t)scene * m * c;
        const int i1 = __ldg(idx + pt * 3), i2 = __ldg(idx + pt * 3 + 1), i3 = __ldg(idx + pt * 3 + 2);
        const float w1 = __ldg(weight + pt * 3), w2 = __ldg(weight + pt * 3 + 1), w3 = __ldg(weight + pt * 3 + 2);
        const float c1 = __ldg(pts + (size_t)i1 * c + ch), c2 = __ldg(pts + (size_t)i2 * c + ch),
                    c3 = __ldg(pts + (size_t)i3 * c + ch);
        out[e] = three_interp_value(w1, w2, w3, c1, c2, c3);
    }
}

// ymax[g, o] = max_{r in group g} y[g*pool + r, o] * (rowmask ? rowmask[g] != 0 : 1)
__global__ void rowgroup_max_kernel(long groups, int pool, int c, const float *__restrict__ y, int ldy,
                                    const int *__restrict__ rowmask, float *__restrict__ out)
{
    const long total = groups * c;
    for (long e = blockIdx.x * (long)blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x) {
        const long g = e / c;
        const int o = (int)(e - g * c);
        float mx = -INFINITY;
        for (int r = 0; r < pool; r++) mx = fmaxf(mx, y[((size_t)g * pool + r) * ldy + o]);
        if (rowmask && rowmask[g] == 0) mx = 0.0f;
        out[e] = mx;
    }
}

int launch_rowgroup_max(long groups, int pool, int c, const float *y, int ldy, const int *rowmask, float *out,
                        cudaStream_t st)
{
    const long total = groups * c;
    if (total == 0) return 0;
    const int threads = 256;
    const long want = (total + threads - 1) / threads;
    const int blocks = (int)(want < (long)kNumSMs * 16 ? want : (long)kNumSMs * 16);
    rowgroup_max_kernel<<<blocks, threads, 0, st>>>(groups, pool, c, y, ldy, rowmask, out);
    SSD3D_LAUNCH_CHECK("rowgroup_max_kernel");
}

}  // namespace ssd3d

using namespace ssd3d;

extern "C" int ssd3d_gather_point(int b, int n, int m, int c, const float *inp, const int *idx, float *out,
                                  ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && n > 0 && m >= 0 && c >= 0, "gather_point: bad shape b=%d n=%d m=%d c=%d", b, n, m, c);
    SSD3D_REQUIRE(inp && idx && out, "gather_point: null pointer");
    return launch_gather((long)b * m, m, n, c, inp, idx, out, 0, (cudaStream_t)stream, "gather_point");
}

// gather_point reading idx rows ld_idx ints apart (a column block of a wider [b, L] index tensor)
extern "C" int ssd3d_gather_point_ex(int b, int n, int m, int c, const float *inp, const int *idx, int ld_idx, float *out,
                                     ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && n > 0 && m >= 0 && c >= 0 && ld_idx >= m, "gather_point: bad shape b=%d n=%d m=%d c=%d ld_idx=%d", b, n, m, c, ld_idx);
    SSD3D_REQUIRE(inp && idx && out, "gather_point: null pointer");
    return launch_gather((long)b * m, m, n, c, inp, idx, out, 0, (cudaStream_t)stream, "gather_point", ld_idx);
}

extern "C" int ssd3d_group_point(int b, int n, int c, int m, int nsample, const float *points, const int *idx,
                                 float *out, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && n > 0 && m >= 0 && c >= 0 && nsample >= 0, "group_point: bad shape");
    SSD3D_REQUIRE(points && idx && out, "group_point: null pointer");
    return launch_gather((long)b * m * nsample, (long)m * nsample, n, c, points, idx, out, 1, (cudaStream_t)stream,
                         "group_point");
}

extern "C" int ssd3d_group_concat(int b, int n, int c, int m, int nsample, const float *xyz, const float *points,
                                  const float *new_xyz, const int *idx, float *x, int ldx, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && n > 0 && m >= 0 && c >= 0 && nsample > 0, "group_concat: bad shape");
    SSD3D_REQUIRE(ldx >= c + 3, "group_concat: ldx=%d < c+3=%d", ldx, c + 3);
    SSD3D_REQUIRE(xyz && new_xyz && idx && x && (points || c == 0), "group_concat: null pointer");
    const long rows = (long)b * m * nsample;
    if (rows == 0) return 0;
    const long total = rows * ldx;
    const int threads = 256;
    const long want = (total + threads - 1) / threads;
    const int blocks = (int)(want < (long)kNumSMs * 16 ? want : (long)kNumSMs * 16);
    group_concat_kernel<<<blocks, threads, 0, (cudaStream_t)stream>>>(rows, n, c, m, nsample, xyz, points, new_xyz, idx,
                                                                      x, ldx);
    SSD3D_LAUNCH_CHECK("group_concat_kernel");
}

extern "C" int ssd3d_three_interpolate(int b, int m, int c, int n, const float *points, const int *idx,
                                       const float *weight, float *out, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && m > 0 && c >= 0 && n >= 0, "three_interpolate: bad shape");
    SSD3D_REQUIRE(points && idx && weight && out, "three_interpolate: null pointer");
    const long total = (long)b * n * c;
    if (total == 0) return 0;
    const int threads = 256;
    const long want = (total + threads - 1) / threads;
    const int blocks = (int)(want < (long)kNumSMs * 16 ? want : (long)kNumSMs * 16);
    three_interpolate_kernel<<<blocks, threads, 0, (cudaStream_t)stream>>>(total, m, c, n, points, idx, weight, out);
    SSD3D_LAUNCH_CHECK("three_interpolate_kernel");
}
