// grad.cu -- backward operators of the index-driven copies (SURVEY.md section 8f, row f3), so that gather_point, group_point
// and three_interpolate stay drop-ins for training graphs as well.
//
// Replaces scatteraddpointKernel (/root/reference/lib/utils/tf_ops/sampling/tf_sampling_g.cu:335-346),
// group_point_grad_gpu (grouping/tf_grouping_g.cu:383-398) and three_interpolate_grad_gpu
// (interpolation/tf_interpolate_g.cu:115-140).  Like the reference they scatter with fp32 atomicAdd (RED.ADD on
// sm_90a), so sums over repeated indices are order-dependent in the last bits: tolerance parity, not bit parity.
// The zero-fill the reference's TF op does with cudaMemset before the launcher (tf_sampling.cpp:286,
// tf_grouping.cpp:510, tf_interpolate.cpp:398) is part of these entry points (cudaMemsetAsync on the same stream).
#include "common.cuh"

namespace ssd3d {

// dst[scene(row), idx[row], :] += w(row) * src[row, :]
__global__ void scatter_add_rows_kernel(long rows, long rows_per_scene, int n, int c, const float *__restrict__ src,
                                        const int *__restrict__ idx, float *__restrict__ dst, int skip_neg)
{
    const long total = rows * c;
    for (long e = blockIdx.x * (long)blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x) {
        const long row = e / c;
        const int ch = (int)(e - row * c);
        const int a = __ldg(idx + row);
        if (skip_neg && a == -1) continue;
        const long scene = row / rows_per_scene;
        atomicAdd(dst + ((size_t)scene * n + a) * c + ch, __ldg(src + e));
    }
}

// grad_points[b, idx[b,i,k], ch] += grad_out[b,i,ch] * weight[b,i,k]   k = 0..2
__global__ void three_interpolate_grad_kernel(long total, int n, int c, int m, const float *__restrict__ grad_out,
                                              const int *__restrict__ idx, const float *__restrict__ weight,
                                              float *__restrict__ grad_points)
{
    for (long e = blockIdx.x * (long)blockDim.x + threadIdx.x; e < total; e += (long)gridDim.x * blockDim.x) {
        const long pt = e / c;
        const int ch = (int)(e - pt * c);
        const long scene = pt / n;
        float *gp = grad_points + (size_t)scene * m * c;
        const float g = __ldg(grad_out + e);
#pragma unroll
        for (int k = 0; k < 3; k++)
            atomicAdd(gp + (size_t)__ldg(idx + pt * 3 + k) * c + ch, __fmul_rn(g, __ldg(weight + pt * 3 + k)));
    }
}

static int grid_for(long total)
{
    const long want = (total + 255) / 256;
    return (int)(want < (long)kNumSMs * 16 ? want : (long)kNumSMs * 16);
}

}  // namespace ssd3d

using namespace ssd3d;

extern "C" int ssd3d_gather_point_grad(int b, int n, int m, int c, const float *out_g, const int *idx, float *inp_g,
                                       ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && n > 0 && m >= 0 && c >= 0, "gather_point_grad: bad shape");
    SSD3D_REQUIRE(out_g && idx && inp_g, "gather_point_grad: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(inp_g, 0, sizeof(float) * (size_t)b * n * c, st);
    if (e != cudaSuccess) return cuda_status(e, "gather_point_grad memset");
    const long total = (long)b * m * c;
    if (total == 0) return 0;
    scatter_add_rows_kernel<<<grid_for(total), 256, 0, st>>>((long)b * m, m, n, c, out_g, idx, inp_g, 0);
    SSD3D_LAUNCH_CHECK("gather_point_grad");
}

extern "C" int ssd3d_group_point_grad(int b, int n, int c, int m, int nsample, const float *grad_out, const int *idx,
                                      float *grad_points, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && n > 0 && m >= 0 && c >= 0 && nsample >= 0, "group_point_grad: bad shape");
    SSD3D_REQUIRE(grad_out && idx && grad_points, "group_point_grad: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(grad_points, 0, sizeof(float) * (size_t)b * n * c, st);
    if (e != cudaSuccess) return cuda_status(e, "group_point_grad memset");
    const long total = (long)b * m * nsample * c;
    if (total == 0) return 0;
    scatter_add_rows_kernel<<<grid_for(total), 256, 0, st>>>((long)b * m * nsample, (long)m * nsample, n, c, grad_out, idx,
                                                            grad_points, 1);
    SSD3D_LAUNCH_CHECK("group_point_grad");
}

extern "C" int ssd3d_three_interpolate_grad(int b, int n, int c, int m, const float *grad_out, const int *idx,
                                            const float *weight, float *grad_points, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && n >= 0 && m > 0 && c >= 0, "three_interpolate_grad: bad shape");
    SSD3D_REQUIRE(grad_out && idx && weight && grad_points, "three_interpolate_grad: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    cudaError_t e = cudaMemsetAsync(grad_points, 0, sizeof(float) * (size_t)b * m * c, st);
    if (e != cudaSuccess) return cuda_status(e, "three_interpolate_grad memset");
    const long total = (long)b * n * c;
    if (total == 0) return 0;
    three_interpolate_grad_kernel<<<grid_for(total), 256, 0, st>>>(total, n, c, m, grad_out, idx, weight, grad_points);
    SSD3D_LAUNCH_CHECK("three_interpolate_grad");
}
