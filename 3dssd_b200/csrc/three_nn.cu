// three_nn.cu -- three nearest known points per unknown point.
//
// Replaces three_nn_gpu (/root/reference/lib/utils/tf_ops/interpolation/tf_interpolate_g.cu:24-84; CPU twin
// tf_interpolate.cpp:86-129).  The reference runs one thread per unknown point with a serial loop over the
// m known points read from global memory; here a block stages the known points once per 1024-point tile in
// shared memory (read by all lanes as a broadcast) and every thread keeps its running best-3 in registers
// (three_nn.cuh, which also states why the indices and distances are the reference's bit for bit).
#include "three_nn.cuh"

namespace ssd3d {

constexpr int TNN_THREADS = 256;

__global__ void __launch_bounds__(TNN_THREADS)
three_nn_kernel(int n, int m, const float *__restrict__ xyz1, const float *__restrict__ xyz2,
                float *__restrict__ dist, int *__restrict__ idx)
{
    __shared__ float tile[TNN_TILE * 3];
    const int scene = blockIdx.y;
    const int i = blockIdx.x * TNN_THREADS + threadIdx.x;
    const bool valid = i < n;
    const float *u = xyz1 + ((size_t)scene * n + (valid ? i : 0)) * 3;
    float best[3];
    int bidx[3];
    three_nn_scan(m, xyz2 + (size_t)scene * m * 3, tile, u[0], u[1], u[2], best, bidx);
    if (valid) {
        const size_t o = ((size_t)scene * n + i) * 3;
        dist[o] = best[0]; dist[o + 1] = best[1]; dist[o + 2] = best[2];
        idx[o] = bidx[0]; idx[o + 1] = bidx[1]; idx[o + 2] = bidx[2];
    }
}

}  // namespace ssd3d

using namespace ssd3d;

extern "C" int ssd3d_three_nn(int b, int n, int m, const float *xyz1, const float *xyz2, float *dist, int *idx,
                              ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && n >= 0 && m >= 0, "three_nn: bad shape b=%d n=%d m=%d", b, n, m);
    SSD3D_REQUIRE(xyz1 && xyz2 && dist && idx, "three_nn: null pointer");
    if (b == 0 || n == 0) return 0;
    dim3 grid((unsigned)ceil_div(n, TNN_THREADS), (unsigned)b);
    three_nn_kernel<<<grid, TNN_THREADS, 0, (cudaStream_t)stream>>>(n, m, xyz1, xyz2, dist, idx);
    SSD3D_LAUNCH_CHECK("three_nn_kernel");
}
