// fp_interp.cu -- the operand of an FP layer's first conv in one launch (DESIGN.md section 3.15).
//
// pointnet_fp_module (/root/reference/lib/utils/layers_util.py:192-225) finds the three nearest known points of every
// unknown point (:206), weights them by inverse distance (:207-210), interpolates the known features (:211), concatenates
// the unknown points' own features (:213-214) and runs the MLP.  Here one kernel does everything up to the MLP and writes
// the concatenated rows directly as the split-bf16 operand [rows, kp] (operand.cuh) that linear_tc reads, so neither the
// interpolated features nor the concatenation exist in HBM in fp32.
//
// Bits: the neighbours come from three_nn_scan and the interpolation from three_interp_value (three_nn.cuh), the code of
// three_nn / three_interpolate themselves; the weights are computed in fp32 with one rounding per operation in the order
// the CPU oracle pins (TF leaves the order of its 3-term reduce_sum open):
//   inv_k = 1 / max(d_k, 1e-10),  norm = (inv_0 + inv_1) + inv_2,  w_k = inv_k / norm.
// The operand is therefore bit for bit split_rows(concat(three_interpolate(points2, idx, w), points1)).
#include "operand.cuh"
#include "three_nn.cuh"

namespace ssd3d {

constexpr int FPI_THREADS = 256;

__global__ void __launch_bounds__(FPI_THREADS)
fp_interp_split_kernel(int n, int m, int c2, int c1, const float *__restrict__ xyz1, const float *__restrict__ xyz2,
                       const float *__restrict__ points2, const float *__restrict__ points1, __nv_bfloat16 *__restrict__ hi,
                       __nv_bfloat16 *__restrict__ lo, int kp)
{
    __shared__ float tile[TNN_TILE * 3];
    __shared__ int s_idx[FPI_THREADS][3];
    __shared__ float s_w[FPI_THREADS][3];
    const int scene = blockIdx.y;
    const int row0 = blockIdx.x * FPI_THREADS;
    const int i = row0 + threadIdx.x;
    const bool valid = i < n;
    const float *u = xyz1 + ((size_t)scene * n + (valid ? i : 0)) * 3;
    float best[3];
    int bidx[3];
    three_nn_scan(m, xyz2 + (size_t)scene * m * 3, tile, u[0], u[1], u[2], best, bidx);
    float inv[3];
#pragma unroll
    for (int k = 0; k < 3; k++) inv[k] = __fdiv_rn(1.0f, fmaxf(best[k], 1e-10f));
    const float norm = __fadd_rn(__fadd_rn(inv[0], inv[1]), inv[2]);
#pragma unroll
    for (int k = 0; k < 3; k++) {
        s_idx[threadIdx.x][k] = bidx[k];
        s_w[threadIdx.x][k] = __fdiv_rn(inv[k], norm);
    }
    __syncthreads();

    // rows of this block, one 8-column chunk per thread and step: consecutive threads write consecutive 16-byte chunks
    const int nrows = min(FPI_THREADS, n - row0);
    const int cpr = kp >> 3;
    const float *p2 = points2 + (size_t)scene * m * c2;
    const int ctot = c2 + c1;
    for (int e = threadIdx.x; e < nrows * cpr; e += FPI_THREADS) {
        const int r = e / cpr, k0 = (e - r * cpr) * 8;
        const size_t grow = (size_t)scene * n + row0 + r;
        const float *q0 = p2 + (size_t)s_idx[r][0] * c2, *q1 = p2 + (size_t)s_idx[r][1] * c2, *q2 = p2 + (size_t)s_idx[r][2] * c2;
        const float w0 = s_w[r][0], w1 = s_w[r][1], w2 = s_w[r][2];
        float f[8];
#pragma unroll
        for (int t = 0; t < 8; t++) {
            const int k = k0 + t;
            float v = 0.0f;
            if (k < c2) v = three_interp_value(w0, w1, w2, __ldg(q0 + k), __ldg(q1 + k), __ldg(q2 + k));
            else if (k < ctot) v = __ldg(points1 + grow * c1 + (k - c2));
            f[t] = v;
        }
        split_store8(hi + grow * kp + k0, lo + grow * kp + k0, f);
    }
}

}  // namespace ssd3d

using namespace ssd3d;

extern "C" int ssd3d_fp_interp_split(int b, int n, int m, int c2, int c1, const float *xyz1, const float *xyz2,
                                     const float *points2, const float *points1, void *out_hi, void *out_lo, int kp,
                                     ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && n >= 0 && m >= 1 && c2 >= 1 && c1 >= 0,
                  "fp_interp_split: bad shape b=%d n=%d m=%d c2=%d c1=%d (at least one known point)", b, n, m, c2, c1);
    SSD3D_REQUIRE(kp >= c2 + c1 && kp % 16 == 0, "fp_interp_split: kp=%d must be a multiple of 16 and >= c2 + c1 = %d", kp,
                  c2 + c1);
    if (b == 0 || n == 0) return 0;
    SSD3D_REQUIRE(xyz1 && xyz2 && points2 && (points1 || c1 == 0) && out_hi && out_lo, "fp_interp_split: null pointer");
    SSD3D_REQUIRE(((reinterpret_cast<uintptr_t>(out_hi) | reinterpret_cast<uintptr_t>(out_lo)) & 15u) == 0,
                  "fp_interp_split: outputs must be 16-byte aligned");
    dim3 grid((unsigned)ceil_div(n, FPI_THREADS), (unsigned)b);
    fp_interp_split_kernel<<<grid, FPI_THREADS, 0, (cudaStream_t)stream>>>(n, m, c2, c1, xyz1, xyz2, points2, points1,
                                                                           (__nv_bfloat16 *)out_hi, (__nv_bfloat16 *)out_lo, kp);
    SSD3D_LAUNCH_CHECK("fp_interp_split_kernel");
}
