// prepare.cu -- the per-point half of the reference's KITTI preprocessing pass (KittiDataset.preprocess_samples,
// kitti_dataloader.py:173-228; DESIGN.md section 3.14) on a batch of ragged raw velodyne frames:
//   prep_count_kernel   one CTA per tile of 1024 points of a frame: velo -> rect -> image, the image-FOV and extents
//                       filters, the tile's kept count
//   prep_scan_kernel    one CTA: exclusive scan of the tile counts in (frame, tile) order -> each tile's first output
//                       row and the kept offsets of the frames
//   prep_write_kernel   the tiles again: the same transform recomputed, the kept points written as float64 in input order
// Every product, sum and quotient is rounded once in float64 (no contraction), so a numpy
// restatement in the same order gives the same bits.
// There are no atomics and nothing synchronises the host.
#include "common.cuh"

namespace ssd3d {

constexpr int kPrepThreads = 256;
constexpr int kPrepChunks = 4;                                  // chunks of kPrepThreads points per tile
constexpr int kPrepTile = kPrepThreads * kPrepChunks;
constexpr int kPrepScanThreads = 1024;
constexpr int kPrepCalib = 33;                                   // V2C [3, 4], R0 [3, 3], P2 [3, 4], row-major

// rect (x, y, z) of a velodyne point and whether it passes both filters, in the canonical order of include/ssd3d.h
__device__ __forceinline__ bool prep_point(const float4 p, const double *__restrict__ c, int h, int w,
                                           const double *__restrict__ ext, double r[3])
{
    const double x = (double)p.x, y = (double)p.y, z = (double)p.z;
    const double *V = c, *R = c + 12, *P = c + 21;
    double ref[3];
#pragma unroll
    for (int j = 0; j < 3; j++)
        ref[j] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, V[4 * j]), __dmul_rn(y, V[4 * j + 1])), __dmul_rn(z, V[4 * j + 2])),
                           V[4 * j + 3]);
#pragma unroll
    for (int i = 0; i < 3; i++)
        r[i] = __dadd_rn(__dadd_rn(__dmul_rn(R[3 * i], ref[0]), __dmul_rn(R[3 * i + 1], ref[1])), __dmul_rn(R[3 * i + 2], ref[2]));
    double hk[3];
#pragma unroll
    for (int k = 0; k < 3; k++)
        hk[k] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(r[0], P[4 * k]), __dmul_rn(r[1], P[4 * k + 1])), __dmul_rn(r[2], P[4 * k + 2])),
                          P[4 * k + 3]);
    const double u = __ddiv_rn(hk[0], hk[2]), v = __ddiv_rn(hk[1], hk[2]);    // h2 == 0: inf or NaN, dropped below
    const bool img = u >= 0.0 && u < (double)w && v >= 0.0 && v < (double)h && r[2] >= 0.0;
    const bool box = r[0] > ext[0] && r[0] < ext[1] && r[1] > ext[2] && r[1] < ext[3] && r[2] > ext[4] && r[2] < ext[5];
    return img && box;
}

__global__ void __launch_bounds__(kPrepThreads) prep_count_kernel(const float *__restrict__ pts, const int *__restrict__ offsets,
                                                                  const double *__restrict__ calib, const int *__restrict__ hw,
                                                                  const double *__restrict__ ext, int *__restrict__ tile_counts)
{
    __shared__ double sc[kPrepCalib + 6];
    const int s = blockIdx.y, t = blockIdx.x, tid = threadIdx.x;
    const int o0 = offsets[s], n = offsets[s + 1] - o0;
    for (int k = tid; k < kPrepCalib + 6; k += kPrepThreads) sc[k] = k < kPrepCalib ? calib[(size_t)s * kPrepCalib + k] : ext[k - kPrepCalib];
    __syncthreads();
    const int h = hw[2 * s], w = hw[2 * s + 1];
    const float4 *src = reinterpret_cast<const float4 *>(pts) + o0;
    int total = 0;
    for (int c = 0; c < kPrepChunks; c++) {
        const int p = t * kPrepTile + c * kPrepThreads + tid;
        double r[3];
        total += __syncthreads_count(p < n && prep_point(src[p], sc, h, w, sc + kPrepCalib, r));
    }
    if (tid == 0) tile_counts[(size_t)s * gridDim.x + t] = total;
}

// exclusive scan of n tile counts in place; out_offsets[s] = the first row of frame s (its tile 0), out_offsets[b] = total
__global__ void __launch_bounds__(kPrepScanThreads) prep_scan_kernel(int b, int tiles, int *__restrict__ tile_counts,
                                                                     int *__restrict__ out_offsets)
{
    __shared__ int part[kPrepScanThreads];
    const int tid = threadIdx.x, n = b * tiles;
    const int per = (n + kPrepScanThreads - 1) / kPrepScanThreads, lo = min(n, tid * per), hi = min(n, lo + per);
    int sum = 0;
    for (int i = lo; i < hi; i++) sum += tile_counts[i];
    part[tid] = sum;
    __syncthreads();
    for (int d = 1; d < kPrepScanThreads; d <<= 1) {                            // Hillis-Steele, inclusive
        const int v = tid >= d ? part[tid - d] : 0;
        __syncthreads();
        part[tid] += v;
        __syncthreads();
    }
    int run = part[tid] - sum;
    for (int i = lo; i < hi; i++) {
        const int c = tile_counts[i];
        tile_counts[i] = run;
        if (i % tiles == 0) out_offsets[i / tiles] = run;
        run += c;
    }
    if (tid == kPrepScanThreads - 1) out_offsets[b] = part[tid];
}

__global__ void __launch_bounds__(kPrepThreads) prep_write_kernel(const float *__restrict__ pts, const int *__restrict__ offsets,
                                                                  const double *__restrict__ calib, const int *__restrict__ hw,
                                                                  const double *__restrict__ ext, const int *__restrict__ tile_base,
                                                                  double *__restrict__ out)
{
    __shared__ double sc[kPrepCalib + 6];
    __shared__ int wsum[kPrepThreads / 32];
    const int s = blockIdx.y, t = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int o0 = offsets[s], n = offsets[s + 1] - o0;
    if (t * kPrepTile >= n) return;                                             // the whole CTA
    for (int k = tid; k < kPrepCalib + 6; k += kPrepThreads) sc[k] = k < kPrepCalib ? calib[(size_t)s * kPrepCalib + k] : ext[k - kPrepCalib];
    __syncthreads();
    const int h = hw[2 * s], w = hw[2 * s + 1];
    const float4 *src = reinterpret_cast<const float4 *>(pts) + o0;
    long long row = tile_base[(size_t)s * gridDim.x + t];
    for (int c = 0; c < kPrepChunks; c++) {                                     // block-wide scan of one chunk, in order
        const int p = t * kPrepTile + c * kPrepThreads + tid;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        double r[3];
        bool in = false;
        if (p < n) {
            v = src[p];
            in = prep_point(v, sc, h, w, sc + kPrepCalib, r);
        }
        const unsigned m = __ballot_sync(0xffffffffu, in);
        if (lane == 0) wsum[warp] = __popc(m);
        __syncthreads();
        int before = 0, total = 0;
        for (int k = 0; k < kPrepThreads / 32; k++) {
            before += k < warp ? wsum[k] : 0;
            total += wsum[k];
        }
        if (in) {
            double2 *o = reinterpret_cast<double2 *>(out + (row + before + __popc(m & ((1u << lane) - 1u))) * 4);
            o[0] = make_double2(r[0], r[1]);
            o[1] = make_double2(r[2], (double)v.w);
        }
        row += total;
        __syncthreads();
    }
}

static int prep_tiles(int max_n) { return max_n > 0 ? ceil_div(max_n, kPrepTile) : 1; }

}  // namespace ssd3d

using namespace ssd3d;

extern "C" size_t ssd3d_prepare_workspace(int b, int max_n)
{
    if (b < 1 || b > SSD3D_PREPARE_MAX_FRAMES || max_n < 0 || max_n > SSD3D_PREPARE_MAX_FRAME_POINTS) return 0;
    return (size_t)b * prep_tiles(max_n) * sizeof(int);
}

extern "C" int ssd3d_prepare_points(int b, int max_n, int total, const float *points, const int *offsets, const double *calib,
                                    const int *image_hw, const double *extents, void *workspace, double *out_points,
                                    int *out_offsets, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 1 && b <= SSD3D_PREPARE_MAX_FRAMES && max_n >= 0 && max_n <= SSD3D_PREPARE_MAX_FRAME_POINTS && total >= 0 &&
                      total <= SSD3D_PREPARE_MAX_BATCH_POINTS,
                  "prepare_points: bad shape b=%d max_n=%d total=%d (b <= %d, max_n <= %d, total <= %d)", b, max_n, total,
                  SSD3D_PREPARE_MAX_FRAMES, SSD3D_PREPARE_MAX_FRAME_POINTS, SSD3D_PREPARE_MAX_BATCH_POINTS);
    SSD3D_REQUIRE(offsets && calib && image_hw && extents && workspace && out_offsets && (total == 0 || (points && out_points)),
                  "prepare_points: null pointer");
    const int tiles = prep_tiles(max_n);
    int *counts = static_cast<int *>(workspace);
    const dim3 grid(tiles, b);
    const cudaStream_t st = (cudaStream_t)stream;
    prep_count_kernel<<<grid, kPrepThreads, 0, st>>>(points, offsets, calib, image_hw, extents, counts);
    int e = cuda_status(cudaGetLastError(), "prep_count_kernel");
    if (e) return e;
    prep_scan_kernel<<<1, kPrepScanThreads, 0, st>>>(b, tiles, counts, out_offsets);
    e = cuda_status(cudaGetLastError(), "prep_scan_kernel");
    if (e) return e;
    prep_write_kernel<<<grid, kPrepThreads, 0, st>>>(points, offsets, calib, image_hw, extents, counts, out_points);
    SSD3D_LAUNCH_CHECK("prep_write_kernel");
}
