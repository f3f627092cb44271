// nms.cu -- per-scene greedy BEV non-maximum suppression on the GPU (SURVEY.md section 8f, row f2).
//
// Replaces the per-scene, per-class tf.image.non_max_suppression call of the reference's post-processor
// (/root/reference/lib/builder/postprocessor.py:76-88), which runs on the CPU in the middle of inference, together
// with the projections that feed it: box_3d_to_anchor (lib/utils/box_3d_utils.py:25-58) and project_to_bev
// (lib/utils/anchors_util.py:11-48).  Semantics kept: candidates in descending score order (ties: lower index
// first), a candidate is dropped when its axis-aligned BEV IoU with an already kept box is > iou_threshold, at most
// max_output boxes are kept.  Output is the fixed-size block the multi-GPU gather moves: [max_output, 9] =
// (x, y, z, l, h, w, ry, score, class) zero padded, plus the number of kept boxes.
//
// One CTA of 1024 threads per scene, up to 16384 candidates: the 64-bit keys are bitonic-sorted in shared memory (128 KiB
// at n = 16384), then the sorted candidates are walked in chunks of 32: each chunk is tested against the kept set (at
// most max_output boxes) and against itself in parallel, then resolved greedily in order; the walk stops once
// max_output boxes are kept; ssd3d_bev_nms_counted takes only the first n_valid[scene] candidates of each scene (PointRCNN's
// stage 2, whose proposal rows past the RPN's count are padding).  (An n x n suppression matrix would need 32 MiB per scene at n = 16384; at 3DSSD's
// n = 256 the chunked walk also measured faster than the matrix kernel it replaced, BASELINE.md.)
//
// The rectangles and the IoU follow the recipe of DESIGN.md section 3.5, which the numpy and C restatements of the test
// suite share, so that all three make the same decision at an IoU an ulp from the threshold:
// |cos ry|, |sin ry| in double rounded once to float; every product, sum and quotient through an _rn intrinsic, which
// nvcc and ptxas never contract into an FMA (the library is built with -fmad=true).
#include "common.cuh"

namespace ssd3d {

constexpr int NMS_THREADS = 1024;
constexpr int NMS_MAX_N = 16384;            // 128 KiB of sort keys
constexpr int NMS_CHUNK = 32;
constexpr size_t NMS_SMEM_MAX = 226 * 1024;   // dynamic shared memory; the static chunk arrays take the rest of 227 KiB

// Order-preserving key of a score; -0 is mapped to +0 first, so equal scores of either sign tie (lower index first).
// NaN scores are outside the contract.
__device__ __forceinline__ uint32_t nms_f2ord(float x)
{
    const uint32_t b = x == 0.0f ? 0u : __float_as_uint(x);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

__device__ __forceinline__ unsigned long long nms_key(const float *sc, int lds, int i)
{
    return ((unsigned long long)nms_f2ord(sc[(size_t)i * lds]) << 32) | (unsigned long long)(0xffffffffu - (uint32_t)i);
}
__device__ __forceinline__ int nms_key_index(unsigned long long key) { return (int)(0xffffffffu - (uint32_t)(key & 0xffffffffull)); }

// BEV rectangle (x1, z1, x2, z2) of a box (x, y, z, l, h, w, ry): box_3d_to_anchor + project_to_bev by DESIGN.md §3.5
__device__ __forceinline__ float4 nms_rect(const float *b7)
{
    const float x = b7[0], z = b7[2], l = b7[3], w = b7[5], ry = b7[6];
    double sd, cd;
    sincos((double)ry, &sd, &cd);
    const float c = fabsf((float)cd), s = fabsf((float)sd);
    const float dimx = __fadd_rn(__fmul_rn(l, c), __fmul_rn(w, s));
    const float dimz = __fadd_rn(__fmul_rn(w, c), __fmul_rn(l, s));
    const float hx = __fmul_rn(dimx, 0.5f), hz = __fmul_rn(dimz, 0.5f);
    return make_float4(__fsub_rn(x, hx), __fsub_rn(z, hz), __fadd_rn(x, hx), __fadd_rn(z, hz));
}
__device__ __forceinline__ float nms_area(float4 a) { return __fmul_rn(__fsub_rn(a.z, a.x), __fsub_rn(a.w, a.y)); }

// Does the IoU of a and b exceed thr?  A rectangle of area <= 0 neither suppresses nor is suppressed.
__device__ __forceinline__ bool nms_over(float4 a, float area_a, float4 b, float area_b, float thr)
{
    if (area_a <= 0.0f || area_b <= 0.0f) return false;
    const float iw = __fsub_rn(fminf(a.z, b.z), fmaxf(a.x, b.x)), ih = __fsub_rn(fminf(a.w, b.w), fmaxf(a.y, b.y));
    // disjoint rectangles (the common case): inter == 0, IoU == 0 (or NaN), never > threshold -- skip the divide
    if (thr >= 0.0f && (!(iw > 0.0f) || !(ih > 0.0f))) return false;
    const float inter = __fmul_rn(fmaxf(iw, 0.0f), fmaxf(ih, 0.0f));
    return __fdiv_rn(inter, __fsub_rn(__fadd_rn(area_a, area_b), inter)) > thr;
}

// Descending bitonic sort of keys[0 .. npow2) by all threads of the block, one compare-exchange pair per thread and step
__device__ __forceinline__ void nms_sort_desc(unsigned long long *keys, int npow2)
{
    for (int k = 2; k <= npow2; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int p = threadIdx.x; p < (npow2 >> 1); p += blockDim.x) {
                const int i = ((p & ~(j - 1)) << 1) | (p & (j - 1)), ixj = i | j;
                const unsigned long long a = keys[i], b = keys[ixj];
                const bool desc = (i & k) == 0;
                if (desc ? (a < b) : (a > b)) { keys[i] = b; keys[ixj] = a; }
            }
            __syncthreads();
        }
}

// The fixed-size output block of one scene from the kept sorted positions (or, kept_src, the kept box indices)
__device__ __forceinline__ void nms_write_block(int cnt, const int *kept_src, const float *bx, const float *sc, int lds, int max_out,
                                                int cls_id, float *ob)
{
    for (int e = threadIdx.x; e < max_out * 9; e += blockDim.x) {
        const int k = e / 9, f = e - k * 9;
        float v = 0.0f;
        if (k < cnt) {
            const int src = kept_src[k];
            v = f < 7 ? bx[(size_t)src * 7 + f] : (f == 7 ? sc[(size_t)src * lds] : (float)cls_id);
        }
        ob[e] = v;
    }
}

// Shared memory of the kernels: keys[npow2] | kept rect[kcap] | kept area[kcap] | kept src[kcap] (kcap = min(n, max_out))
__host__ __device__ static size_t nms_keys_bytes(int npow2) { return ((size_t)npow2 * 8 + 15) & ~(size_t)15; }
static size_t nms_smem_bytes(int npow2, int kcap) { return nms_keys_bytes(npow2) + (size_t)kcap * (16 + 4 + 4); }

// The static shared state of one chunked walk
struct NmsChunk {
    float4 crect[NMS_CHUNK];
    float carea[NMS_CHUNK];
    uint32_t cself[NMS_CHUNK];     // cself[t] bit j: chunk candidate j (< t) suppresses candidate t
    uint32_t cbykept;              // bit t: candidate t is suppressed by an already kept box
    int nkept;
};

// The greedy NMS of one scene by the whole CTA: candidates 0 .. nv-1 with scores sc[i * lds] sorted by key, then walked
// in chunks of 32.  On return (after a barrier) ch.nkept boxes are kept, their box indices in ksrc[0 .. nkept).
__device__ __forceinline__ void nms_walk(int npow2, int kcap, int nv, const float *bx, const float *sc, int lds, float iou_thr,
                                         int max_out, unsigned char *smem, NmsChunk &ch, int *&ksrc_out)
{
    unsigned long long *keys = reinterpret_cast<unsigned long long *>(smem);
    float4 *krect = reinterpret_cast<float4 *>(smem + nms_keys_bytes(npow2));
    float *karea = reinterpret_cast<float *>(krect + kcap);
    int *ksrc = reinterpret_cast<int *>(karea + kcap);
    ksrc_out = ksrc;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

    for (int i = tid; i < npow2; i += NMS_THREADS) keys[i] = i < nv ? nms_key(sc, lds, i) : 0ull;
    if (tid == 0) ch.nkept = 0;
    __syncthreads();
    nms_sort_desc(keys, npow2);

    for (int base = 0; base < nv; base += NMS_CHUNK) {
        const int nk = ch.nkept;              // read by all threads after the barrier that ended the last step
        if (nk >= max_out) break;
        const int cn = min(NMS_CHUNK, nv - base);
        if (tid < cn) {
            const float4 r = nms_rect(bx + (size_t)nms_key_index(keys[base + tid]) * 7);
            ch.crect[tid] = r;
            ch.carea[tid] = nms_area(r);
        }
        if (tid == 0) ch.cbykept = 0u;
        __syncthreads();
        // candidate `lane` against kept boxes warp, warp + 32, ...; warp t also builds row t of the chunk's own matrix
        if (lane < cn) {
            const float4 a = ch.crect[lane];
            const float aa = ch.carea[lane];
            bool hit = false;
            for (int u = warp; u < nk && !hit; u += NMS_THREADS / 32) hit = nms_over(krect[u], karea[u], a, aa, iou_thr);
            if (hit) atomicOr(&ch.cbykept, 1u << lane);
        }
        if (warp < cn) {
            const bool sup = lane < warp && nms_over(ch.crect[lane], ch.carea[lane], ch.crect[warp], ch.carea[warp], iou_thr);
            const uint32_t row = __ballot_sync(0xffffffffu, sup);
            if (lane == 0) ch.cself[warp] = row;
        }
        __syncthreads();
        if (tid == 0) {                       // greedy, in sorted order, within the chunk
            const uint32_t alive = ~ch.cbykept;
            uint32_t taken = 0u;
            int k = nk;
            for (int t = 0; t < cn && k < max_out; t++) {
                if (!((alive >> t) & 1u) || (ch.cself[t] & taken)) continue;
                taken |= 1u << t;
                krect[k] = ch.crect[t];
                karea[k] = ch.carea[t];
                ksrc[k] = nms_key_index(keys[base + t]);
                k++;
            }
            ch.nkept = k;
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(NMS_THREADS)
bev_nms_kernel(int n, int npow2, int kcap, const float *__restrict__ boxes, const float *__restrict__ scores,
                     const int *__restrict__ n_valid, float iou_thr, int max_out, int cls_id, float *__restrict__ out_block,
                     int *__restrict__ out_cnt)
{
    extern __shared__ __align__(16) unsigned char nms_smem[];
    __shared__ NmsChunk ch;
    const int scene = blockIdx.x;
    const float *bx = boxes + (size_t)scene * n * 7;
    const float *sc = scores + (size_t)scene * n;
    // candidates n_valid[scene] .. n-1 are padding: key 0 sorts them last and the walk stops before them
    const int nv = n_valid == nullptr ? n : max(0, min(n, n_valid[scene]));
    int *ksrc;
    nms_walk(npow2, kcap, nv, bx, sc, 1, iou_thr, max_out, nms_smem, ch, ksrc);
    const int cnt = ch.nkept;
    nms_write_block(cnt, ksrc, bx, sc, 1, max_out, cls_id, out_block + (size_t)scene * max_out * 9);
    if (threadIdx.x == 0) out_cnt[scene] = cnt;
}

// Per-class NMS of one scene by a cluster of ncls CTAs (DESIGN.md section 3.17): CTA rank c walks class c's scores
// (scores[scene, i, c]); the kept counts are exchanged over distributed shared memory, so that each CTA writes its rows
// at the sum of the lower ranks' counts, class-major and compacted, in the same launch.
__global__ void __launch_bounds__(NMS_THREADS)
bev_nms_classes_kernel(int n, int npow2, int kcap, int ncls, const float *__restrict__ boxes, const float *__restrict__ scores,
                       float iou_thr, int max_out, float *__restrict__ out_block, int *__restrict__ out_cnt)
{
    extern __shared__ __align__(16) unsigned char nms_smem[];
    __shared__ NmsChunk ch;
    __shared__ int row0, total;
    const int c = (int)cluster_ctarank(), scene = (int)cluster_id_x();
    const float *bx = boxes + (size_t)scene * n * 7;
    const float *sc = scores + (size_t)scene * n * ncls + c;
    int *ksrc;
    nms_walk(npow2, kcap, n, bx, sc, ncls, iou_thr, max_out, nms_smem, ch, ksrc);
    cluster_sync_all();                                    // every rank's ch.nkept is final
    if (threadIdx.x == 0) {
        int below = 0, all = 0;
        const uint32_t at = smem_u32(&ch.nkept);
        for (int r = 0; r < ncls; r++) {
            int v;
            asm volatile("ld.shared::cluster.s32 %0, [%1];" : "=r"(v) : "r"(mapa(at, (uint32_t)r)) : "memory");
            if (r < c) below += v;
            all += v;
        }
        row0 = below;
        total = all;
    }
    cluster_sync_all();                                    // no CTA leaves while a peer may still read its count
    const int cnt = ch.nkept, rows = ncls * max_out;
    float *ob = out_block + (size_t)scene * rows * 9;
    for (int e = threadIdx.x; e < cnt * 9; e += blockDim.x) {
        const int k = e / 9, f = e - k * 9, src = ksrc[k];
        ob[(size_t)row0 * 9 + e] = f < 7 ? bx[(size_t)src * 7 + f] : (f == 7 ? sc[(size_t)src * ncls] : (float)c);
    }
    if (c == ncls - 1)
        for (int e = total * 9 + threadIdx.x; e < rows * 9; e += blockDim.x) ob[e] = 0.0f;
    if (c == 0 && threadIdx.x == 0) out_cnt[scene] = total;
}

}  // namespace ssd3d

using namespace ssd3d;

// The shared memory of one scene's walk: sort keys of npow2 >= n candidates and kcap = min(n, max_output) kept boxes
static size_t nms_plan(int n, int max_output, int &npow2, int &kcap)
{
    npow2 = 1;
    while (npow2 < n) npow2 <<= 1;
    kcap = max_output < n ? max_output : n;
    return nms_smem_bytes(npow2, kcap);
}

static int bev_nms_launch(const char *op, int b, int n, const float *boxes, const float *scores, const int *n_valid,
                          float iou_threshold, int max_output, int cls_id, float *out_block, int *out_cnt, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && n > 0 && max_output > 0, "%s: bad shape b=%d n=%d max_output=%d", op, b, n, max_output);
    SSD3D_REQUIRE(n <= NMS_MAX_N, "%s: at most %d candidates per scene (got %d)", op, NMS_MAX_N, n);
    if (b == 0) return 0;                    // nothing read or written: an empty tensor may have a null data pointer
    SSD3D_REQUIRE(boxes && scores && out_block && out_cnt, "%s: null pointer", op);
    int npow2, kcap;
    const size_t smem = nms_plan(n, max_output, npow2, kcap);
    SSD3D_REQUIRE(smem <= NMS_SMEM_MAX, "%s: max_output=%d at n=%d needs %zu bytes of shared memory (at most %zu)",
                  op, max_output, n, smem, NMS_SMEM_MAX);
    const int e = cuda_status(cudaFuncSetAttribute(bev_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                              "bev_nms_kernel shared memory");
    if (e) return e;
    bev_nms_kernel<<<b, NMS_THREADS, smem, (cudaStream_t)stream>>>(n, npow2, kcap, boxes, scores, n_valid, iou_threshold,
                                                                   max_output, cls_id, out_block, out_cnt);
    SSD3D_LAUNCH_CHECK("bev_nms_kernel");
}

extern "C" int ssd3d_bev_nms(int b, int n, const float *boxes, const float *scores, float iou_threshold, int max_output,
                             int cls_id, float *out_block, int *out_cnt, ssd3d_stream_t stream)
{
    return bev_nms_launch("bev_nms", b, n, boxes, scores, nullptr, iou_threshold, max_output, cls_id, out_block, out_cnt,
                          stream);
}

extern "C" int ssd3d_bev_nms_counted(int b, int n, const float *boxes, const float *scores, const int *n_valid,
                                     float iou_threshold, int max_output, int cls_id, float *out_block, int *out_cnt,
                                     ssd3d_stream_t stream)
{
    if (b > 0) SSD3D_REQUIRE(n_valid != nullptr, "bev_nms_counted: null n_valid");
    return bev_nms_launch("bev_nms_counted", b, n, boxes, scores, n_valid, iou_threshold, max_output, cls_id, out_block,
                          out_cnt, stream);
}

extern "C" int ssd3d_bev_nms_classes(int b, int n, int cls_num, const float *boxes, const float *scores, float iou_threshold,
                                     int max_output, float *out_block, int *out_cnt, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && n > 0 && max_output > 0 && cls_num >= 1 && cls_num <= SSD3D_MAX_CLASSES,
                  "bev_nms_classes: bad shape b=%d n=%d max_output=%d cls_num=%d (1..%d)", b, n, max_output, cls_num,
                  SSD3D_MAX_CLASSES);
    SSD3D_REQUIRE(n <= NMS_MAX_N, "bev_nms_classes: at most %d candidates per scene (got %d)", NMS_MAX_N, n);
    if (b == 0) return 0;
    SSD3D_REQUIRE(boxes && scores && out_block && out_cnt, "bev_nms_classes: null pointer");
    int npow2, kcap;
    const size_t smem = nms_plan(n, max_output, npow2, kcap);
    SSD3D_REQUIRE(smem <= NMS_SMEM_MAX, "bev_nms_classes: max_output=%d at n=%d needs %zu bytes of shared memory (at most %zu)",
                  max_output, n, smem, NMS_SMEM_MAX);
    int e = cuda_status(cudaFuncSetAttribute(bev_nms_classes_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                        "bev_nms_classes_kernel shared memory");
    if (e) return e;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)(b * cls_num));
    cfg.blockDim = dim3(NMS_THREADS);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = (cudaStream_t)stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)cls_num;
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    int clusters = 0;
    e = cuda_status(cudaOccupancyMaxActiveClusters(&clusters, bev_nms_classes_kernel, &cfg), "bev_nms_classes occupancy");
    if (e) return e;
    SSD3D_REQUIRE(clusters >= 1, "bev_nms_classes: a cluster of %d CTAs with %zu bytes of shared memory each cannot be placed",
                  cls_num, smem);
    e = cuda_status(cudaLaunchKernelEx(&cfg, bev_nms_classes_kernel, n, npow2, kcap, cls_num, boxes, scores, iou_threshold,
                                       max_output, out_block, out_cnt), "bev_nms_classes_kernel");
    if (e) return e;
    SSD3D_LAUNCH_CHECK("bev_nms_classes_kernel");
}
