// mixup.cu -- the mixup paste of 3dssd.yaml (MIXUP.OPEN, DESIGN.md section 3.13) on ragged scenes, and the object
// database it draws from.
//   mix_db_count      one thread per point: how many points of its frame each GT row grown by 0.1 holds
//   mix_db_write      one CTA per database object: its frame's points inside the grown row, in frame order
//   mix_paste_boxes   one CTA per scene: box_3d_collision_test (voxelnet_aug.py:197-248), every pair in parallel, then
//                     the reference's loop in draw order; the kept boxes stand on the frame's ground plane
//   mix_paste_points  one thread per output slot: the scene's points, then each drawn object's points (label -1 when the
//                     object was dropped: the slot holds no point)
// There are no float atomics and the integer atomics only count, so the same inputs give the same bits on every run.
#include <math.h>

#include "box_geom.cuh"

namespace ssd3d {

constexpr int kMixMaxRows = 256;               // G + S per scene
constexpr int kMixMaxSlots = 131072;           // points per scene, before and after the paste
constexpr int kMixThreads = 256;
constexpr float kMixExpand = 0.1f;             // EXPAND_DIMS_LENGTH: the database's membership box
constexpr float kMixGrowL = 0.5f, kMixGrowW = 0.5f;   // enlarge_range (l, w) of box_3d_collision_test; h is not in the BEV

__device__ __forceinline__ void row_planes(const float *b, Planes &P)
{
    float sn, cs;
    sincos32((double)b[6], sn, cs);
    box_planes(b, kMixExpand, sn, cs, P);
}

// box_3d_collision_test's height move in float64 with the float64 plane (a, b, c, d):
// h = ((-d - a x) - c z) / b, move = y - h; a y becomes rn32(rn64(y - move))
__device__ __forceinline__ double move_height(const float *box, const double *pl)
{
    const double h = __ddiv_rn(__dsub_rn(__dsub_rn(-pl[3], __dmul_rn(pl[0], (double)box[0])), __dmul_rn(pl[2], (double)box[2])), pl[1]);
    return __dsub_rn((double)box[1], h);
}

__global__ void __launch_bounds__(kMixThreads) mix_db_count_kernel(int g, const float *__restrict__ pts, const int *__restrict__ offsets,
                                                                   const float *__restrict__ boxes, int *__restrict__ counts)
{
    __shared__ Planes sp[kMixMaxRows];
    __shared__ unsigned char sv[kMixMaxRows];
    __shared__ int sc[kMixMaxRows];
    const int s = blockIdx.y, p = blockIdx.x * blockDim.x + threadIdx.x;
    const int o0 = offsets[s], n = offsets[s + 1] - o0;
    if (blockIdx.x * blockDim.x >= n) return;                                   // the whole CTA
    for (int j = threadIdx.x; j < g; j += blockDim.x) {
        const float *b = boxes + ((size_t)s * g + j) * 7;
        sv[j] = box_is_valid(b);
        sc[j] = 0;
        if (sv[j]) row_planes(b, sp[j]);
    }
    __syncthreads();
    if (p < n) {
        const size_t gi = (size_t)o0 + p;
        const float x = pts[gi * 4], y = pts[gi * 4 + 1], z = pts[gi * 4 + 2];
        for (int j = 0; j < g; j++)
            if (sv[j] && inside(sp[j], x, z, y)) atomicAdd(&sc[j], 1);
    }
    __syncthreads();
    for (int j = threadIdx.x; j < g; j += blockDim.x)
        if (sc[j]) atomicAdd(counts + (size_t)s * g + j, sc[j]);
}

__global__ void __launch_bounds__(kMixThreads) mix_db_write_kernel(
    int g, const float *__restrict__ pts, const int *__restrict__ offsets, const float *__restrict__ boxes,
    const int *__restrict__ objects, const long long *__restrict__ obj_off, float *__restrict__ out)
{
    __shared__ int wsum[kMixThreads / 32];
    __shared__ Planes P;
    const int o = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int s = objects[2 * o], j = objects[2 * o + 1];
    const int o0 = offsets[s], n = offsets[s + 1] - o0;
    if (tid == 0) row_planes(boxes + ((size_t)s * g + j) * 7, P);
    __syncthreads();
    long long w = obj_off[o];
    const float4 *src = reinterpret_cast<const float4 *>(pts) + o0;
    for (int c0 = 0; c0 < n; c0 += kMixThreads) {                              // block-wide scan of one chunk, in order
        const int p = c0 + tid;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        bool in = false;
        if (p < n) {
            v = src[p];
            in = inside(P, v.x, v.z, v.y);
        }
        const unsigned m = __ballot_sync(0xffffffffu, in);
        if (lane == 0) wsum[warp] = __popc(m);
        __syncthreads();
        int before = 0, total = 0;
        for (int k = 0; k < kMixThreads / 32; k++) {
            before += k < warp ? wsum[k] : 0;
            total += wsum[k];
        }
        if (in) reinterpret_cast<float4 *>(out)[w + before + __popc(m & ((1u << lane) - 1u))] = v;
        w += total;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kMixThreads) mix_paste_boxes_kernel(
    int g, int ns, const float *__restrict__ boxes, const int *__restrict__ labels, const int *__restrict__ ids,
    const float *__restrict__ db_boxes, const int *__restrict__ db_classes, const double *__restrict__ planes,
    float *__restrict__ out_boxes, int *__restrict__ out_labels, int *__restrict__ accepted)
{
    __shared__ float qc[kMixMaxRows][4][2];         // BEV corners of the scene's rows
    __shared__ float dc[kMixMaxRows][4][2];         // ... of the drawn boxes as they are (they join q_boxes when kept)
    __shared__ float ec[kMixMaxRows][4][2];         // ... of the drawn boxes grown by enlarge_range
    __shared__ unsigned pm[kMixMaxRows][kMixMaxRows / 32];   // bit k of row i: grown drawn i collides with drawn k < i
    __shared__ int hit[kMixMaxRows];                // grown drawn i collides with a valid scene row
    __shared__ unsigned char qv[kMixMaxRows];
    __shared__ short src[kMixMaxRows];              // output row -> scene row j, g + drawn i, or -1 (zeros)
    __shared__ unsigned char keep[kMixMaxRows];
    __shared__ unsigned kept[kMixMaxRows / 32];    // bit i: drawn i is kept
    const int s = blockIdx.x, tid = threadIdx.x, rows = g + ns;
    const int *sid = ids + (size_t)s * ns;
    for (int j = tid; j < g; j += blockDim.x) {
        const float *b = boxes + ((size_t)s * g + j) * 7;
        qv[j] = box_is_valid(b);
        if (qv[j]) {
            float sn, cs;
            sincos32((double)b[6], sn, cs);
            bev_corners(b[0], b[2], b[3], b[5], sn, cs, qc[j]);
        }
    }
    for (int i = tid; i < ns; i += blockDim.x) {
        hit[i] = 0;
        for (int k = 0; k < kMixMaxRows / 32; k++) pm[i][k] = 0u;
        if (sid[i] < 0) continue;
        const float *b = db_boxes + (size_t)sid[i] * 7;
        float sn, cs;
        sincos32((double)b[6], sn, cs);
        bev_corners(b[0], b[2], b[3], b[5], sn, cs, dc[i]);
        bev_corners(b[0], b[2], __fadd_rn(b[3], kMixGrowL), __fadd_rn(b[5], kMixGrowW), sn, cs, ec[i]);
    }
    __syncthreads();
    for (int t = tid; t < ns * rows; t += blockDim.x) {                         // every pair at once
        const int i = t / rows, r = t - i * rows;
        if (sid[i] < 0) continue;
        if (r < g) {
            if (qv[r] && collide(ec[i], qc[r])) atomicOr(&hit[i], 1);
        } else {
            const int k = r - g;
            if (k < i && sid[k] >= 0 && collide(ec[i], dc[k])) atomicOr(&pm[i][k >> 5], 1u << (k & 31));
        }
    }
    __syncthreads();
    if (tid == 0) {
        // the reference's loop: box i is kept iff it collides with no scene row and no box kept before it
        for (int k = 0; k < kMixMaxRows / 32; k++) kept[k] = 0u;
        int r = 0;
        for (int j = 0; j < g; j++)
            if (qv[j]) src[r++] = (short)j;
        for (int i = 0; i < ns; i++) {
            bool ok = sid[i] >= 0 && !hit[i];
            for (int k = 0; k <= (i >> 5) && ok; k++)
                if (pm[i][k] & kept[k]) ok = false;
            keep[i] = ok;
            if (ok) {
                kept[i >> 5] |= 1u << (i & 31);
                src[r++] = (short)(g + i);
            }
        }
        for (; r < rows; r++) src[r] = -1;
    }
    __syncthreads();
    for (int r = tid; r < rows; r += blockDim.x) {
        float *o = out_boxes + ((size_t)s * rows + r) * 7;
        const int q = src[r];
        int lab = 0;
        if (q < 0) {
            for (int k = 0; k < 7; k++) o[k] = 0.0f;
        } else if (q < g) {
            const float *b = boxes + ((size_t)s * g + q) * 7;
            for (int k = 0; k < 7; k++) o[k] = b[k];
            lab = labels[(size_t)s * g + q];
        } else {
            const int id = sid[q - g];
            const float *b = db_boxes + (size_t)id * 7;
            for (int k = 0; k < 7; k++) o[k] = b[k];
            o[1] = (float)__dsub_rn((double)b[1], move_height(b, planes + (size_t)s * 4));
            lab = db_classes[id];
        }
        out_labels[(size_t)s * rows + r] = lab;
    }
    for (int i = tid; i < ns; i += blockDim.x) accepted[(size_t)s * ns + i] = keep[i];
}

__global__ void __launch_bounds__(kMixThreads) mix_paste_points_kernel(
    int ns, const float *__restrict__ pts, const int *__restrict__ offsets, const int *__restrict__ sem, const int *__restrict__ ids,
    const float *__restrict__ db_points, const long long *__restrict__ db_off, const float *__restrict__ db_boxes,
    const int *__restrict__ db_classes, const double *__restrict__ planes, const int *__restrict__ accepted,
    const int *__restrict__ out_off, const int *__restrict__ slot_start, float *__restrict__ out, int *__restrict__ out_sem)
{
    const int s = blockIdx.y, p = blockIdx.x * blockDim.x + threadIdx.x;
    const int q0 = out_off[s], m = out_off[s + 1] - q0;
    if (p >= m) return;
    const int o0 = offsets[s], n = offsets[s + 1] - o0;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    int lab = -1;
    if (p < n) {
        v = reinterpret_cast<const float4 *>(pts)[(size_t)o0 + p];
        lab = sem[(size_t)o0 + p];
    } else {
        const int *st = slot_start + (size_t)s * (ns + 1);                      // st[0] = n, st[ns] = m
        int i = 0;
        while (st[i + 1] <= p) i++;                                             // drawn -1 ids own no slot
        if (accepted[(size_t)s * ns + i]) {
            const int id = ids[(size_t)s * ns + i];
            v = reinterpret_cast<const float4 *>(db_points)[db_off[id] + (p - st[i])];
            v.y = (float)__dsub_rn((double)v.y, move_height(db_boxes + (size_t)id * 7, planes + (size_t)s * 4));
            lab = db_classes[id];
        }
    }
    reinterpret_cast<float4 *>(out)[(size_t)q0 + p] = v;
    out_sem[(size_t)q0 + p] = lab;
}

}  // namespace ssd3d

using namespace ssd3d;

extern "C" int ssd3d_mixup_db_count(int b, int g, int max_n, const float *points, const int *offsets, const float *gt_boxes,
                                    int *counts, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 1 && g >= 1 && g <= kMixMaxRows && max_n >= 1 && max_n <= kMixMaxSlots,
                  "mixup_db_count: bad shape b=%d g=%d max_n=%d (1 <= g <= %d, 1 <= max_n <= %d)", b, g, max_n, kMixMaxRows,
                  kMixMaxSlots);
    SSD3D_REQUIRE(points && offsets && gt_boxes && counts, "mixup_db_count: null pointer");
    const int e = cuda_status(cudaMemsetAsync(counts, 0, (size_t)b * g * sizeof(int), (cudaStream_t)stream), "mixup_db_count memset");
    if (e) return e;
    const dim3 grid(ceil_div(max_n, kMixThreads), b);
    mix_db_count_kernel<<<grid, kMixThreads, 0, (cudaStream_t)stream>>>(g, points, offsets, gt_boxes, counts);
    SSD3D_LAUNCH_CHECK("mix_db_count_kernel");
}

extern "C" int ssd3d_mixup_db_write(int g, int n_objects, const float *points, const int *offsets, const float *gt_boxes,
                                    const int *objects, const long long *object_offsets, float *out_points, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(g >= 1 && g <= kMixMaxRows && n_objects >= 1, "mixup_db_write: bad shape g=%d n_objects=%d", g, n_objects);
    SSD3D_REQUIRE(points && offsets && gt_boxes && objects && object_offsets && out_points, "mixup_db_write: null pointer");
    mix_db_write_kernel<<<n_objects, kMixThreads, 0, (cudaStream_t)stream>>>(g, points, offsets, gt_boxes, objects, object_offsets,
                                                                             out_points);
    SSD3D_LAUNCH_CHECK("mix_db_write_kernel");
}

extern "C" int ssd3d_mixup_paste_boxes(int b, int g, int s, const float *gt_boxes, const int *gt_labels, const int *ids,
                                       const float *db_boxes, const int *db_classes, const double *planes, float *out_boxes,
                                       int *out_labels, int *accepted, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 1 && g >= 0 && s >= 1 && g + s <= kMixMaxRows, "mixup_paste_boxes: bad shape b=%d g=%d s=%d (g + s <= %d)",
                  b, g, s, kMixMaxRows);
    SSD3D_REQUIRE(ids && db_boxes && db_classes && planes && out_boxes && out_labels && accepted && (g == 0 || (gt_boxes && gt_labels)),
                  "mixup_paste_boxes: null pointer");
    mix_paste_boxes_kernel<<<b, kMixThreads, 0, (cudaStream_t)stream>>>(g, s, gt_boxes, gt_labels, ids, db_boxes, db_classes, planes,
                                                                        out_boxes, out_labels, accepted);
    SSD3D_LAUNCH_CHECK("mix_paste_boxes_kernel");
}

extern "C" int ssd3d_mixup_paste_points(int b, int s, int max_slots, const float *points, const int *offsets, const int *sem_labels,
                                        const int *ids, const float *db_points, const long long *db_offsets, const float *db_boxes,
                                        const int *db_classes, const double *planes, const int *accepted, const int *out_offsets,
                                        const int *slot_start, float *out_points, int *out_sem_labels, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 1 && s >= 1 && s <= kMixMaxRows && max_slots >= 1 && max_slots <= kMixMaxSlots,
                  "mixup_paste_points: bad shape b=%d s=%d max_slots=%d (s <= %d, 1 <= max_slots <= %d)", b, s, max_slots, kMixMaxRows,
                  kMixMaxSlots);
    SSD3D_REQUIRE(points && offsets && sem_labels && ids && db_points && db_offsets && db_boxes && db_classes && planes && accepted &&
                  out_offsets && slot_start && out_points && out_sem_labels, "mixup_paste_points: null pointer");
    const dim3 grid(ceil_div(max_slots, kMixThreads), b);
    mix_paste_points_kernel<<<grid, kMixThreads, 0, (cudaStream_t)stream>>>(s, points, offsets, sem_labels, ids, db_points, db_offsets,
                                                                            db_boxes, db_classes, planes, accepted, out_offsets,
                                                                            slot_start, out_points, out_sem_labels);
    SSD3D_LAUNCH_CHECK("mix_paste_points_kernel");
}
