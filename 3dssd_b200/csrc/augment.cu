// augment.cu -- the training-scene augmentation of 3dssd.yaml after the mixup paste (DESIGN.md section 3.12):
// DataAugmentor.kitti_forward (lib/builder/data_augmentor.py:62-100) followed by the 16384-point choice of
// kitti_dataloader.py:137-147, on ragged scenes.
//   aug_sem_labels  the semantic label of every point when the sample has none (kitti_dataloader.py:211-219)
//   aug_boxes       one CTA per scene: flip, the per-object noise search (voxelnet_aug.py:402-438, one thread per try),
//                   the box transforms, global rotation and scale; the membership planes go to a workspace
//   aug_points      one thread per point: flip, noise move, global transform, context filter, sort key
//   aug_choose      one CTA per scene: radix-select the num_points smallest keys, sort them, gather, refill
// Every random number comes from the caller's draw block; there are no float atomics, and integer atomics only count,
// so the same draws give the same bits on every run.
#include <math.h>

#include "box_geom.cuh"

namespace ssd3d {

constexpr int kAugTries = 100;                 // num_try of noise_per_object_v3_
constexpr int kAugMaxBoxes = 256;
constexpr int kAugMaxPoints = 131072;          // per scene
constexpr int kAugMaxChoose = 16384;           // the sorted choice lives in shared memory
constexpr int kAugBoxThreads = 128;
constexpr int kAugPointThreads = 256;
constexpr int kAugChooseThreads = 1024;
constexpr float kAugExpand = 0.1f;             // EXPAND_DIMS_LENGTH
constexpr double kRotPerturb = M_PI / 3.0;     // SINGLE_AUG.ROTATION_PERTURB = [-pi/3, pi/3]
constexpr double kGlobalRot = M_PI / 4.0;      // RANDOM_ROTATION_RANGE = 45 / 180 * pi
constexpr double kGlobalScale = 0.1;           // RANDOM_SCALE_RANGE
constexpr float kGrowL = 0.5f, kGrowH = 2.0f, kGrowW = 0.5f;   // filter_points_boxes_3d enlarge_range (l, h, w)

struct AugScene {
    int flip, noise, grot, gscale;
    double gs, gc;          // sin, cos of the global angle
    double pscale;          // the factor the points are multiplied by in double
    float angle, scale;     // the angle and factor as the float32 boxes take them
};

struct AugBox {
    Planes pre;             // pre-noise box grown by 0.1: which points move with it
    Planes fin;             // final box grown by (0.5, 2, 0.5): the context filter
    float cx, cy, cz;       // pre-noise centre
    float sr, cr;           // sin, cos of the chosen rotation, float32
    int valid, ok;          // not a padded row; its noise search succeeded
    double lx, lz;          // the chosen translation
};

// np.random.uniform(-pi/3, pi/3) from its uniform draw: low + (high - low) * u
__device__ __forceinline__ double rot_of(double u) { return __dadd_rn(-kRotPerturb, __dmul_rn(2.0 * kRotPerturb, u)); }

__global__ void __launch_bounds__(kAugBoxThreads) aug_boxes_kernel(
    int g, const float *__restrict__ boxes, const double *__restrict__ scene_u, const double *__restrict__ loc_noise,
    const double *__restrict__ rot_u, float *__restrict__ out_boxes, int *__restrict__ chosen, AugScene *__restrict__ ws_scene,
    AugBox *__restrict__ ws_box)
{
    __shared__ float sb[kAugMaxBoxes][7];
    __shared__ float sc[kAugMaxBoxes][4][2];        // current BEV corners (x, z) of the 0.1-grown boxes
    __shared__ unsigned char sv[kAugMaxBoxes];
    __shared__ int stry[kAugMaxBoxes];
    __shared__ unsigned wmask[kAugBoxThreads / 32];
    const int s = blockIdx.x, tid = threadIdx.x;
    const double *u = scene_u + (size_t)s * 6;
    const bool flip = u[0] >= 0.5, noise = u[1] <= 0.5, grot = u[2] <= 0.5, gscale = u[3] <= 0.5;
    const float pi32 = (float)M_PI;
    for (int j = tid; j < g; j += blockDim.x) {
        const float *b = boxes + ((size_t)s * g + j) * 7;
        const bool v = box_is_valid(b);
        for (int k = 0; k < 7; k++) sb[j][k] = b[k];
        if (v && flip) {                                                        // flip_boxes_3d (kitti_aug.py:48-72)
            sb[j][0] = -sb[j][0];
            sb[j][6] = sb[j][6] >= 0.0f ? __fsub_rn(pi32, sb[j][6]) : __fsub_rn(-pi32, sb[j][6]);
        }
        sv[j] = v;
        stry[j] = -1;
        if (noise && v) {                                                       // the corners of the grown box
            float sn, cs;
            sincos32((double)sb[j][6], sn, cs);
            bev_corners(sb[j][0], sb[j][2], __fadd_rn(sb[j][3], kAugExpand), __fadd_rn(sb[j][5], kAugExpand), sn, cs, sc[j]);
        }
    }
    __syncthreads();
    if (noise) {
        // noise_per_box (voxelnet_aug.py:402-438): box i takes its first try that collides with no other box's current
        // corners; try j runs on thread j, and the lowest successful thread is the sequential loop's first success
        for (int i = 0; i < g; i++) {
            if (!sv[i]) continue;
            bool ok = false;
            float cand[4][2];
            if (tid < kAugTries) {
                const size_t t = ((size_t)s * g + i) * kAugTries + tid;
                float sr, cr;
                sincos32(rot_of(rot_u[t]), sr, cr);
                const double tx = __dadd_rn((double)sb[i][0], loc_noise[t * 2]), tz = __dadd_rn((double)sb[i][2], loc_noise[t * 2 + 1]);
                for (int k = 0; k < 4; k++) {
                    const float r0 = __fsub_rn(sc[i][k][0], sb[i][0]), r1 = __fsub_rn(sc[i][k][1], sb[i][2]);
                    const float q0 = __fadd_rn(__fmul_rn(r0, cr), __fmul_rn(r1, sr));
                    const float q1 = __fsub_rn(__fmul_rn(r1, cr), __fmul_rn(r0, sr));
                    cand[k][0] = (float)__dadd_rn((double)q0, tx);
                    cand[k][1] = (float)__dadd_rn((double)q1, tz);
                }
                ok = true;
                for (int k = 0; k < g && ok; k++)
                    if (k != i && sv[k] && collide(cand, sc[k])) ok = false;
            }
            const unsigned m = __ballot_sync(0xffffffffu, ok);
            if ((tid & 31) == 0) wmask[tid >> 5] = m;
            __syncthreads();
            int first = -1;
            for (int w = 0; w < kAugBoxThreads / 32 && first < 0; w++)
                if (wmask[w]) first = w * 32 + __ffs(wmask[w]) - 1;
            if (tid == first) {
                for (int k = 0; k < 4; k++) { sc[i][k][0] = cand[k][0]; sc[i][k][1] = cand[k][1]; }
                stry[i] = first;
            }
            __syncthreads();
        }
    }
    double gs = 0.0, gc = 1.0, pscale = 1.0;
    float angle = 0.0f, scale = 1.0f;
    if (grot) {
        const double a = __dmul_rn(__dsub_rn(__dmul_rn(u[4], 2.0), 1.0), kGlobalRot);
        eval_sincos(a, gs, gc);
        angle = (float)a;
    }
    if (gscale) {
        const double f = __dadd_rn(__dmul_rn(__dsub_rn(__dmul_rn(u[5], 2.0), 1.0), kGlobalScale), 1.0);
        scale = (float)f;
        pscale = grot ? f : (double)scale;           // float32 points take the factor as float32 (data_augmentor.py:94)
    }
    if (tid == 0) ws_scene[s] = AugScene{flip, noise, grot, gscale, gs, gc, pscale, angle, scale};
    for (int j = tid; j < g; j += blockDim.x) {
        AugBox &W = ws_box[(size_t)s * g + j];
        float *o = out_boxes + ((size_t)s * g + j) * 7;
        chosen[(size_t)s * g + j] = stry[j];
        W.valid = sv[j];
        W.ok = stry[j] >= 0;
        if (!sv[j]) {
            for (int k = 0; k < 7; k++) o[k] = 0.0f;                            // padded rows take part in nothing
            continue;
        }
        float b[7];
        for (int k = 0; k < 7; k++) b[k] = sb[j][k];
        float sn, cs;
        sincos32((double)b[6], sn, cs);
        box_planes(b, kAugExpand, sn, cs, W.pre);
        W.cx = b[0]; W.cy = b[1]; W.cz = b[2];
        W.sr = 0.0f; W.cr = 1.0f; W.lx = 0.0; W.lz = 0.0;
        if (W.ok) {                                                             // box3d_transform_ (voxelnet_aug.py:735-742)
            const size_t t = ((size_t)s * g + j) * kAugTries + stry[j];
            const double rot = rot_of(rot_u[t]);
            sincos32(rot, W.sr, W.cr);
            W.lx = loc_noise[t * 2];
            W.lz = loc_noise[t * 2 + 1];
            b[0] = (float)__dadd_rn((double)b[0], W.lx);
            b[2] = (float)__dadd_rn((double)b[2], W.lz);
            b[6] = (float)__dadd_rn((double)b[6], rot);
        }
        if (grot) {                                                             // roty (rotation_util.py:74-80), double
            const double x = b[0], z = b[2];
            b[0] = (float)__dadd_rn(__dmul_rn(gc, x), __dmul_rn(gs, z));
            b[2] = (float)__dsub_rn(__dmul_rn(gc, z), __dmul_rn(gs, x));
            b[6] = __fadd_rn(b[6], angle);
        }
        if (gscale)
            for (int k = 0; k < 6; k++) b[k] = __fmul_rn(b[k], scale);
        // filter_points_boxes_3d grows the dims in place, tests, and shrinks them back: rn(rn(d + e) - e) stays
        b[3] = __fadd_rn(b[3], kGrowL); b[4] = __fadd_rn(b[4], kGrowH); b[5] = __fadd_rn(b[5], kGrowW);
        sincos32((double)b[6], sn, cs);
        box_planes(b, 0.0f, sn, cs, W.fin);
        b[3] = __fsub_rn(b[3], kGrowL); b[4] = __fsub_rn(b[4], kGrowH); b[5] = __fsub_rn(b[5], kGrowW);
        for (int k = 0; k < 7; k++) o[k] = b[k];
    }
}

__global__ void __launch_bounds__(kAugPointThreads) aug_points_kernel(
    int g, const float *__restrict__ pts, const int *__restrict__ offsets, const int *__restrict__ sem,
    const unsigned *__restrict__ keys, const AugScene *__restrict__ ws_scene, const AugBox *__restrict__ ws_box,
    float *__restrict__ out, unsigned long long *__restrict__ sort_keys, int *__restrict__ survivors, int *__restrict__ moved)
{
    const int s = blockIdx.y, p = blockIdx.x * blockDim.x + threadIdx.x;
    const int o0 = offsets[s], n = offsets[s + 1] - o0;
    if (p >= n) return;
    const size_t gi = (size_t)o0 + p;
    const AugScene S = ws_scene[s];
    const AugBox *W = ws_box + (size_t)s * g;
    float x = pts[gi * 4], y = pts[gi * 4 + 1], z = pts[gi * 4 + 2];
    const float in = pts[gi * 4 + 3];
    const int lab = sem[gi];
    if (lab < 0) {                                                              // an absent slot of the mixup layout
        out[gi * 4] = 0.0f; out[gi * 4 + 1] = 0.0f; out[gi * 4 + 2] = 0.0f; out[gi * 4 + 3] = 0.0f;
        if (moved) moved[gi] = -1;
        sort_keys[gi] = ~0ull;
        return;
    }
    if (S.flip) x = -x;                                                      // flip_points (kitti_aug.py:14-19)
    int mover = -1;
    if (S.noise && lab != 0) {
        // points_transform_ (voxelnet_aug.py:590-618): the first pre-noise box holding the point moves it
        for (int j = 0; j < g; j++) {
            if (!W[j].valid || !inside(W[j].pre, x, z, y)) continue;
            if (W[j].ok) {
                mover = j;
                const float p0 = __fsub_rn(x, W[j].cx), p1 = __fsub_rn(z, W[j].cz), p2 = __fsub_rn(y, W[j].cy);
                const float q0 = __fadd_rn(__fmul_rn(p0, W[j].cr), __fmul_rn(p1, W[j].sr));
                const float q1 = __fsub_rn(__fmul_rn(p1, W[j].cr), __fmul_rn(p0, W[j].sr));
                x = (float)__dadd_rn((double)__fadd_rn(q0, W[j].cx), W[j].lx);
                z = (float)__dadd_rn((double)__fadd_rn(q1, W[j].cz), W[j].lz);
                y = __fadd_rn(p2, W[j].cy);
            }
            break;
        }
    }
    double X = x, Y = y, Z = z;
    if (S.grot) {
        const double x0 = X;
        X = __dadd_rn(__dmul_rn(S.gc, x0), __dmul_rn(S.gs, Z));
        Z = __dsub_rn(__dmul_rn(S.gc, Z), __dmul_rn(S.gs, x0));
    }
    if (S.gscale) { X = __dmul_rn(X, S.pscale); Y = __dmul_rn(Y, S.pscale); Z = __dmul_rn(Z, S.pscale); }
    x = (float)X; y = (float)Y; z = (float)Z;
    bool keep = true;
    if (lab == 0)                                                               // filter_points_boxes_3d (voxelnet_aug.py:345-372)
        for (int j = 0; j < g && keep; j++)
            if (W[j].valid && inside(W[j].fin, x, z, y)) keep = false;
    out[gi * 4] = x; out[gi * 4 + 1] = y; out[gi * 4 + 2] = z; out[gi * 4 + 3] = in;
    if (moved) moved[gi] = mover;
    sort_keys[gi] = keep ? ((unsigned long long)keys[gi] << 32 | (unsigned)p) : ~0ull;
    if (keep) atomicAdd(survivors + s, 1);
}

__global__ void __launch_bounds__(kAugChooseThreads) aug_choose_kernel(
    int m, const float *__restrict__ pts, const int *__restrict__ offsets, const unsigned long long *__restrict__ sort_keys,
    const int *__restrict__ survivors, const unsigned *__restrict__ refill, float *__restrict__ out)
{
    extern __shared__ unsigned long long buf[];                                 // [pow2 >= min(N, m)]
    __shared__ unsigned hist[256];
    __shared__ unsigned long long s_prefix;
    __shared__ unsigned s_rem, s_fill;
    const int s = blockIdx.x, tid = threadIdx.x;
    const int o0 = offsets[s], n = offsets[s + 1] - o0, N = survivors[s];
    const int K = min(N, m);
    const unsigned long long *key = sort_keys + o0;
    unsigned long long thr = ~0ull - 1;                                         // every survivor when N <= m
    if (N > m) {
        // radix select of the K-th smallest key, 8 bits at a time from the top; the keys are distinct
        unsigned long long prefix = 0, mask = 0;
        if (tid == 0) s_rem = K;
        for (int shift = 56; shift >= 0; shift -= 8) {
            for (int d = tid; d < 256; d += blockDim.x) hist[d] = 0;
            __syncthreads();
            for (int p = tid; p < n; p += blockDim.x) {
                const unsigned long long v = key[p];
                if ((v & mask) == prefix) atomicAdd(&hist[(v >> shift) & 255], 1u);
            }
            __syncthreads();
            if (tid == 0) {
                unsigned cum = 0, d = 0;
                while (cum + hist[d] < s_rem) cum += hist[d++];
                s_rem -= cum;
                s_prefix = prefix | ((unsigned long long)d << shift);
            }
            __syncthreads();
            prefix = s_prefix;
            mask |= 255ull << shift;
        }
        thr = prefix;
    }
    int P = 1;
    while (P < K) P <<= 1;
    if (tid == 0) s_fill = 0;
    for (int i = tid; i < P; i += blockDim.x) buf[i] = ~0ull;
    __syncthreads();
    for (int p = tid; p < n; p += blockDim.x) {
        const unsigned long long v = key[p];
        if (v <= thr) buf[atomicAdd(&s_fill, 1u)] = v;
    }
    for (int k = 2; k <= P; k <<= 1)                                            // bitonic sort, ascending
        for (int j = k >> 1; j > 0; j >>= 1) {
            __syncthreads();
            for (int i = tid; i < P; i += blockDim.x) {
                const int l = i ^ j;
                if (l > i) {
                    const unsigned long long a = buf[i], b = buf[l];
                    if (((i & k) == 0) == (a > b)) { buf[i] = b; buf[l] = a; }
                }
            }
        }
    __syncthreads();
    for (int t = tid; t < m; t += blockDim.x) {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (N > 0) {
            const int r = t < K ? t : (int)(((unsigned long long)refill[(size_t)s * m + t] * (unsigned)N) >> 32);
            const unsigned idx = (unsigned)(buf[r] & 0xffffffffu);
            v = reinterpret_cast<const float4 *>(pts)[(size_t)o0 + idx];
        }
        reinterpret_cast<float4 *>(out)[(size_t)s * m + t] = v;
    }
}

__global__ void __launch_bounds__(kAugPointThreads) aug_sem_labels_kernel(
    int g, const float *__restrict__ pts, const int *__restrict__ offsets, const float *__restrict__ boxes,
    const int *__restrict__ labels, int *__restrict__ sem)
{
    __shared__ Planes sp[kAugMaxBoxes];
    __shared__ unsigned char sv[kAugMaxBoxes];
    const int s = blockIdx.y, p = blockIdx.x * blockDim.x + threadIdx.x;
    const int o0 = offsets[s], n = offsets[s + 1] - o0;
    if (blockIdx.x * blockDim.x >= n) return;                                   // the whole CTA
    for (int j = threadIdx.x; j < g; j += blockDim.x) {
        const float *b = boxes + ((size_t)s * g + j) * 7;
        sv[j] = box_is_valid(b);
        if (sv[j]) {
            float sn, cs;
            sincos32((double)b[6], sn, cs);
            box_planes(b, kAugExpand, sn, cs, sp[j]);
        }
    }
    __syncthreads();
    if (p >= n) return;
    const size_t gi = (size_t)o0 + p;
    const float x = pts[gi * 4], y = pts[gi * 4 + 1], z = pts[gi * 4 + 2];
    int lab = 0;
    for (int j = 0; j < g; j++)
        if (sv[j] && inside(sp[j], x, z, y)) { lab = labels[(size_t)s * g + j]; break; }
    sem[gi] = lab;
}

static size_t aug_scene_bytes(int b) { return ((size_t)b * sizeof(AugScene) + 255) & ~(size_t)255; }

static int aug_shape(int b, int g, int max_n, const char *what)
{
    SSD3D_REQUIRE(b >= 1 && g >= 0 && g <= kAugMaxBoxes && max_n >= 1 && max_n <= kAugMaxPoints,
                  "%s: bad shape b=%d g=%d max_n=%d (g <= %d, 1 <= max_n <= %d)", what, b, g, max_n, kAugMaxBoxes, kAugMaxPoints);
    return 0;
}

}  // namespace ssd3d

using namespace ssd3d;

extern "C" size_t ssd3d_augment_workspace(int b, int g)
{
    if (b < 1 || g < 0) return 0;
    return aug_scene_bytes(b) + (size_t)b * g * sizeof(AugBox);
}

extern "C" int ssd3d_augment_sem_labels(int b, int g, int max_n, const float *points, const int *offsets, const float *gt_boxes,
                                        const int *gt_labels, int *sem_labels, ssd3d_stream_t stream)
{
    const int st = aug_shape(b, g, max_n, "augment_sem_labels");
    if (st) return st;
    SSD3D_REQUIRE(points && offsets && sem_labels && (g == 0 || (gt_boxes && gt_labels)), "augment_sem_labels: null pointer");
    const dim3 grid(ceil_div(max_n, kAugPointThreads), b);
    aug_sem_labels_kernel<<<grid, kAugPointThreads, 0, (cudaStream_t)stream>>>(g, points, offsets, gt_boxes, gt_labels, sem_labels);
    SSD3D_LAUNCH_CHECK("aug_sem_labels_kernel");
}

extern "C" int ssd3d_augment_boxes(int b, int g, const float *gt_boxes, const double *scene_u, const double *loc_noise,
                                   const double *rot_u, float *out_boxes, int *chosen_try, void *workspace, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 1 && g >= 0 && g <= kAugMaxBoxes, "augment_boxes: bad shape b=%d g=%d (g <= %d)", b, g, kAugMaxBoxes);
    SSD3D_REQUIRE(scene_u && workspace && (g == 0 || (gt_boxes && loc_noise && rot_u && out_boxes && chosen_try)),
                  "augment_boxes: null pointer");
    char *ws = (char *)workspace;
    aug_boxes_kernel<<<b, kAugBoxThreads, 0, (cudaStream_t)stream>>>(g, gt_boxes, scene_u, loc_noise, rot_u, out_boxes, chosen_try,
                                                                     (AugScene *)ws, (AugBox *)(ws + aug_scene_bytes(b)));
    SSD3D_LAUNCH_CHECK("aug_boxes_kernel");
}

extern "C" int ssd3d_augment_points(int b, int g, int max_n, const float *points, const int *offsets, const int *sem_labels,
                                    const unsigned *keys, const void *workspace, float *out_points,
                                    unsigned long long *sort_keys, int *survivors, int *moved_by, ssd3d_stream_t stream)
{
    const int st = aug_shape(b, g, max_n, "augment_points");
    if (st) return st;
    SSD3D_REQUIRE(points && offsets && sem_labels && keys && workspace && out_points && sort_keys && survivors,
                  "augment_points: null pointer");
    const int e = cuda_status(cudaMemsetAsync(survivors, 0, (size_t)b * sizeof(int), (cudaStream_t)stream), "augment_points memset");
    if (e) return e;
    const char *ws = (const char *)workspace;
    const dim3 grid(ceil_div(max_n, kAugPointThreads), b);
    aug_points_kernel<<<grid, kAugPointThreads, 0, (cudaStream_t)stream>>>(
        g, points, offsets, sem_labels, keys, (const AugScene *)ws, (const AugBox *)(ws + aug_scene_bytes(b)), out_points, sort_keys,
        survivors, moved_by);
    SSD3D_LAUNCH_CHECK("aug_points_kernel");
}

extern "C" int ssd3d_augment_choose(int b, int num_points, const float *points, const int *offsets,
                                    const unsigned long long *sort_keys, const int *survivors, const unsigned *refill,
                                    float *out, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 1 && num_points >= 1 && num_points <= kAugMaxChoose, "augment_choose: bad shape b=%d num_points=%d (<= %d)",
                  b, num_points, kAugMaxChoose);
    SSD3D_REQUIRE(points && offsets && sort_keys && survivors && refill && out, "augment_choose: null pointer");
    int pow2 = 1;
    while (pow2 < num_points) pow2 <<= 1;
    const size_t smem = (size_t)pow2 * sizeof(unsigned long long);
    const int e = cuda_status(cudaFuncSetAttribute(aug_choose_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                              "aug_choose_kernel attribute");
    if (e) return e;
    aug_choose_kernel<<<b, kAugChooseThreads, smem, (cudaStream_t)stream>>>(num_points, points, offsets, sort_keys, survivors, refill,
                                                                            out);
    SSD3D_LAUNCH_CHECK("aug_choose_kernel");
}
