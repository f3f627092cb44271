// fps_plan.h -- which FPS kernel a call runs: the selection rule of the farthest-point-sampling entry points, stated
// once.  The launchers (fps.cu) run what the plan says and the query entry points read the same plan, so a query
// cannot drift from the launch it describes.  Plain C++17 without CUDA, so the rule builds and is tested on any host.
#pragma once
#include <cstddef>

namespace ssd3d {

constexpr int FPS_T = 256;                      // threads per CTA of the cluster kernels
constexpr int FPS_NW = FPS_T / 32;
constexpr size_t FPS_SMEM_BUDGET = 200 * 1024;  // dynamic shared memory a cluster kernel may plan for
constexpr int FB_MAXN = 16384;                  // points the single-CTA pruned kernel holds (fps_bucket.cu)

enum class FpsKind {
    Bucket,          // fps3_bucket_kernel: one CTA per scene with spatial pruning (c == 3)
    Direct,          // fps3_direct_kernel<CL,P>: scene resident in every CTA (c == 3)
    Packet,          // fps3_cluster_kernel<CL,P>: coordinates travel in the packets (c == 3)
    Generic,         // fpsc_cluster_kernel<CL,P>: any c, features in the cluster's shared memory
    Dist,            // fpsdist_cluster_kernel<CL,P>: given distance matrix
    Features,        // ffps_cluster_kernel<CL,P,CP>: matrix-free F-FPS
    FeaturesBucket,  // ffps_bucket_kernel: matrix-free F-FPS on 4 CTAs with bucket pruning
    Fallback,        // no on-chip kernel: fps_fallback_kernel with temp[b,n]; for features, SSD3D_ERR_UNSUPPORTED
};

struct FpsPlan {
    FpsKind kind = FpsKind::Fallback;
    int cl = 0, p = 0, cp = 0;  // CTAs per scene, points per thread, padded channels (Features, FeaturesBucket)
    size_t smem = 0;            // dynamic shared memory per CTA, bytes
    long temp = 0;              // floats of temp per scene the call uses (0: temp may be NULL)
    bool rounds = false;        // the route runs a partial range of rounds
};

// smallest power of two P >= need with P >= residue classes per thread
static inline int pick_p(int n, int cl)
{
    const int tt = cl * FPS_T;
    const int r = tt >= 1024 ? 1 : 1024 / tt;
    // a residue class holds ceil(n/1024) points; slots per class J = P/R must cover them
    const int per_class = (n + 1023) / 1024;
    const int s = tt >= 1024 ? tt / 1024 : 1;
    const int need = r * ((per_class + s - 1) / s);
    int p = r;
    while (p < need) p *= 2;
    return p;
}

// the smallest cluster from `cl` up to 16 whose threads hold n points at P <= 16
static inline int grow_cl(int n, int cl)
{
    while (cl < 16 && pick_p(n, cl) > 16) cl *= 2;
    return cl;
}

// Cluster-size request of one call (the `cluster` argument of the *_ex entry points): 0 = heuristic, > 0 = exactly
// that many CTAs per scene, < 0 = heuristic capped at -cluster (throughput mode: FPS is latency-bound, so fewer SMs
// per scene cost little time and free SMs for work running concurrently).
static inline int cap_cl(int cl, int n, int hint)
{
    if (hint < 0)
        while (cl > -hint && cl > 1 && (n + (cl / 2) * FPS_T - 1) / ((cl / 2) * FPS_T) <= 16) cl /= 2;
    return cl;
}

static inline int pick_cl_xyz(int n, int hint)
{
    if (hint > 0) return hint;
    int cl;
    if (n <= 1024) cl = 1;
    else if (n <= 2048) cl = 2;
    else if (n <= 4096) cl = 4;
    else if (n <= 32768) cl = 8;
    else cl = 16;
    return cap_cl(cl, n, hint);
}

static inline size_t fps3_direct_smem(int n) { return (size_t)n * 12 + 16; }
static inline size_t fps3_packet_smem(int p) { return (size_t)p * FPS_T * 16; }
static inline size_t fpsc_smem(int c, int p) { return ((size_t)c * (p * FPS_T + 1) + c) * sizeof(float) + 16; }
static inline size_t ffps_smem(int cl, int p, int cp) { return (size_t)p * FPS_T * cp * 4 + (size_t)p * FPS_T * 4 + (size_t)2 * cl * (16 + 4 * cp); }
constexpr size_t FB_SMEM = (size_t)3 * FB_MAXN * sizeof(float);

// cluster size for the generic-c kernel: smallest CL whose per-CTA feature slab fits in shared memory
static inline int pick_cl_generic(int n, int c, int hint)
{
    if (hint > 0) return hint;
    for (int cl = 1; cl <= 16; cl *= 2) {
        const int p = pick_p(n, cl);
        if (p <= 16 && fpsc_smem(c, p) <= FPS_SMEM_BUDGET && (cl >= 8 || n <= cl * 1024)) return cl;
    }
    for (int cl = 1; cl <= 16; cl *= 2) {
        const int p = pick_p(n, cl);
        if (p <= 16 && fpsc_smem(c, p) <= FPS_SMEM_BUDGET) return cl;
    }
    return 0;
}

// (c == 3) does the resumable direct kernel cover n?  It needs the scene resident in one CTA's shared memory, and the
// bulk copy that loads it a 16-byte aligned source and size.
static inline bool fps3_direct_fits(int n, int cl, bool aligned, long long sa)
{
    return cl >= 2 && fps3_direct_smem(n) <= FPS_SMEM_BUDGET && (n % 4) == 0 && aligned && (sa % 4) == 0 &&
           pick_p(n, cl) <= 16;
}

static inline bool fps3_bucket_applies(int n, int m, int flags)
{
    if (flags & 2) return false;                                   // caller forbids it (tests, experiments)
    if (n > FB_MAXN || n < 64 || m < 2) return false;
    if (flags & 4) return true;                                    // caller forces it (tests: any n in range)
    return n > 8192 && m >= 256;
}

// matrix-free F-FPS: CP = 68 (P = 2 points per thread) or 132 (P = 1); smallest cluster that holds n
static inline int ffps_cluster_for(int n, int c)
{
    const int per_cta = c <= 68 ? 2 * FPS_T : (c <= 132 ? FPS_T : 0);
    if (per_cta == 0) return 0;
    for (int cl = 1; cl <= 8; cl *= 2)
        if (n <= cl * per_cta) return cl;
    return 0;
}

// ssd3d_farthest_point_sample_ex: inp[b,n,c] with scene stride sa; `aligned` = inp is 16-byte aligned
static inline FpsPlan plan_fps(int n, int c, int m, int cluster, int flags, bool aligned, long long sa, bool partial)
{
    FpsPlan pl;
    if (c == 3 && fps3_bucket_applies(n, m, flags)) {
        // large scenes: one CTA per scene with spatial pruning; `cluster` does not apply
        pl.kind = FpsKind::Bucket, pl.cl = 1, pl.smem = FB_SMEM, pl.rounds = true;
    } else if (c == 3) {
        const int cl = grow_cl(n, pick_cl_xyz(n, cluster)), p = pick_p(n, cl);
        if ((flags & 1) == 0 && fps3_direct_fits(n, cl, aligned, sa))
            pl.kind = FpsKind::Direct, pl.cl = cl, pl.p = p, pl.smem = fps3_direct_smem(n), pl.rounds = true;
        else if (p <= 16)
            pl.kind = FpsKind::Packet, pl.cl = cl, pl.p = p, pl.smem = fps3_packet_smem(p);
    } else {
        const int cl = pick_cl_generic(n, c, cluster), p = cl > 0 ? pick_p(n, cl) : 0;
        if (cl > 0 && p <= 16) pl.kind = FpsKind::Generic, pl.cl = cl, pl.p = p, pl.smem = fpsc_smem(c, p);
    }
    // a partial range carries the running distances (bucket kernel: + its point permutation); the fallback keeps its
    // distances there anyway
    if (partial) pl.temp = pl.kind == FpsKind::Bucket ? 2L * n : n;
    else if (pl.kind == FpsKind::Fallback) pl.temp = n;
    return pl;
}

// ssd3d_farthest_point_sample_with_distance_ex: the per-round row read is a DRAM-latency-bound gather, so more CTAs
// per scene (more loads in flight) than for xyz
static inline FpsPlan plan_fps_dist(int n, int cluster)
{
    FpsPlan pl;
    const int cl = grow_cl(n, cluster > 0 ? cluster : cap_cl(n <= 1024 ? 1 : (n <= 2048 ? 4 : 8), n, cluster));
    const int p = pick_p(n, cl);
    if (p <= 16) pl.kind = FpsKind::Dist, pl.cl = cl, pl.p = p;
    else pl.temp = n;
    return pl;
}

// ffps_bucket_kernel (fps_bucket.cu): 4 CTAs per scene, 4 points of 68 channels per thread, bucket pruning
constexpr int FFB_CL = 4;
constexpr int FFB_MAXN = FFB_CL * FPS_T * 4;
// rows of slots 2-3, sort keys, bucket centres, per-warp staged rows of both parities, packets
constexpr size_t ffps_bucket_smem() { return (size_t)2 * FPS_T * 68 * 4 + (size_t)FFB_MAXN * 8 + 8 * 4 * 72 * 4 + 2 * 8 * 72 * 4 + 2 * FFB_CL * 288; }

// ssd3d_farthest_point_sample_features_cl: c = channels of the concatenated feature, `cluster` = 0 or a cap (< 0).  A
// full-range call whose cap is below the 8 CTAs that 2048 < n <= 4096 at 3 <= c <= 68 needs runs ffps_bucket_kernel
// on 4 CTAs -- the fewest that hold such a scene on chip; its partial ranges stay on ffps_cluster_kernel.
static inline FpsPlan plan_ffps(int n, int c, int cluster, bool partial)
{
    FpsPlan pl;
    const int cl = n > 0 && c > 0 ? ffps_cluster_for(n, c) : 0;
    if (cl > FFB_CL && cluster < 0 && -cluster < cl && !partial && c >= 3 && c <= 68 && n <= FFB_MAXN) {
        pl.kind = FpsKind::FeaturesBucket, pl.cl = FFB_CL, pl.p = 4, pl.cp = 68, pl.smem = ffps_bucket_smem();
    } else if (cl > 0) {
        pl.kind = FpsKind::Features, pl.cl = cl, pl.p = c <= 68 ? 2 : 1, pl.cp = c <= 68 ? 68 : 132;
        pl.smem = ffps_smem(cl, pl.p, pl.cp), pl.rounds = true;
    }
    if (partial) pl.temp = n;
    return pl;
}

}  // namespace ssd3d
