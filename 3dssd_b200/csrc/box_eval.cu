// box_eval.cu -- the KITTI evaluator on the GPU: rotated BEV / 3-D box overlaps, the reference's 41-point precision
// passes, and the calc_iou / calc_iou_match operators built on the same overlaps (DESIGN.md section 3.10).
//
// Replaces the reference's Evaluate op (lib/utils/tf_ops/evaluation/tf_evaluate.cpp:14-33,75-139, eval() at
// evaluate.cpp:1229), which runs on the CPU and recomputes a Boost polygon intersection for every (label, detection) pair
// once per score threshold, difficulty and metric (evaluate.cpp:649-830, :835-928).  Here the overlaps of a pair are
// computed once (eval_overlap_kernel), the first pass of computeStatistics runs one thread per (frame, class,
// difficulty, metric) (eval_first_pass_kernel) and the counting pass one thread per (frame, class, difficulty, metric,
// threshold) (eval_count_kernel), its tp / fp / fn reduced with integer atomics, so the totals do not depend on the
// order the threads finish in.  getThresholds and the precision curve run on the host between and after the passes.
//
// Arithmetic recipe (shared with the C twin of the test suite, which gives the same bits): every double operation
// through an _rn intrinsic, which nvcc never contracts into a DFMA (the library is built with -fmad=true); cos / sin by
// one recipe (Cody-Waite reduction by pi/2, fdlibm's minimax polynomials with explicit fma), because CUDA's sincos and
// glibc's differ in the last bit on some inputs; corners rn(rn(rn(c*a) + rn(s*b)) + t) from |l|/2 and |w|/2;
// Sutherland-Hodgman clipping of the detection rectangle by the label rectangle, then a shoelace area in vertex order.
#include "box_geom.cuh"

namespace ssd3d {

constexpr int EVAL_THREADS = 256;
constexpr int EVAL_MAX_DETS = 1024;      // per frame
constexpr int EVAL_MAX_LABELS = 256;     // per frame
constexpr int EVAL_CASES = 27;           // metric * 9 + class * 3 + difficulty
constexpr int EVAL_NSAMPLE = 41;         // N_SAMPLE_PTS (evaluate.cpp:55)
constexpr int CLIP_MAXV = 16;

enum { T_CAR = 0, T_PED = 1, T_CYC = 2, T_VAN = 3, T_SIT = 4, T_DONTCARE = 5 };

// ---- rotated rectangles --------------------------------------------------------------------------------------------
// Corners as toPolygon builds them (evaluate.cpp:461-485): (l/2, w/2), (l/2, -w/2), (-l/2, -w/2), (-l/2, w/2) turned by
// [[cos, sin], [-sin, cos]] and offset by (t1, t3) -- a clockwise polygon in the (x, z) plane.
__device__ __forceinline__ void rect_corners(double t1, double t3, double l, double w, double ry, double *px, double *pz)
{
    double s, c;
    eval_sincos(ry, s, c);
    const double a = __dmul_rn(fabs(l), 0.5), b = __dmul_rn(fabs(w), 0.5);
#pragma unroll
    for (int k = 0; k < 4; k++) {
        const double u = k < 2 ? a : -a, v = (k == 0 || k == 3) ? b : -b;
        px[k] = __dadd_rn(__dadd_rn(__dmul_rn(c, u), __dmul_rn(s, v)), t1);
        pz[k] = __dadd_rn(__dadd_rn(__dmul_rn(-s, u), __dmul_rn(c, v)), t3);
    }
}

__device__ __forceinline__ double cross3(double ax, double az, double bx, double bz, double px, double pz)
{
    return __dsub_rn(__dmul_rn(__dsub_rn(bx, ax), __dsub_rn(pz, az)), __dmul_rn(__dsub_rn(bz, az), __dsub_rn(px, ax)));
}

// Area of the detection rectangle (dx, dz) clipped by the label rectangle (gx, gz).
__device__ double clip_area(const double *dx, const double *dz, const double *gx, const double *gz)
{
    double bx[2][CLIP_MAXV], bz[2][CLIP_MAXV];
    int n = 4, cur = 0;
    for (int k = 0; k < 4; k++) { bx[0][k] = dx[k]; bz[0][k] = dz[k]; }
    for (int e = 0; e < 4 && n > 0; e++) {
        const double ax = gx[e], az = gz[e], ex = gx[(e + 1) & 3], ez = gz[(e + 1) & 3];
        int m = 0;
        for (int i = 0; i < n; i++) {
            const int p = i == 0 ? n - 1 : i - 1;
            const double spx = bx[cur][p], spz = bz[cur][p], six = bx[cur][i], siz = bz[cur][i];
            const double dp = cross3(ax, az, ex, ez, spx, spz), di = cross3(ax, az, ex, ez, six, siz);
            const bool in_p = dp <= 0.0, in_i = di <= 0.0;
            if (in_i != in_p) {
                const double t = __ddiv_rn(dp, __dsub_rn(dp, di));
                if (m < CLIP_MAXV) {
                    bx[cur ^ 1][m] = __dadd_rn(spx, __dmul_rn(t, __dsub_rn(six, spx)));
                    bz[cur ^ 1][m] = __dadd_rn(spz, __dmul_rn(t, __dsub_rn(siz, spz)));
                    m++;
                }
            }
            if (in_i && m < CLIP_MAXV) { bx[cur ^ 1][m] = six; bz[cur ^ 1][m] = siz; m++; }
        }
        n = m;
        cur ^= 1;
    }
    if (n < 3) return 0.0;
    double acc = 0.0;
    for (int i = 0; i < n; i++) {
        const int j = i + 1 == n ? 0 : i + 1;
        acc = __dadd_rn(acc, __dsub_rn(__dmul_rn(bx[cur][i], bz[cur][j]), __dmul_rn(bx[cur][j], bz[cur][i])));
    }
    return __dmul_rn(fabs(acc), 0.5);
}

// A pair whose union (criterion -1) or detection (criterion 0) area / volume is <= 0 has overlap 0; the reference
// divides 0 by 0 there.
__device__ __forceinline__ double safe_div(double num, double den) { return den > 0.0 ? __ddiv_rn(num, den) : 0.0; }

// One side of a pair as the overlaps read it.
struct EvalBox {
    double x1, y1, x2, y2;            // image rectangle
    double t1, t2, t3, l, h, w, ry;   // location, dimensions, heading
};

// imageBoxOverlap (evaluate.cpp:420-454); d is the detection.
__device__ double image_overlap(const EvalBox &d, const EvalBox &g, bool crit0)
{
    const double w = __dsub_rn(fmin(d.x2, g.x2), fmax(d.x1, g.x1)), h = __dsub_rn(fmin(d.y2, g.y2), fmax(d.y1, g.y1));
    if (w <= 0.0 || h <= 0.0) return 0.0;
    const double inter = __dmul_rn(w, h);
    const double ad = __dmul_rn(__dsub_rn(d.x2, d.x1), __dsub_rn(d.y2, d.y1));
    const double ag = __dmul_rn(__dsub_rn(g.x2, g.x1), __dsub_rn(g.y2, g.y1));
    return crit0 ? safe_div(inter, ad) : safe_div(inter, __dsub_rn(__dadd_rn(ad, ag), inter));
}

// groundBoxOverlap and box3DOverlap (evaluate.cpp:487-537) from the corners of both rectangles.
__device__ void box_overlaps(const EvalBox &d, const double *dx, const double *dz, const EvalBox &g, const double *gx,
                             const double *gz, bool crit0, double &bev, double &v3)
{
    const double inter = clip_area(dx, dz, gx, gz);
    const double ad = __dmul_rn(fabs(d.l), fabs(d.w)), ag = __dmul_rn(fabs(g.l), fabs(g.w));
    const double ymax = fmin(d.t2, g.t2), ymin = fmax(__dsub_rn(d.t2, d.h), __dsub_rn(g.t2, g.h));
    const double iv = __dmul_rn(inter, fmax(0.0, __dsub_rn(ymax, ymin)));
    const double vd = __dmul_rn(__dmul_rn(d.h, d.l), d.w), vg = __dmul_rn(__dmul_rn(g.h, g.l), g.w);
    if (crit0) {
        bev = safe_div(inter, ad);
        v3 = safe_div(iv, vd);
    } else {
        bev = safe_div(inter, __dsub_rn(__dadd_rn(ad, ag), inter));
        v3 = safe_div(iv, __dsub_rn(__dadd_rn(vd, vg), iv));
    }
}

__device__ __forceinline__ EvalBox det_box(const float *r)     // evaluate_map's 14 columns
{
    return EvalBox{r[1], r[2], r[3], r[4], r[6], r[7], r[8], r[11], r[9], r[10], r[12]};
}

__device__ __forceinline__ EvalBox label_box(const double *r)  // a KITTI label line, type coded
{
    return EvalBox{r[4], r[5], r[6], r[7], r[11], r[12], r[13], r[10], r[8], r[9], r[14]};
}

__device__ __forceinline__ EvalBox box7(const float *r)        // (x, y, z, l, h, w, ry)
{
    return EvalBox{0.0, 0.0, 0.0, 0.0, r[0], r[1], r[2], r[3], r[4], r[5], r[6]};
}

// ---- calc_iou / calc_iou_match --------------------------------------------------------------------------------------
__global__ void __launch_bounds__(EVAL_THREADS)
box_iou_kernel(long pairs, int n, int m, int matched, const float *__restrict__ dets, const float *__restrict__ gts,
               float *__restrict__ iou_bev, float *__restrict__ iou_3d)
{
    for (long p = blockIdx.x * (long)blockDim.x + threadIdx.x; p < pairs; p += (long)gridDim.x * blockDim.x) {
        long di = p, gi = p;
        if (!matched) {
            const long s = p / ((long)n * m), r = p - s * n * m, i = r / m, j = r - i * m;
            di = s * n + i;
            gi = s * m + j;
        }
        const EvalBox d = box7(dets + 7 * di), g = box7(gts + 7 * gi);
        double dx[4], dz[4], gx[4], gz[4], bev, v3;
        rect_corners(d.t1, d.t3, d.l, d.w, d.ry, dx, dz);
        rect_corners(g.t1, g.t3, g.l, g.w, g.ry, gx, gz);
        box_overlaps(d, dx, dz, g, gx, gz, false, bev, v3);
        iou_bev[p] = (float)bev;
        iou_3d[p] = (float)v3;
    }
}

// ---- the evaluation ------------------------------------------------------------------------------------------------
// Overlaps of every (detection, label row) pair of a frame, one CTA per frame: ov[(pair_off[f] + j * ng + i) * 3 + metric]
// = image / BEV / 3-D IoU, or for DontCare rows the overlap over the detection (criterion 0), the only one they are
// used with (evaluate.cpp:778).
__global__ void __launch_bounds__(EVAL_THREADS)
eval_overlap_kernel(const float *__restrict__ dets, const int *__restrict__ det_off, const double *__restrict__ labels,
                    const int *__restrict__ label_off, const long *__restrict__ pair_off, double *__restrict__ ov)
{
    __shared__ double s_gx[EVAL_MAX_LABELS][4], s_gz[EVAL_MAX_LABELS][4];
    __shared__ EvalBox s_box[EVAL_MAX_LABELS];
    __shared__ int s_dc[EVAL_MAX_LABELS];
    const int f = blockIdx.x;
    const int d0 = det_off[f], nd = det_off[f + 1] - d0, g0 = label_off[f], ng = label_off[f + 1] - g0;
    for (int i = threadIdx.x; i < ng; i += blockDim.x) {
        const double *r = labels + 15 * (long)(g0 + i);
        const EvalBox g = label_box(r);
        s_box[i] = g;
        s_dc[i] = (int)r[0] == T_DONTCARE;
        rect_corners(g.t1, g.t3, g.l, g.w, g.ry, s_gx[i], s_gz[i]);
    }
    __syncthreads();
    double *o = ov + 3 * pair_off[f];
    const long np = (long)nd * ng;
    for (long p = threadIdx.x; p < np; p += blockDim.x) {
        const int j = (int)(p / ng), i = (int)(p - (long)j * ng);
        const EvalBox d = det_box(dets + 14 * (long)(d0 + j));
        double dx[4], dz[4], bev, v3;
        rect_corners(d.t1, d.t3, d.l, d.w, d.ry, dx, dz);
        const bool crit0 = s_dc[i] != 0;
        box_overlaps(d, dx, dz, s_box[i], s_gx[i], s_gz[i], crit0, bev, v3);
        o[3 * p + 0] = image_overlap(d, s_box[i], crit0);
        o[3 * p + 1] = bev;
        o[3 * p + 2] = v3;
    }
}

__device__ __forceinline__ int min_height(int diff) { return diff == 0 ? 40 : 25; }

// cleanData (evaluate.cpp:574-647) for one label row: 0 counted, 1 ignored, -1 another class.
__device__ int ignored_gt(const double *r, int cls, int diff)
{
    const int type = (int)r[0];
    const double height = __dsub_rn(r[7], r[5]);
    const double max_trunc = diff == 0 ? 0.15 : (diff == 1 ? 0.3 : 0.5);
    int valid;
    if (type == cls) valid = 1;
    else if ((cls == T_PED && type == T_SIT) || (cls == T_CAR && type == T_VAN)) valid = 0;
    else valid = -1;
    const bool ignore = (int)r[2] > diff || r[1] > max_trunc || height <= (double)min_height(diff);   // MAX_OCCLUSION = diff
    if (valid == 1 && !ignore) return 0;
    if (valid == 0 || (ignore && valid == 1)) return 1;
    return -1;
}

// cleanData for one detection row: int32 height below the minimum -> 1, the class -> 0, otherwise -1.
__device__ int ignored_det(const float *r, int cls, int diff)
{
    const double h = fabs(__dsub_rn((double)r[2], (double)r[4]));
    const int height = h >= 2147483647.0 ? 2147483647 : (int)h;
    if (height < min_height(diff)) return 1;
    const float c = r[0];
    const int dc = (c > -1.0f && c < 3.0f) ? (int)c : 3;      // int(class); anything but 0, 1, 2 is "DontCare"
    return dc == cls ? 0 : -1;
}

constexpr double NO_DETECTION = -10000000.0;
constexpr unsigned char ST_COUNTED = 1, ST_IGNORED = 2, ST_BELOW = 4, ST_ASSIGNED = 8;

// computeStatistics (evaluate.cpp:649-830) for one frame and case.  First pass (compute_fp false): writes the scores of
// the true positives to v.  Counting pass: tp, fp, fn at score threshold `thresh`.
__device__ void frame_stats(int nd, int ng, const float *det, const double *lab, const double *ov, int cls, int diff,
                            int metric, bool compute_fp, double thresh, int &tp, int &fp, int &fn, double *v)
{
    unsigned char st[EVAL_MAX_DETS];
    const double min_ov = cls == T_CAR ? 0.7 : 0.5;
    for (int j = 0; j < nd; j++) {
        const float *r = det + 14 * (long)j;
        const int id = ignored_det(r, cls, diff);
        st[j] = (id == 0 ? ST_COUNTED : (id == 1 ? ST_IGNORED : 0)) | (compute_fp && (double)r[13] < thresh ? ST_BELOW : 0);
    }
    tp = fp = fn = 0;
    for (int i = 0; i < ng; i++) {
        const int ig = ignored_gt(lab + 15 * (long)i, cls, diff);
        if (ig == -1) continue;
        int det_idx = -1;
        bool aid = false;
        double valid = NO_DETECTION, max_overlap = 0.0;
        for (int j = 0; j < nd; j++) {
            const unsigned char s = st[j];
            if (!(s & (ST_COUNTED | ST_IGNORED)) || (s & (ST_ASSIGNED | ST_BELOW))) continue;
            const double o = ov[((long)j * ng + i) * 3 + metric];
            if (!compute_fp) {
                const double score = (double)det[14 * (long)j + 13];
                if (o > min_ov && score > valid) { det_idx = j; valid = score; }
            } else if (o > min_ov && (o > max_overlap || aid) && (s & ST_COUNTED)) {
                max_overlap = o; det_idx = j; valid = 1.0; aid = false;
            } else if (o > min_ov && valid == NO_DETECTION && (s & ST_IGNORED)) {
                det_idx = j; valid = 1.0; aid = true;
            }
        }
        if (valid == NO_DETECTION) {
            if (ig == 0) fn++;
        } else if (ig == 1 || (st[det_idx] & ST_IGNORED)) {
            st[det_idx] |= ST_ASSIGNED;
        } else {
            if (v) v[tp] = (double)det[14 * (long)det_idx + 13];
            tp++;
            st[det_idx] |= ST_ASSIGNED;
        }
    }
    if (!compute_fp) return;
    for (int j = 0; j < nd; j++)
        if ((st[j] & (ST_COUNTED | ST_ASSIGNED | ST_BELOW)) == ST_COUNTED) fp++;
    int nstuff = 0;
    for (int i = 0; i < ng; i++) {
        if ((int)lab[15 * (long)i] != T_DONTCARE) continue;
        for (int j = 0; j < nd; j++) {
            if ((st[j] & (ST_COUNTED | ST_ASSIGNED | ST_BELOW)) != ST_COUNTED) continue;
            if (ov[((long)j * ng + i) * 3 + metric] > min_ov) { st[j] |= ST_ASSIGNED; nstuff++; }
        }
    }
    fp -= nstuff;
}

// First pass, one thread per (frame, case): tp_scores[case * label_rows + label_off[f] + k], k < tp_count[case, f];
// n_gt[case, f] = labels counted in the recall denominator.
__global__ void __launch_bounds__(128)
eval_first_pass_kernel(int frames, const float *__restrict__ dets, const int *__restrict__ det_off,
                       const double *__restrict__ labels, const int *__restrict__ label_off, const long *__restrict__ pair_off,
                       const double *__restrict__ ov, long label_rows, double *__restrict__ tp_scores,
                       int *__restrict__ tp_count, int *__restrict__ n_gt)
{
    const long t = blockIdx.x * (long)blockDim.x + threadIdx.x;
    if (t >= (long)frames * EVAL_CASES) return;
    const int f = (int)(t / EVAL_CASES), cs = (int)(t - (long)f * EVAL_CASES);
    const int metric = cs / 9, cls = (cs / 3) % 3, diff = cs % 3;
    const int d0 = det_off[f], nd = det_off[f + 1] - d0, g0 = label_off[f], ng = label_off[f + 1] - g0;
    const double *lab = labels + 15 * (long)g0;
    int cnt = 0;
    for (int i = 0; i < ng; i++) cnt += ignored_gt(lab + 15 * (long)i, cls, diff) == 0;
    int tp, fp, fn;
    frame_stats(nd, ng, dets + 14 * (long)d0, lab, ov + 3 * pair_off[f], cls, diff, metric, false, 0.0, tp, fp, fn,
                tp_scores + cs * label_rows + g0);
    tp_count[cs * frames + f] = tp;
    n_gt[cs * frames + f] = cnt;
}

// Counting pass, one thread per (frame, case, threshold): counts[(case * 41 + t) * 3 + {0, 1, 2}] += tp, fp, fn.
__global__ void __launch_bounds__(128)
eval_count_kernel(int frames, const float *__restrict__ dets, const int *__restrict__ det_off,
                  const double *__restrict__ labels, const int *__restrict__ label_off, const long *__restrict__ pair_off,
                  const double *__restrict__ ov, const double *__restrict__ thresholds, const int *__restrict__ n_thresholds,
                  int *__restrict__ counts)
{
    const long t = blockIdx.x * (long)blockDim.x + threadIdx.x;
    if (t >= (long)frames * EVAL_CASES * EVAL_NSAMPLE) return;
    const int k = (int)(t % EVAL_NSAMPLE);
    const long fc = t / EVAL_NSAMPLE;
    const int f = (int)(fc / EVAL_CASES), cs = (int)(fc - (long)f * EVAL_CASES);
    if (k >= n_thresholds[cs]) return;
    const int metric = cs / 9, cls = (cs / 3) % 3, diff = cs % 3;
    const int d0 = det_off[f], nd = det_off[f + 1] - d0, g0 = label_off[f], ng = label_off[f + 1] - g0;
    int tp, fp, fn;
    frame_stats(nd, ng, dets + 14 * (long)d0, labels + 15 * (long)g0, ov + 3 * pair_off[f], cls, diff, metric, true,
                thresholds[cs * EVAL_NSAMPLE + k], tp, fp, fn, nullptr);
    int *c = counts + 3 * ((long)cs * EVAL_NSAMPLE + k);
    if (tp) atomicAdd(c + 0, tp);
    if (fp) atomicAdd(c + 1, fp);
    if (fn) atomicAdd(c + 2, fn);
}

}  // namespace ssd3d

using namespace ssd3d;

static int box_iou_launch(long pairs, int n, int m, int matched, const float *dets, const float *gts, float *iou_bev,
                          float *iou_3d, ssd3d_stream_t stream)
{
    if (pairs == 0) return 0;                // nothing read or written: an empty tensor may have a null data pointer
    SSD3D_REQUIRE(dets && gts && iou_bev && iou_3d, "box_iou: null pointer");
    const long blocks = (pairs + EVAL_THREADS - 1) / EVAL_THREADS;
    box_iou_kernel<<<(int)(blocks < 65535L * 16 ? blocks : 65535L * 16), EVAL_THREADS, 0, (cudaStream_t)stream>>>(
        pairs, n, m, matched, dets, gts, iou_bev, iou_3d);
    SSD3D_LAUNCH_CHECK("box_iou_kernel");
}

extern "C" int ssd3d_box_iou(int b, int n, int m, const float *dets, const float *gts, float *iou_bev, float *iou_3d,
                             ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && n >= 0 && m >= 0, "box_iou: bad shape b=%d n=%d m=%d", b, n, m);
    return box_iou_launch((long)b * n * m, n, m, 0, dets, gts, iou_bev, iou_3d, stream);
}

extern "C" int ssd3d_box_iou_matched(long n, const float *dets, const float *gts, float *iou_bev, float *iou_3d,
                                     ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(n >= 0, "box_iou_matched: bad row count %ld", n);
    return box_iou_launch(n, 1, 1, 1, dets, gts, iou_bev, iou_3d, stream);
}

extern "C" size_t ssd3d_eval_workspace(long pairs)
{
    return pairs > 0 ? (size_t)pairs * 3 * sizeof(double) : 0;
}

#define EVAL_COMMON_CHECKS(op)                                                                                          \
    SSD3D_REQUIRE(frames >= 0, op ": bad frame count %d", frames);                                                       \
    SSD3D_REQUIRE(max_dets >= 0 && max_dets <= EVAL_MAX_DETS, op ": at most %d detections per frame (got %d)",         \
                  EVAL_MAX_DETS, max_dets);                                                                              \
    SSD3D_REQUIRE(max_labels >= 0 && max_labels <= EVAL_MAX_LABELS, op ": at most %d label rows per frame (got %d)",   \
                  EVAL_MAX_LABELS, max_labels)

extern "C" int ssd3d_eval_overlaps(int frames, int max_dets, int max_labels, const float *dets, const int *det_off,
                                   const double *labels, const int *label_off, const long *pair_off, void *workspace,
                                   ssd3d_stream_t stream)
{
    EVAL_COMMON_CHECKS("eval_overlaps");
    if (frames == 0 || max_dets == 0 || max_labels == 0) return 0;
    SSD3D_REQUIRE(dets && det_off && labels && label_off && pair_off && workspace, "eval_overlaps: null pointer");
    eval_overlap_kernel<<<frames, EVAL_THREADS, 0, (cudaStream_t)stream>>>(dets, det_off, labels, label_off, pair_off,
                                                                          (double *)workspace);
    SSD3D_LAUNCH_CHECK("eval_overlap_kernel");
}

extern "C" int ssd3d_eval_first_pass(int frames, int max_dets, int max_labels, const float *dets, const int *det_off,
                                     const double *labels, const int *label_off, const long *pair_off,
                                     const void *workspace, long label_rows, double *tp_scores, int *tp_count, int *n_gt,
                                     ssd3d_stream_t stream)
{
    EVAL_COMMON_CHECKS("eval_first_pass");
    SSD3D_REQUIRE(label_rows >= 0, "eval_first_pass: bad label row count %ld", label_rows);
    if (frames == 0) return 0;
    SSD3D_REQUIRE(det_off && label_off && pair_off && tp_count && n_gt, "eval_first_pass: null pointer");
    const long threads = (long)frames * EVAL_CASES;
    eval_first_pass_kernel<<<ceil_div(threads, 128), 128, 0, (cudaStream_t)stream>>>(
        frames, dets, det_off, labels, label_off, pair_off, (const double *)workspace, label_rows, tp_scores, tp_count, n_gt);
    SSD3D_LAUNCH_CHECK("eval_first_pass_kernel");
}

extern "C" int ssd3d_eval_count(int frames, int max_dets, int max_labels, const float *dets, const int *det_off,
                                const double *labels, const int *label_off, const long *pair_off, const void *workspace,
                                const double *thresholds, const int *n_thresholds, int *counts, ssd3d_stream_t stream)
{
    EVAL_COMMON_CHECKS("eval_count");
    SSD3D_REQUIRE(counts && n_thresholds && thresholds, "eval_count: null pointer");
    cudaError_t e = cudaMemsetAsync(counts, 0, sizeof(int) * 3 * EVAL_CASES * EVAL_NSAMPLE, (cudaStream_t)stream);
    if (e != cudaSuccess) return cuda_status(e, "eval_count: clearing the counts");
    if (frames == 0) return 0;
    SSD3D_REQUIRE(det_off && label_off && pair_off, "eval_count: null pointer");
    const long threads = (long)frames * EVAL_CASES * EVAL_NSAMPLE;
    eval_count_kernel<<<ceil_div(threads, 128), 128, 0, (cudaStream_t)stream>>>(
        frames, dets, det_off, labels, label_off, pair_off, (const double *)workspace, thresholds, n_thresholds, counts);
    SSD3D_LAUNCH_CHECK("eval_count_kernel");
}
