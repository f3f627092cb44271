/* C twin of the GPU KITTI evaluator (3dssd_b200/csrc/box_eval.cu), test-only.
 *
 * It follows the arithmetic recipe of DESIGN.md section 3.10 operation for operation, so that it and the kernels give
 * the same bits: one double-precision sincos (Cody-Waite reduction by pi/2, fdlibm's minimax polynomials evaluated with
 * explicit fma), rectangle corners rn(rn(rn(c*a) + rn(s*b)) + t) from |l|/2 and |w|/2, Sutherland-Hodgman clipping of
 * the detection rectangle by the label rectangle and a shoelace area in vertex order.  Built with -ffp-contract=off,
 * so every other operation is rounded on its own.
 *
 * The rules (which overlap each metric uses, cleanData, computeStatistics, getThresholds, eval_class) are those of the
 * reference's evaluator, lib/utils/tf_ops/evaluation/evaluate.cpp; oracle/kitti_eval.py restates them readably in
 * float64 with math.sin / math.cos, and the tests hold this file to that restatement.
 *
 * Detection rows: 14 floats (class, x1, y1, x2, y2, alpha, t1, t2, t3, h, w, l, ry, score), evaluate_map's layout.
 * Label rows: 15 doubles (type code, truncation, occlusion, alpha, x1, y1, x2, y2, h, w, l, t1, t2, t3, ry): the 15
 * fields of a KITTI label line with the type name replaced by its code (0 Car, 1 Pedestrian, 2 Cyclist, 3 Van,
 * 4 Person_sitting, 5 DontCare, 6 anything else).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define NSAMPLE 41
#define MAXV 16

enum { T_CAR = 0, T_PED = 1, T_CYC = 2, T_VAN = 3, T_SIT = 4, T_DONTCARE = 5, T_OTHER = 6 };

/* ---- sincos: Cody-Waite by pi/2, fdlibm kernels ------------------------------------------------------------------ */
static const double INV_PIO2 = 0x1.45f306dc9c883p-1;
static const double PIO2_HI = 0x1.921fb54442d18p+0;
static const double PIO2_MID = 0x1.1a62633145c07p-54;
static const double S1 = -1.66666666666666324348e-01, S2 = 8.33333333332248946124e-03, S3 = -1.98412698298579493134e-04,
                    S4 = 2.75573137070700676789e-06, S5 = -2.50507602534068634195e-08, S6 = 1.58969099521155010221e-10;
static const double C1 = 4.16666666666666019037e-02, C2 = -1.38888888888741095749e-03, C3 = 2.48015872894767294178e-05,
                    C4 = -2.75573143513906633035e-07, C5 = 2.08757232129817482790e-09, C6 = -1.13596475577881948265e-11;

static double k_sin(double r)
{
    const double z = r * r;
    double p = fma(z, S6, S5);
    p = fma(z, p, S4);
    p = fma(z, p, S3);
    p = fma(z, p, S2);
    p = fma(z, p, S1);
    return fma(r * z, p, r);
}

static double k_cos(double r)
{
    const double z = r * r;
    double p = fma(z, C6, C5);
    p = fma(z, p, C4);
    p = fma(z, p, C3);
    p = fma(z, p, C2);
    p = fma(z, p, C1);
    const double hz = 0.5 * z, w = 1.0 - hz;
    return w + fma(z, z * p, (1.0 - w) - hz);
}

void kitti_sincos(double x, double *s, double *c)
{
    const double n = rint(x * INV_PIO2);
    double r = fma(-n, PIO2_HI, x);
    r = fma(-n, PIO2_MID, r);
    const double sr = k_sin(r), cr = k_cos(r);
    switch (((long long)n) & 3) {
        case 0: *s = sr; *c = cr; break;
        case 1: *s = cr; *c = -sr; break;
        case 2: *s = -sr; *c = -cr; break;
        default: *s = -cr; *c = sr; break;
    }
}

void kitti_sincos_n(long n, const double *x, double *s, double *c)
{
    for (long i = 0; i < n; i++) kitti_sincos(x[i], s + i, c + i);
}

/* ---- rotated rectangles ---------------------------------------------------------------------------------------- */
/* Corners in the order of toPolygon (evaluate.cpp:461-485): (l/2, w/2), (l/2, -w/2), (-l/2, -w/2), (-l/2, w/2) rotated
 * by [[cos, sin], [-sin, cos]] and offset by (t1, t3); a clockwise polygon in the (x, z) plane. */
static void rect_corners(double t1, double t3, double l, double w, double ry, double *px, double *pz)
{
    double s, c;
    kitti_sincos(ry, &s, &c);
    const double a = fabs(l) * 0.5, b = fabs(w) * 0.5;
    const double la[4] = {a, a, -a, -a}, wb[4] = {b, -b, -b, b};
    for (int k = 0; k < 4; k++) {
        px[k] = ((c * la[k]) + (s * wb[k])) + t1;
        pz[k] = ((-s * la[k]) + (c * wb[k])) + t3;
    }
}

static double cross3(double ax, double az, double bx, double bz, double px, double pz)
{
    return ((bx - ax) * (pz - az)) - ((bz - az) * (px - ax));
}

/* Area of (detection rectangle) clipped by (label rectangle). */
static double clip_area(const double *dx, const double *dz, const double *gx, const double *gz)
{
    double bx[2][MAXV], bz[2][MAXV];
    int n = 4, cur = 0;
    for (int k = 0; k < 4; k++) { bx[0][k] = dx[k]; bz[0][k] = dz[k]; }
    for (int e = 0; e < 4 && n > 0; e++) {
        const double ax = gx[e], az = gz[e], ex = gx[(e + 1) & 3], ez = gz[(e + 1) & 3];
        const double *sx = bx[cur], *sz = bz[cur];
        double *ox = bx[cur ^ 1], *oz = bz[cur ^ 1];
        int m = 0;
        for (int i = 0; i < n; i++) {
            const int p = i == 0 ? n - 1 : i - 1;
            const double dp = cross3(ax, az, ex, ez, sx[p], sz[p]), di = cross3(ax, az, ex, ez, sx[i], sz[i]);
            const int in_p = dp <= 0.0, in_i = di <= 0.0;
            if (in_i != in_p) {
                const double t = dp / (dp - di);
                if (m < MAXV) { ox[m] = sx[p] + t * (sx[i] - sx[p]); oz[m] = sz[p] + t * (sz[i] - sz[p]); m++; }
            }
            if (in_i && m < MAXV) { ox[m] = sx[i]; oz[m] = sz[i]; m++; }
        }
        n = m;
        cur ^= 1;
    }
    if (n < 3) return 0.0;
    double acc = 0.0;
    for (int i = 0; i < n; i++) {
        const int j = i + 1 == n ? 0 : i + 1;
        acc = acc + ((bx[cur][i] * bz[cur][j]) - (bx[cur][j] * bz[cur][i]));
    }
    return fabs(acc) * 0.5;
}

/* A box as the overlaps see it: (t1, t2, t3, l, h, w, ry) plus the image rectangle. */
typedef struct { double x1, y1, x2, y2, t1, t2, t3, l, h, w, ry; } Box;

static Box det_box(const float *r)
{
    Box b = {r[1], r[2], r[3], r[4], r[6], r[7], r[8], r[11], r[9], r[10], r[12]};
    return b;
}

static Box label_box(const double *r)
{
    Box b = {r[4], r[5], r[6], r[7], r[11], r[12], r[13], r[10], r[8], r[9], r[14]};
    return b;
}

static double safe_div(double num, double den) { return den > 0.0 ? num / den : 0.0; }

/* imageBoxOverlap (evaluate.cpp:420-454); criterion -1: union, 0: detection area. */
static double image_overlap(const Box *a, const Box *b, int crit)
{
    const double x1 = fmax(a->x1, b->x1), y1 = fmax(a->y1, b->y1), x2 = fmin(a->x2, b->x2), y2 = fmin(a->y2, b->y2);
    const double w = x2 - x1, h = y2 - y1;
    if (w <= 0.0 || h <= 0.0) return 0.0;
    const double inter = w * h;
    const double a_area = (a->x2 - a->x1) * (a->y2 - a->y1), b_area = (b->x2 - b->x1) * (b->y2 - b->y1);
    return crit < 0 ? safe_div(inter, (a_area + b_area) - inter) : safe_div(inter, a_area);
}

/* groundBoxOverlap / box3DOverlap (evaluate.cpp:487-537): out[0] BEV, out[1] 3-D. */
static void box_overlaps(const Box *d, const Box *g, int crit, double *bev, double *v3)
{
    double dx[4], dz[4], gx[4], gz[4];
    rect_corners(d->t1, d->t3, d->l, d->w, d->ry, dx, dz);
    rect_corners(g->t1, g->t3, g->l, g->w, g->ry, gx, gz);
    const double inter = clip_area(dx, dz, gx, gz);
    const double area_d = fabs(d->l) * fabs(d->w), area_g = fabs(g->l) * fabs(g->w);
    const double ymax = fmin(d->t2, g->t2), ymin = fmax(d->t2 - d->h, g->t2 - g->h);
    const double inter_vol = inter * fmax(0.0, ymax - ymin);
    const double det_vol = (d->h * d->l) * d->w, gt_vol = (g->h * g->l) * g->w;
    if (crit < 0) {
        *bev = safe_div(inter, (area_d + area_g) - inter);
        *v3 = safe_div(inter_vol, (det_vol + gt_vol) - inter_vol);
    } else {
        *bev = safe_div(inter, area_d);
        *v3 = safe_div(inter_vol, det_vol);
    }
}

/* Row-wise overlaps of detection rows [n,14] with label rows [n,15]: out [n,6] = image, BEV, 3-D IoU, then the same
 * three over the detection (criterion 0). */
void kitti_pair_overlaps(long n, const float *det, const double *lab, double *out)
{
    for (long i = 0; i < n; i++) {
        const Box d = det_box(det + 14 * i), g = label_box(lab + 15 * i);
        out[6 * i + 0] = image_overlap(&d, &g, -1);
        box_overlaps(&d, &g, -1, out + 6 * i + 1, out + 6 * i + 2);
        out[6 * i + 3] = image_overlap(&d, &g, 0);
        box_overlaps(&d, &g, 0, out + 6 * i + 4, out + 6 * i + 5);
    }
}

static Box box7(const float *r)
{
    Box b = {0, 0, 0, 0, r[0], r[1], r[2], r[3], r[4], r[5], r[6]};
    return b;
}

/* calc_iou (tf_evaluate.cpp:35-48,142-179): [b,n,7] x [b,m,7] -> [b,n,m] BEV and 3-D IoU, float32. */
void kitti_box_iou(int b, int n, int m, const float *dets, const float *gts, float *iou_bev, float *iou_3d)
{
    for (long s = 0; s < b; s++)
        for (long i = 0; i < n; i++)
            for (long j = 0; j < m; j++) {
                const Box d = box7(dets + (s * n + i) * 7), g = box7(gts + (s * m + j) * 7);
                double bev, v3;
                box_overlaps(&d, &g, -1, &bev, &v3);
                iou_bev[(s * n + i) * m + j] = (float)bev;
                iou_3d[(s * n + i) * m + j] = (float)v3;
            }
}

/* calc_iou_match (tf_evaluate.cpp:50-63,182-217): row i of dets against row i of gts. */
void kitti_box_iou_matched(long n, const float *dets, const float *gts, float *iou_bev, float *iou_3d)
{
    for (long i = 0; i < n; i++) {
        const Box d = box7(dets + 7 * i), g = box7(gts + 7 * i);
        double bev, v3;
        box_overlaps(&d, &g, -1, &bev, &v3);
        iou_bev[i] = (float)bev;
        iou_3d[i] = (float)v3;
    }
}

/* ---- the evaluation ------------------------------------------------------------------------------------------------ */
static const int MIN_HEIGHT[3] = {40, 25, 25};
static const int MAX_OCCLUSION[3] = {0, 1, 2};
static const double MAX_TRUNCATION[3] = {0.15, 0.3, 0.5};
static const double MIN_OVERLAP[3] = {0.7, 0.5, 0.5};          /* per class, every metric (evaluate.cpp:52) */
#define NO_DETECTION (-10000000.0)

/* Detection class of a row: int(row[0]) as evaluate.cpp:279-303 reads it; anything but 0, 1, 2 is "DontCare". */
static int det_class(float v) { return (v > -1.0f && v < 3.0f) ? (int)v : 3; }

/* cleanData (evaluate.cpp:574-647) for one label row: 0 valid, 1 ignored, -1 other class. */
static int ignored_gt(const double *r, int cls, int diff)
{
    const int type = (int)r[0];
    const double height = r[7] - r[5];
    int valid;
    if (type == cls) valid = 1;
    else if ((cls == T_PED && type == T_SIT) || (cls == T_CAR && type == T_VAN)) valid = 0;
    else valid = -1;
    const int ignore = (int)r[2] > MAX_OCCLUSION[diff] || r[1] > MAX_TRUNCATION[diff] || height <= MIN_HEIGHT[diff];
    if (valid == 1 && !ignore) return 0;
    if (valid == 0 || (ignore && valid == 1)) return 1;
    return -1;
}

/* int32_t height = fabs(y1 - y2) (evaluate.cpp:637), saturated where the conversion would overflow. */
static int det_height(const float *r)
{
    const double h = fabs((double)r[2] - (double)r[4]);
    return h >= 2147483647.0 ? 2147483647 : (int)h;
}

static int ignored_det(const float *r, int cls, int diff)
{
    if (det_height(r) < MIN_HEIGHT[diff]) return 1;
    return det_class(r[0]) == cls ? 0 : -1;
}

typedef struct {
    int nd, ng;
    const float *det;
    const double *lab;
    double *ov;          /* [nd][ng][3]: IoU per metric; criterion 0 for DontCare rows */
} Frame;

/* computeStatistics (evaluate.cpp:649-830) for one frame; thresh < 0 with compute_fp = 0 is the first pass. */
static void frame_stats(const Frame *f, int cls, int diff, int metric, int compute_fp, double thresh, int *tp, int *fp,
                        int *fn, double *v, int *nv)
{
    unsigned char assigned[1024], ign_thr[1024];
    int idet[1024];
    const double min_ov = MIN_OVERLAP[cls];
    for (int j = 0; j < f->nd; j++) {
        assigned[j] = 0;
        idet[j] = ignored_det(f->det + 14 * j, cls, diff);
        ign_thr[j] = compute_fp && (double)f->det[14 * j + 13] < thresh;
    }
    *tp = *fp = *fn = 0;
    for (int i = 0; i < f->ng; i++) {
        const int ig = ignored_gt(f->lab + 15 * i, cls, diff);
        if (ig == -1) continue;
        int det_idx = -1, aid = 0;
        double valid = NO_DETECTION, max_overlap = 0.0;
        for (int j = 0; j < f->nd; j++) {
            if (idet[j] == -1 || assigned[j] || ign_thr[j]) continue;
            const double o = f->ov[((long)j * f->ng + i) * 3 + metric];
            const double score = (double)f->det[14 * j + 13];
            if (!compute_fp && o > min_ov && score > valid) {
                det_idx = j;
                valid = score;
            } else if (compute_fp && o > min_ov && (o > max_overlap || aid) && idet[j] == 0) {
                max_overlap = o;
                det_idx = j;
                valid = 1;
                aid = 0;
            } else if (compute_fp && o > min_ov && valid == NO_DETECTION && idet[j] == 1) {
                det_idx = j;
                valid = 1;
                aid = 1;
            }
        }
        if (valid == NO_DETECTION && ig == 0) {
            (*fn)++;
        } else if (valid != NO_DETECTION && (ig == 1 || idet[det_idx] == 1)) {
            assigned[det_idx] = 1;
        } else if (valid != NO_DETECTION) {
            (*tp)++;
            if (v) v[(*nv)++] = (double)f->det[14 * det_idx + 13];
            assigned[det_idx] = 1;
        }
    }
    if (!compute_fp) return;
    for (int j = 0; j < f->nd; j++)
        if (!(assigned[j] || idet[j] == -1 || idet[j] == 1 || ign_thr[j])) (*fp)++;
    int nstuff = 0;
    for (int i = 0; i < f->ng; i++) {
        if ((int)f->lab[15 * i] != T_DONTCARE) continue;
        for (int j = 0; j < f->nd; j++) {
            if (assigned[j] || idet[j] == -1 || idet[j] == 1 || ign_thr[j]) continue;
            if (f->ov[((long)j * f->ng + i) * 3 + metric] > min_ov) {
                assigned[j] = 1;
                nstuff++;
            }
        }
    }
    *fp -= nstuff;
}

static int cmp_desc(const void *a, const void *b)
{
    const double x = *(const double *)a, y = *(const double *)b;
    return x < y ? 1 : (x > y ? -1 : 0);
}

/* getThresholds (evaluate.cpp:539-572): v sorted in place, at most NSAMPLE thresholds written to t. */
int kitti_get_thresholds(double *v, long nv, double n_gt, double *t)
{
    qsort(v, (size_t)nv, sizeof(double), cmp_desc);
    double current_recall = 0.0;
    int nt = 0;
    for (long i = 0; i < nv; i++) {
        const double l_recall = (double)(i + 1) / n_gt;
        const double r_recall = i < nv - 1 ? (double)(i + 2) / n_gt : l_recall;
        if ((r_recall - current_recall) < (current_recall - l_recall) && i < nv - 1) continue;
        if (nt < NSAMPLE) t[nt] = v[i];   /* never reached in practice: the walk yields at most NSAMPLE */
        nt++;
        current_recall += 1.0 / (NSAMPLE - 1.0);
    }
    return nt;
}

/* eval() (evaluate.cpp:1229-1343) on in-memory rows: out = 6 arrays [3 classes][3 difficulties][41] in the order
 * precision_image, aos_image, precision_ground, aos_ground, precision_3d, aos_3d.  Returns 0, or -1 when a frame exceeds
 * 1024 detections. */
int kitti_evaluate(int frames, const float *det, const int *numlist, const double *lab, const int *label_count, float *out)
{
    const int per = 3 * 3 * NSAMPLE;
    for (int i = 0; i < 6 * per; i++) out[i] = -1.0f;
    long nd_all = 0, ng_all = 0;
    for (int f = 0; f < frames; f++) {
        if (numlist[f] > 1024 || numlist[f] < 0 || label_count[f] < 0) return -1;
        nd_all += numlist[f];
        ng_all += label_count[f];
    }
    Frame *fr = (Frame *)calloc((size_t)(frames > 0 ? frames : 1), sizeof(Frame));
    long od = 0, og = 0;
    for (int f = 0; f < frames; f++) {
        Frame *F = fr + f;
        F->nd = numlist[f];
        F->ng = label_count[f];
        F->det = det + 14 * od;
        F->lab = lab + 15 * og;
        F->ov = (double *)malloc(sizeof(double) * 3 * ((size_t)F->nd * F->ng + 1));
        for (int j = 0; j < F->nd; j++) {
            const Box d = det_box(F->det + 14 * j);
            for (int i = 0; i < F->ng; i++) {
                const Box g = label_box(F->lab + 15 * i);
                const int crit = (int)F->lab[15 * i] == T_DONTCARE ? 0 : -1;
                double *o = F->ov + ((long)j * F->ng + i) * 3;
                o[0] = image_overlap(&d, &g, crit);
                box_overlaps(&d, &g, crit, o + 1, o + 2);
            }
        }
        od += F->nd;
        og += F->ng;
    }
    /* a class is evaluated in a metric only if one of its detections has the fields that metric needs (:316-331) */
    int eval_flag[3][3] = {{0}};
    for (long j = 0; j < nd_all; j++) {
        const float *r = det + 14 * j;
        const int c = det_class(r[0]);
        if (c > 2) continue;
        if (r[1] >= 0.0f) eval_flag[0][c] = 1;
        if (r[6] != -1000.0f && r[8] != -1000.0f && r[10] > 0.0f && r[11] > 0.0f) eval_flag[1][c] = 1;
        if (r[6] != -1000.0f && r[7] != -1000.0f && r[8] != -1000.0f && r[9] > 0.0f && r[10] > 0.0f && r[11] > 0.0f)
            eval_flag[2][c] = 1;
    }
    double *v = (double *)malloc(sizeof(double) * (size_t)(ng_all + 1));
    for (int m = 0; m < 3; m++)
        for (int c = 0; c < 3; c++) {
            if (!eval_flag[m][c]) continue;
            for (int d = 0; d < 3; d++) {
                long nv = 0;
                int n_gt = 0;
                for (int f = 0; f < frames; f++) {
                    for (int i = 0; i < fr[f].ng; i++) n_gt += ignored_gt(fr[f].lab + 15 * i, c, d) == 0;
                    int tp, fp, fn, k = 0;
                    frame_stats(fr + f, c, d, m, 0, 0.0, &tp, &fp, &fn, v + nv, &k);
                    nv += k;
                }
                double thr[NSAMPLE];
                const int nt = kitti_get_thresholds(v, nv, (double)n_gt, thr);
                long tp[NSAMPLE] = {0}, fp[NSAMPLE] = {0};
                for (int f = 0; f < frames; f++)
                    for (int t = 0; t < nt; t++) {
                        int a, b, e;
                        frame_stats(fr + f, c, d, m, 1, thr[t], &a, &b, &e, NULL, NULL);
                        tp[t] += a;
                        fp[t] += b;
                    }
                double prec[NSAMPLE];
                for (int t = 0; t < NSAMPLE; t++) prec[t] = t < nt ? (double)tp[t] / (double)(tp[t] + fp[t]) : 0.0;
                for (int t = 0; t < nt; t++) {           /* max_element over [t, end): the first of the largest */
                    double best = prec[t];
                    for (int u = t + 1; u < NSAMPLE; u++)
                        if (best < prec[u]) best = prec[u];
                    prec[t] = best;
                }
                float *dst = out + (2 * m) * per + (c * 3 + d) * NSAMPLE;
                for (int t = 0; t < NSAMPLE; t++) dst[t] = (float)prec[t];
            }
        }
    free(v);
    for (int f = 0; f < frames; f++) free(fr[f].ov);
    free(fr);
    return 0;
}
