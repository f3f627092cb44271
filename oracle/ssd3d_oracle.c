/*
 * ssd3d_oracle.c -- CPU restatement of the reference's set-abstraction operators.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is part of the product: only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may load it.
 * The product path (3dssd_b200/) never imports, links or calls this file.
 *
 * Every function restates one reference CUDA kernel for a scalar CPU, reproducing the
 * kernel's arithmetic *as nvcc contracts it* (verified in PTX, see DESIGN.md "Arithmetic
 * recipes") so that integer outputs are bit-exact.  Build with -ffp-contract=off: every
 * fused multiply-add below is an explicit fmaf().
 *
 * Parity pin: the reference has no golden vectors for this path (SURVEY.md section 8c); the pins
 * are tests/golden/*.npz, produced by running the reference's own kernels (oracle/_ref,
 * compiled unmodified from the reference sources) on a GPU -- see tests/golden/make_golden.py.
 *
 * Citations are file:line under /root/reference/lib/utils/tf_ops/.
 */
#include <math.h>
#include <pthread.h>
#include <stdatomic.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>

/* ---- minimal pthread parallel-for (this image has no libgomp) -------------------------------- */
typedef void (*pf_body)(long i, void *ctx);
typedef struct { pf_body fn; void *ctx; long n; long chunk; atomic_long next; } pf_job;

static int g_threads = 0;
void oracle_set_threads(int t) { g_threads = t; }
int oracle_get_threads(void)
{
    if (g_threads > 0) return g_threads;
    const char *e = getenv("ORACLE_THREADS");
    if (e && atoi(e) > 0) return atoi(e);
    long nc = sysconf(_SC_NPROCESSORS_ONLN);
    return nc > 0 ? (int)nc : 1;
}
static void *pf_worker(void *p)
{
    pf_job *j = (pf_job *)p;
    for (;;) {
        long s = atomic_fetch_add(&j->next, j->chunk);
        if (s >= j->n) break;
        long e = s + j->chunk < j->n ? s + j->chunk : j->n;
        for (long i = s; i < e; i++) j->fn(i, j->ctx);
    }
    return NULL;
}
static void parallel_for(long n, long chunk, pf_body fn, void *ctx)
{
    int nt = oracle_get_threads();
    if (nt > n) nt = (int)(n > 0 ? n : 1);
    pf_job job;
    job.fn = fn; job.ctx = ctx; job.n = n; job.chunk = chunk > 0 ? chunk : 1;
    atomic_init(&job.next, 0);
    if (nt <= 1) { pf_worker(&job); return; }
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * nt);
    for (int t = 1; t < nt; t++) pthread_create(&th[t], NULL, pf_worker, &job);
    pf_worker(&job);
    for (int t = 1; t < nt; t++) pthread_join(th[t], NULL);
    free(th);
}

/* ---- farthest point sampling ------------------------------------------------------------------ */
#define REF_FPS_THREADS 1024 /* sampling/tf_sampling_g.cu:393 launches <<<b,1024>>> */

/* The block-wide arg-max of sampling/tf_sampling_g.cu:159-173: a left-biased binary tree
 * over the 1024 per-thread (best, besti) slots; slot i1 is replaced only when strictly
 * smaller than slot i2, so among equal maxima the lowest slot (thread id) survives. */
static int ref_tree_argmax(float *dists, int *dists_i)
{
    for (int u = 0; (1 << u) < REF_FPS_THREADS; u++) {
        int active = REF_FPS_THREADS >> (u + 1);
        for (int t = 0; t < active; t++) {
            int i1 = (t * 2) << u;
            int i2 = (t * 2 + 1) << u;
            if (dists[i1] < dists[i2]) {
                dists[i1] = dists[i2];
                dists_i[i1] = dists_i[i2];
            }
        }
    }
    return dists_i[0];
}

typedef struct { int n, c, m; const float *inp; float *temp; int *out; } fps_ctx;

/* farthest_point_sample: sampling/tf_sampling_g.cu:124-178 (kernel), :392-394 (launcher). */
static void fps_scene(long i, void *vp)
{
    fps_ctx *a = (fps_ctx *)vp;
    int n = a->n, c = a->c, m = a->m;
    const float *data = a->inp + (size_t)i * n * c;
    float *td = a->temp + (size_t)i * n;
    int *idxs = a->out + (size_t)i * m;
    float dists[REF_FPS_THREADS];
    int dists_i[REF_FPS_THREADS];
    int old = 0;
    idxs[0] = old;                                  /* :131-133 */
    for (int j = 0; j < n; j++) td[j] = 1e38f;      /* :135-137 */
    for (int j = 1; j < m; j++) {
        for (int t = 0; t < REF_FPS_THREADS; t++) { dists[t] = -1.0f; dists_i[t] = 0; } /* :140-141 */
        const float *p_old = data + (size_t)old * c;
        for (int k = 0; k < n; k++) {               /* thread t = k % 1024 scans its k ascending (:142) */
            int t = k & (REF_FPS_THREADS - 1);
            const float *p = data + (size_t)k * c;
            float d = 0.0f;
            for (int l = 0; l < c; l++) {           /* :146-150, contracted by nvcc to fma(diff,diff,d) */
                float diff = p[l] - p_old[l];
                d = fmaf(diff, diff, d);
            }
            float d2 = fminf(d, td[k]);             /* :151 */
            if (d2 != td[k]) td[k] = d2;            /* :152-153 */
            if (d2 > dists[t]) { dists[t] = d2; dists_i[t] = k; } /* :154-157, strict */
        }
        old = ref_tree_argmax(dists, dists_i);      /* :159-173 */
        idxs[j] = old;                              /* :174-175 */
    }
}

/* inp [b,n,c], out [b,m]; temp is [b,n] scratch, caller-allocated like the reference's
 * allocate_temp (sampling/tf_sampling.cpp:152-155). */
void oracle_farthest_point_sample(int b, int n, int c, int m, const float *inp, float *temp, int *out)
{
    if (m <= 0) return; /* :126-127 */
    fps_ctx a = { n, c, m, inp, temp, out };
    parallel_for(b, 1, fps_scene, &a);
}

/* farthest_point_sample_with_distance: sampling/tf_sampling_g.cu:181-230, launcher :396-398. */
static void fpsd_scene(long i, void *vp)
{
    fps_ctx *a = (fps_ctx *)vp;
    int n = a->n, m = a->m;
    const float *mat = a->inp + (size_t)i * n * n;
    float *td = a->temp + (size_t)i * n;
    int *idxs = a->out + (size_t)i * m;
    float dists[REF_FPS_THREADS];
    int dists_i[REF_FPS_THREADS];
    int old = 0;
    idxs[0] = old;
    for (int j = 0; j < n; j++) td[j] = 1e38f;
    for (int j = 1; j < m; j++) {
        for (int t = 0; t < REF_FPS_THREADS; t++) { dists[t] = -1.0f; dists_i[t] = 0; }
        const float *row = mat + (size_t)old * n;   /* :202 */
        for (int k = 0; k < n; k++) {
            int t = k & (REF_FPS_THREADS - 1);
            float d2 = fminf(row[k], td[k]);
            if (d2 != td[k]) td[k] = d2;
            if (d2 > dists[t]) { dists[t] = d2; dists_i[t] = k; }
        }
        old = ref_tree_argmax(dists, dists_i);
        idxs[j] = old;
    }
}

/* dist [b,n,n] precomputed, out [b,m]. */
void oracle_farthest_point_sample_with_distance(int b, int n, int m, const float *dist, float *temp, int *out)
{
    if (m <= 0) return;
    fps_ctx a = { n, 0, m, dist, temp, out };
    parallel_for(b, 1, fpsd_scene, &a);
}

/* ---- gather_point: sampling/tf_sampling_g.cu:320-331.  out[b,j,:] = inp[b,idx[b,j],:] ---------- */
typedef struct { int n, m, c; const float *inp; const int *idx; float *out; } gat_ctx;
static void gat_row(long r, void *vp)
{
    gat_ctx *a = (gat_ctx *)vp;
    long bi = r / a->m;
    int src = a->idx[r];
    memcpy(a->out + (size_t)r * a->c, a->inp + ((size_t)bi * a->n + src) * a->c, sizeof(float) * a->c);
}
void oracle_gather_point(int b, int n, int m, int c, const float *inp, const int *idx, float *out)
{
    gat_ctx a = { n, m, c, inp, idx, out };
    parallel_for((long)b * m, 256, gat_row, &a);
}

/* ---- ball query ------------------------------------------------------------------------------- */
/* Distance recipe shared by ball query and three_nn (PTX of grouping/tf_grouping_g.cu:243 and
 * interpolation/tf_interpolate_g.cu:54): t = dy*dy ; t = fma(dx,dx,t) ; t = fma(dz,dz,t). */
static inline float ref_sqdist(float x2, float y2, float z2, float x1, float y1, float z1)
{
    float dx = x2 - x1, dy = y2 - y1, dz = z2 - z1;
    float t = dy * dy;
    t = fmaf(dx, dx, t);
    t = fmaf(dz, dz, t);
    return t;
}

typedef struct {
    int n, m, nsample, dilated;
    float r0, r1;
    const float *xyz1, *xyz2;
    int *idx, *cnt;
} bq_ctx;

/* query_ball_point: grouping/tf_grouping_g.cu:215-255; _dilated: :308-357.
 * Rows with no hit are left untouched by the reference (uninitialised memory); the oracle
 * zero-fills them, and callers compare idx*(cnt>0) exactly as lib/utils/layers_util.py:157-159 does. */
static void bq_query(long q, void *vp)
{
    bq_ctx *a = (bq_ctx *)vp;
    int n = a->n, ns = a->nsample;
    long bi = q / a->m;
    const float *p1 = a->xyz1 + (size_t)bi * n * 3;
    const float *p2 = a->xyz2 + (size_t)q * 3;
    int *cur = a->idx + (size_t)q * ns;
    for (int l = 0; l < ns; l++) cur[l] = 0;
    float x2 = p2[0], y2 = p2[1], z2 = p2[2];
    int cnt = 0;
    for (int k = 0; k < n; k++) {
        if (cnt == ns) break;                                            /* :238-239 / :331-332 */
        float t = ref_sqdist(x2, y2, z2, p1[k * 3], p1[k * 3 + 1], p1[k * 3 + 2]);
        int hit;
        if (a->dilated) {
            float d = sqrtf(t);                                          /* :336 */
            hit = (d == 0.0f) || (d >= a->r0 && d < a->r1);              /* :337,:346 */
        } else {
            float d = fmaxf(sqrtf(t), 1e-20f);                           /* :243 (max.f32: NaN -> 1e-20) */
            hit = d < a->r1;
        }
        if (hit) {
            if (cnt == 0) for (int l = 0; l < ns; l++) cur[l] = k;       /* :245-248 */
            cur[cnt] = k;
            cnt++;
        }
    }
    a->cnt[q] = cnt;
}
void oracle_query_ball_point(int b, int n, int m, float radius, int nsample,
                             const float *xyz1, const float *xyz2, int *idx, int *pts_cnt)
{
    bq_ctx a = { n, m, nsample, 0, 0.0f, radius, xyz1, xyz2, idx, pts_cnt };
    parallel_for((long)b * m, 16, bq_query, &a);
}
void oracle_query_ball_point_dilated(int b, int n, int m, float min_radius, float max_radius, int nsample,
                                     const float *xyz1, const float *xyz2, int *idx, int *pts_cnt)
{
    bq_ctx a = { n, m, nsample, 1, min_radius, max_radius, xyz1, xyz2, idx, pts_cnt };
    parallel_for((long)b * m, 16, bq_query, &a);
}

/* ---- group_point: grouping/tf_grouping_g.cu:362-379 ------------------------------------------- */
typedef struct { int n, c, m, ns; const float *points; const int *idx; float *out; } grp_ctx;
static void grp_row(long r, void *vp)
{
    grp_ctx *a = (grp_ctx *)vp;
    long bi = r / ((long)a->m * a->ns);
    int src = a->idx[r];
    float *o = a->out + (size_t)r * a->c;
    if (src == -1) memset(o, 0, sizeof(float) * a->c);                   /* :373-374 */
    else memcpy(o, a->points + ((size_t)bi * a->n + src) * a->c, sizeof(float) * a->c);
}
void oracle_group_point(int b, int n, int c, int m, int nsample, const float *points, const int *idx, float *out)
{
    grp_ctx a = { n, c, m, nsample, points, idx, out };
    parallel_for((long)b * m * nsample, 256, grp_row, &a);
}

/* ---- three_nn: interpolation/tf_interpolate_g.cu:24-84 (== CPU kernel tf_interpolate.cpp:86-129) */
typedef struct { int n, m; const float *xyz1, *xyz2; float *dist; int *idx; } tnn_ctx;
static void tnn_point(long q, void *vp)
{
    tnn_ctx *a = (tnn_ctx *)vp;
    long bi = q / a->n;
    const float *u = a->xyz1 + (size_t)q * 3;
    const float *kn = a->xyz2 + (size_t)bi * a->m * 3;
    double best1 = 1e40, best2 = 1e40, best3 = 1e40;                     /* :41-43 */
    int i1 = 0, i2 = 0, i3 = 0;
    for (int i = 0; i < a->m; i++) {
        /* fp32 squared distance, widened to double only for the comparisons (:54, PTX cvt.f64.f32) */
        double d = (double)ref_sqdist(kn[i * 3], kn[i * 3 + 1], kn[i * 3 + 2], u[0], u[1], u[2]);
        if (d < best1) { best3 = best2; i3 = i2; best2 = best1; i2 = i1; best1 = d; i1 = i; }
        else if (d < best2) { best3 = best2; i3 = i2; best2 = d; i2 = i; }
        else if (d < best3) { best3 = d; i3 = i; }
    }
    a->dist[q * 3 + 0] = (float)best1; a->dist[q * 3 + 1] = (float)best2; a->dist[q * 3 + 2] = (float)best3;
    a->idx[q * 3 + 0] = i1; a->idx[q * 3 + 1] = i2; a->idx[q * 3 + 2] = i3;
}
void oracle_three_nn(int b, int n, int m, const float *xyz1, const float *xyz2, float *dist, int *idx)
{
    tnn_ctx a = { n, m, xyz1, xyz2, dist, idx };
    parallel_for((long)b * n, 16, tnn_point, &a);
}

/* ---- three_interpolate: interpolation/tf_interpolate_g.cu:87-113 -------------------------------
 * PTX: t = w2*c2 ; t = fma(w1,c1,t) ; out = fma(w3,c3,t). */
typedef struct { int m, c, n; const float *points; const int *idx; const float *w; float *out; } tin_ctx;
static void tin_point(long q, void *vp)
{
    tin_ctx *a = (tin_ctx *)vp;
    long bi = q / a->n;
    int c = a->c;
    const float *pts = a->points + (size_t)bi * a->m * c;
    const int *id = a->idx + q * 3;
    const float *w = a->w + q * 3;
    for (int ch = 0; ch < c; ch++) {
        float c1 = pts[(size_t)id[0] * c + ch], c2 = pts[(size_t)id[1] * c + ch], c3 = pts[(size_t)id[2] * c + ch];
        float t = w[1] * c2;
        t = fmaf(w[0], c1, t);
        a->out[(size_t)q * c + ch] = fmaf(w[2], c3, t);
    }
}
void oracle_three_interpolate(int b, int m, int c, int n, const float *points, const int *idx,
                              const float *weight, float *out)
{
    tin_ctx a = { m, c, n, points, idx, weight, out };
    parallel_for((long)b * n, 64, tin_point, &a);
}

/* ---- calc_square_dist(a, a, norm=False): lib/utils/model_util.py:144-160 ------------------------
 * The reference evaluates |a|^2 + |b|^2 - 2 a.b^T with a TF-1.4 cuBLAS SGEMM whose summation order
 * is not reproducible; this restatement (and the product kernel) pin the order: sq[i] and dot[i,j]
 * are sequential fmaf() chains over the channel index starting from 0, out = (sq[i]+sq[j]) - 2*dot. */
typedef struct { int n, c; const float *a; float *sq; float *out; } csd_ctx;
static void csd_sq(long r, void *vp)
{
    csd_ctx *a = (csd_ctx *)vp;
    const float *x = a->a + (size_t)r * a->c;
    float s = 0.0f;
    for (int l = 0; l < a->c; l++) s = fmaf(x[l], x[l], s);
    a->sq[r] = s;
}
static void csd_row(long r, void *vp)
{
    csd_ctx *a = (csd_ctx *)vp;
    int n = a->n, c = a->c;
    long bi = r / n;
    const float *A = a->a + (size_t)bi * n * c;
    const float *xi = a->a + (size_t)r * c;
    const float *sq = a->sq + (size_t)bi * n;
    float si = a->sq[r];
    float *o = a->out + (size_t)r * n;
    for (int j = 0; j < n; j++) {
        const float *xj = A + (size_t)j * c;
        float dot = 0.0f;
        for (int l = 0; l < c; l++) dot = fmaf(xi[l], xj[l], dot);
        o[j] = (si + sq[j]) - 2.0f * dot;
    }
}
void oracle_calc_square_dist(int b, int n, int c, const float *a, float *out)
{
    csd_ctx x = { n, c, a, (float *)malloc(sizeof(float) * (size_t)b * n), out };
    parallel_for((long)b * n, 256, csd_sq, &x);
    parallel_for((long)b * n, 4, csd_row, &x);
    free(x.sq);
}

/* ---- conv(1x1)+BN+ReLU: lib/utils/tf_util.py:127-201 (conv2d), :51-124 (conv1d), :424-444 (BN) ---
 * Inference BN with moving statistics and tf.contrib.layers.batch_norm's default eps=0.001:
 *   y = relu( ((x.W + bias) - mean) * gamma * rsqrt(var + eps) + beta )
 * evaluated in double and rounded once: a TOLERANCE oracle (<=1e-3 relative), not a bit-exact one,
 * because the reference's SGEMM summation order is unspecified.  x [rows,cin]; w [cin,cout] (the TF
 * kernel layout [1,1,cin,cout]); gamma==NULL disables BN. */
typedef struct {
    int cin, cout, relu;
    const float *x, *w, *bias, *gamma, *beta, *mean, *var;
    float *y;
} lin_ctx;
static void lin_row(long r, void *vp)
{
    lin_ctx *a = (lin_ctx *)vp;
    int cin = a->cin, cout = a->cout;
    const float *xr = a->x + (size_t)r * cin;
    double acc[2048];
    double *ac = cout <= 2048 ? acc : (double *)malloc(sizeof(double) * cout);
    for (int o = 0; o < cout; o++) ac[o] = 0.0;
    for (int k = 0; k < cin; k++) {
        double xv = xr[k];
        const float *wk = a->w + (size_t)k * cout;
        for (int o = 0; o < cout; o++) ac[o] += xv * (double)wk[o];
    }
    for (int o = 0; o < cout; o++) {
        double v = ac[o] + (a->bias ? (double)a->bias[o] : 0.0);
        if (a->gamma)
            v = (v - (double)a->mean[o]) * ((double)a->gamma[o] / sqrt((double)a->var[o] + 0.001)) + (double)a->beta[o];
        if (a->relu && v < 0.0) v = 0.0;
        a->y[(size_t)r * cout + o] = (float)v;
    }
    if (ac != acc) free(ac);
}
void oracle_linear_bn_relu(long rows, int cin, int cout, const float *x, const float *w, const float *bias,
                           const float *gamma, const float *beta, const float *mean, const float *var,
                           int relu, float *y)
{
    lin_ctx a = { cin, cout, relu, x, w, bias, gamma, beta, mean, var, y };
    parallel_for(rows, 8, lin_row, &a);
}

int oracle_version(void) { return 1; }

/* ---- backward ops (row f3): sampling/tf_sampling_g.cu:335-346, grouping/tf_grouping_g.cu:383-398,
 *      interpolation/tf_interpolate_g.cu:115-140.  Sequential double-precision accumulation (the GPU kernels use
 *      fp32 atomics whose order is not fixed): tolerance oracle. */
void oracle_scatter_add_rows(long rows, long rows_per_scene, int n, int c, const float *src, const int *idx, float *dst,
                             long dst_elems, int skip_neg)
{
    double *acc = (double *)calloc((size_t)dst_elems, sizeof(double));
    for (long r = 0; r < rows; r++) {
        int a = idx[r];
        if (skip_neg && a == -1) continue;
        long scene = r / rows_per_scene;
        for (int ch = 0; ch < c; ch++) acc[((size_t)scene * n + a) * c + ch] += (double)src[(size_t)r * c + ch];
    }
    for (long i = 0; i < dst_elems; i++) dst[i] = (float)acc[i];
    free(acc);
}

void oracle_three_interpolate_grad(int b, int n, int c, int m, const float *grad_out, const int *idx, const float *weight,
                                   float *grad_points)
{
    size_t total = (size_t)b * m * c;
    double *acc = (double *)calloc(total, sizeof(double));
    for (long q = 0; q < (long)b * n; q++) {
        long bi = q / n;
        for (int k = 0; k < 3; k++) {
            size_t base = ((size_t)bi * m + idx[q * 3 + k]) * c;
            for (int ch = 0; ch < c; ch++) acc[base + ch] += (double)(grad_out[(size_t)q * c + ch] * weight[q * 3 + k]);
        }
    }
    for (size_t i = 0; i < total; i++) grad_points[i] = (float)acc[i];
    free(acc);
}

/* ---- greedy BEV NMS (C twin of oracle/head.py:bev_nms; TensorFlow's non_max_suppression semantics) ----------------
 * Follows /root/reference/lib/builder/postprocessor.py:76-88 with lib/utils/box_3d_utils.py:25-58 (box_3d_to_anchor)
 * and lib/utils/anchors_util.py:11-48 (project_to_bev): candidates in descending score order (ties: lower index), a
 * candidate is dropped when its axis-aligned BEV IoU with a kept box is > thr, at most max_out kept.  Used by the
 * `--impl reference` arm of bench.py (the reference runs this stage on the CPU) and by the CPU baseline.
 * Arithmetic: the recipe of DESIGN.md §3.5, shared with csrc/nms.cu and oracle/head.py -- cos / sin in double rounded
 * once to float, every product and sum rounded (the library is built with -ffp-contract=off).  The comparator treats
 * -0 and +0 as equal; NaN scores are outside the contract (it is not a consistent order on them). */
typedef struct { float s; int i; } nms_key;
static int nms_cmp(const void *a, const void *b)
{
    const nms_key *x = (const nms_key *)a, *y = (const nms_key *)b;
    if (x->s > y->s) return -1;
    if (x->s < y->s) return 1;
    return x->i - y->i;
}
void oracle_bev_nms(int b, int n, const float *boxes, const float *scores, float thr, int max_out, int cls_id,
                    float *out_block, int *out_cnt)
{
    nms_key *keys = (nms_key *)malloc(sizeof(nms_key) * (size_t)(n > 0 ? n : 1));
    float *rect = (float *)malloc(sizeof(float) * 5 * (size_t)(n > 0 ? n : 1));
    int *kept = (int *)malloc(sizeof(int) * (size_t)(max_out > 0 ? max_out : 1));
    for (int s = 0; s < b; s++) {
        const float *bx = boxes + (size_t)s * n * 7, *sc = scores + (size_t)s * n;
        float *blk = out_block + (size_t)s * max_out * 9;
        memset(blk, 0, sizeof(float) * (size_t)max_out * 9);
        for (int i = 0; i < n; i++) {
            const double ry = (double)bx[i * 7 + 6];
            const float c = fabsf((float)cos(ry)), sn = fabsf((float)sin(ry));
            const float dimx = bx[i * 7 + 3] * c + bx[i * 7 + 5] * sn, dimz = bx[i * 7 + 5] * c + bx[i * 7 + 3] * sn;
            rect[i * 5 + 0] = bx[i * 7 + 0] - dimx * 0.5f; rect[i * 5 + 1] = bx[i * 7 + 2] - dimz * 0.5f;
            rect[i * 5 + 2] = bx[i * 7 + 0] + dimx * 0.5f; rect[i * 5 + 3] = bx[i * 7 + 2] + dimz * 0.5f;
            rect[i * 5 + 4] = (rect[i * 5 + 2] - rect[i * 5 + 0]) * (rect[i * 5 + 3] - rect[i * 5 + 1]);
            keys[i].s = sc[i]; keys[i].i = i;
        }
        qsort(keys, (size_t)n, sizeof(nms_key), nms_cmp);
        int nk = 0;
        for (int t = 0; t < n && nk < max_out; t++) {
            const int i = keys[t].i;
            int ok = 1;
            for (int u = 0; u < nk && ok; u++) {
                const int j = kept[u];
                if (rect[i * 5 + 4] <= 0 || rect[j * 5 + 4] <= 0) continue;
                float iw = fminf(rect[i * 5 + 2], rect[j * 5 + 2]) - fmaxf(rect[i * 5 + 0], rect[j * 5 + 0]);
                float ih = fminf(rect[i * 5 + 3], rect[j * 5 + 3]) - fmaxf(rect[i * 5 + 1], rect[j * 5 + 1]);
                iw = iw > 0 ? iw : 0; ih = ih > 0 ? ih : 0;
                const float inter = iw * ih;
                if (inter / ((rect[i * 5 + 4] + rect[j * 5 + 4]) - inter) > thr) ok = 0;
            }
            if (ok) kept[nk++] = i;
        }
        for (int u = 0; u < nk; u++) {
            for (int e = 0; e < 7; e++) blk[u * 9 + e] = bx[kept[u] * 7 + e];
            blk[u * 9 + 7] = sc[kept[u]];
            blk[u * 9 + 8] = (float)cls_id;
        }
        out_cnt[s] = nk;
    }
    free(keys); free(rect); free(kept);
}
