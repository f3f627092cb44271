/* ffps_prune_model.c -- TEST INFRASTRUCTURE ONLY (like everything under oracle/).
 *
 * CPU model of the skip rule of the PRODUCT's pruned F-FPS, ffps_bucket_kernel (3dssd_b200/csrc/fps_bucket.cu), for
 * tests/test_ffps_bucket_cpu.py and tools/fps_prune_stats.py.  One scene of n <= 4096 points with c <= 68 channels (row-major [n][c]) runs the
 * F-FPS with the kernel's fp32 arithmetic: sqdist's pinned chains for the value (sq_w + sq_x) - 2 dot(w, x), 3-D Morton
 * buckets of 32 points with mean-row centres, and the kernel's skip test.  Every round it also computes the value of
 * every point of every SKIPPED bucket and counts the points whose value is below their running distance: a skip that
 * would have changed a result.  with_margin = 0 drops the rounding margin E from the test.
 * Returns the number of such points; idx[m] receives the sampled indices (skipped buckets left as they are). */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define CP 68
#define BS 32

static uint32_t spread10(uint32_t v)
{
    v &= 0x3ffu;
    v = (v | (v << 16)) & 0x030000ffu;
    v = (v | (v << 8)) & 0x0300f00fu;
    v = (v | (v << 4)) & 0x030c30c3u;
    v = (v | (v << 2)) & 0x09249249u;
    return v;
}

static int cmp_u64(const void *a, const void *b)
{
    const uint64_t x = *(const uint64_t *)a, y = *(const uint64_t *)b;
    return x < y ? -1 : (x > y ? 1 : 0);
}

static float value(const float *w, float sw, const float *x, float sx)
{
    float dot = 0.0f;
    for (int l = 0; l < CP; l++) dot = fmaf(w[l], x[l], dot);
    return (sw + sx) - 2.0f * dot;
}

long long oracle_ffps_prune_model(int n, int c, int m, const float *data, int with_margin, int *idx, long long *touched)
{
    if (n < 1 || n > 4096 || c < 3 || c > CP) return -1;
    const int nb = (n + BS - 1) / BS;
    float *rows = calloc((size_t)n * CP, sizeof(float)), *sq = malloc(sizeof(float) * n), *td = malloc(sizeof(float) * n);
    float *cen = calloc((size_t)nb * CP, sizeof(float)), *rho = malloc(sizeof(float) * nb), *sqm = malloc(sizeof(float) * nb);
    uint64_t *key = malloc(sizeof(uint64_t) * n);
    int *ord = malloc(sizeof(int) * n);
    for (int k = 0; k < n; k++)
        for (int l = 0; l < c; l++) rows[(size_t)k * CP + l] = data[(size_t)k * c + l];
    float lo[3] = {3.0e38f, 3.0e38f, 3.0e38f}, hi[3] = {-3.0e38f, -3.0e38f, -3.0e38f}, ext = 0.0f;
    for (int k = 0; k < n; k++)
        for (int a = 0; a < 3; a++) { lo[a] = fminf(lo[a], rows[k * CP + a]); hi[a] = fmaxf(hi[a], rows[k * CP + a]); }
    for (int a = 0; a < 3; a++) ext = fmaxf(ext, hi[a] - lo[a]);
    const float scale = ext > 0.0f ? 1023.999f / ext : 0.0f;
    for (int k = 0; k < n; k++) {
        uint32_t mc = 0;
        for (int a = 0; a < 3; a++) {
            int q = (int)((rows[k * CP + a] - lo[a]) * scale);
            q = q < 0 ? 0 : (q > 1023 ? 1023 : q);
            mc |= spread10((uint32_t)q) << a;
        }
        key[k] = ((uint64_t)mc << 12) | (uint64_t)k;
    }
    qsort(key, (size_t)n, sizeof(uint64_t), cmp_u64);
    for (int q = 0; q < n; q++) ord[q] = (int)(key[q] & 4095u);
    for (int k = 0; k < n; k++) {
        float s2 = 0.0f;
        for (int l = 0; l < CP; l++) s2 = fmaf(rows[k * CP + l], rows[k * CP + l], s2);
        sq[k] = s2;
        td[k] = 1e38f;
    }
    for (int b = 0; b < nb; b++) {
        const int q0 = b * BS, q1 = q0 + BS < n ? q0 + BS : n;
        float r2max = 0.0f, sm = 0.0f;
        for (int l = 0; l < CP; l++) {
            float acc = 0.0f;
            for (int q = q0; q < q1; q++) acc += rows[ord[q] * CP + l];
            cen[b * CP + l] = acc / (float)(q1 - q0);
        }
        for (int q = q0; q < q1; q++) {
            float r2 = 0.0f;
            for (int l = 0; l < CP; l++) { const float d = rows[ord[q] * CP + l] - cen[b * CP + l]; r2 = fmaf(d, d, r2); }
            r2max = fmaxf(r2max, r2);
            sm = fmaxf(sm, sq[ord[q]]);
        }
        rho[b] = sqrtf(r2max * 1.0001f + 1e-36f) * 1.0001f;
        sqm[b] = sm;
    }
    long long bad = 0, tch = 0;
    int old = 0;
    idx[0] = 0;
    for (int j = 1; j < m; j++) {
        const float *w = rows + (size_t)old * CP;
        const float so = sq[old];
        for (int b = 0; b < nb; b++) {
            const int q0 = b * BS, q1 = q0 + BS < n ? q0 + BS : n;
            float dc2 = 0.0f, bmax = 0.0f;
            for (int l = 0; l < CP; l++) { const float d = w[l] - cen[b * CP + l]; dc2 = fmaf(d, d, dc2); }
            for (int q = q0; q < q1; q++) bmax = fmaxf(bmax, td[ord[q]]);
            const float dc_lo = sqrtf(fmaxf(dc2 * 0.9999f - 1e-36f, 0.0f)) * 0.9999f;
            const float g = fmaxf(dc_lo - rho[b], 0.0f);
            const float e = with_margin ? 8.4e-6f * (so + sqm[b]) + 1e-36f : 0.0f;
            const int skip = g * g * 0.9999f - e >= bmax;
            tch += !skip;
            for (int q = q0; q < q1; q++) {
                const int k = ord[q];
                const float v = value(w, so, rows + (size_t)k * CP, sq[k]);
                if (skip) bad += v < td[k];
                else td[k] = fminf(v, td[k]);
            }
        }
        /* arg-max: value desc, then (k mod 1024, k div 1024) asc; negative values never win (fps_candidate) */
        int best = -1;
        uint32_t bv = 0u, bk = 0x7FFFFFFFu;
        for (int k = 0; k < n; k++) {
            if (!(td[k] >= 0.0f)) continue;
            uint32_t u;
            memcpy(&u, &td[k], 4);
            const uint32_t kk = ((uint32_t)(k & 1023) << 21) | (uint32_t)(k >> 10);
            if (best < 0 || u > bv || (u == bv && kk < bk)) { best = k; bv = u; bk = kk; }
        }
        old = best < 0 ? 0 : best;
        idx[j] = old;
    }
    if (touched) *touched = tch;
    free(rows); free(sq); free(td); free(cen); free(rho); free(sqm); free(key); free(ord);
    return bad;
}
