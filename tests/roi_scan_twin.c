/* C twin of the region pool's membership scan (3dssd_b200/csrc/roi_pool.cu, point_inside_box_3d of the reference's
 * tf_grouping_g.cu:27-94) for tests/test_pointrcnn_rcnn_cpu.py.  Built with -ffp-contract=off, so every operation
 * rounds on its own and the fused multiply-adds are the explicit fma / fmaf calls the device code makes.  glibc's cosf
 * / sinf are not CUDA's: within a few ulp of a face the twin and the device may legitimately differ.
 *
 *   roi_scan(n, xyz[n*3], m, boxes[m*7], nsample, idx[m*nsample], cnt[m])
 */
#include <math.h>

static int inside(float x, float y, float z, float cx, float by, float cz, float h, float c, float s, float maxd,
                  double hl, double hw)
{
    const float dx = x - cx, dz = z - cz;
    if (fabsf(dx) > maxd || y > by || by - y > h || fabsf(dz) > maxd) return 0;
    const double u = (double)fmaf(dx, c, -(dz * s));
    const double v = (double)fmaf(dz, c, dx * s);
    return u >= -hl && u <= hl && v >= -hw && v <= hw;
}

void roi_scan(int n, const float *xyz, int m, const float *boxes, int nsample, int *idx, int *cnt)
{
    for (int r = 0; r < m; r++) {
        const float *b = boxes + (long)r * 7;
        const double hl = (double)b[3] * 0.5, hw = (double)b[5] * 0.5;
        const float maxd = fmaxf(sqrtf((float)fma(hl, hl, hw * hw)), 1e-20f);
        const float c = cosf(b[6]), s = sinf(b[6]);
        int *o = idx + (long)r * nsample, k = 0;
        for (int p = 0; p < n && k < nsample; p++)
            if (inside(xyz[3 * p], xyz[3 * p + 1], xyz[3 * p + 2], b[0], b[1], b[2], b[4], c, s, maxd, hl, hw)) o[k++] = p;
        for (int q = k; q < nsample; q++) o[q] = k ? o[0] : 0;
        cnt[r] = k;
    }
}
