// det_loss.cu -- training targets and detection losses of the shipped 3DSSD configuration (DESIGN.md section 3.8):
//   det_assign       'Mask' target assignment + vote targets, one CTA per scene
//                    (lib/np_functions/gt_sampler.py:168-259 and :28-61, lib/utils/voxelnet_aug.py:318-342, :532-567,
//                    the centre-ness label of lib/builder/loss_builder.py:99-137, encode_angle2class and
//                    encode_dist_anchor_free of lib/utils/anchor_encoder.py)
//   det_loss         the six losses of LossBuilder.forward (loss_builder.py) for 'Center-ness' sigmoid classification,
//                    'Dist-Anchor-free' regression, the corner loss and the vote loss: per-scene partial sums in double,
//                    then one fixed-order sum over the scenes
//   det_loss_grad    their gradients w.r.t. the head outputs, the candidate points and the raw vote offsets
// No float atomics anywhere: every run gives the same bits.
#include <math.h>

#include "box_geom.cuh"

namespace ssd3d {

constexpr int kDetThreads = 256;
constexpr int kBoxTile = 64;          // GT boxes staged in shared memory per round
constexpr int kMaxBins = 32;
constexpr float kExpand = 0.1f;       // TRAIN.AUGMENTATIONS.EXPAND_DIMS_LENGTH (lib/core/config.py:84)
constexpr float kSampleRange = 10.0f; // CLASSIFICATION_LOSS.SOFTMAX_SAMPLE_RANGE (configs/kitti/3dssd/3dssd.yaml:80)
constexpr double kCtrEps = 1e-6;      // epsilon of _generate_centerness_label (loss_builder.py:99)

// encode_angle2class_tf (anchor_encoder.py:21-33) in float32, tf.mod / np.mod being a floor-mod
__device__ __forceinline__ float floor_mod(float a, float b)
{
    float m = fmodf(a, b);                       // exact
    if (m != 0.0f && (m < 0.0f) != (b < 0.0f)) m = __fadd_rn(m, b);
    return m;
}

__device__ __forceinline__ void encode_angle(float ry, int nbins, int &bin, float &res)
{
    const float two_pi = (float)(2.0 * M_PI);
    const float per = (float)(2.0 * M_PI / nbins), half = (float)(2.0 * M_PI / nbins / 2.0);
    const float a = floor_mod(ry, two_pi);
    const float sh = floor_mod(__fadd_rn(a, half), two_pi);
    const float cf = floorf(__fdiv_rn(sh, per));
    bin = min((int)cf, nbins - 1);               // a shift that rounds up to 2*pi would name bin nbins
    res = __fdiv_rn(__fsub_rn(sh, __fadd_rn(__fmul_rn(cf, per), half)), per);
}

// encode_dist_anchor_free (anchor_encoder.py:151-173) in float32: box centre moved up by h/2 minus the point, then half sizes
__device__ __forceinline__ void encode_offset(const float *bx, const float *t, float *o)
{
    const float hh = __fmul_rn(bx[4], 0.5f);
    o[0] = __fsub_rn(bx[0], t[0]);
    o[1] = __fsub_rn(__fsub_rn(bx[1], hh), t[1]);
    o[2] = __fsub_rn(bx[2], t[2]);
    o[3] = __fmul_rn(bx[3], 0.5f);
    o[4] = hh;
    o[5] = __fmul_rn(bx[5], 0.5f);
}

__device__ __forceinline__ bool box_valid(const float *b)
{
    return b[0] != 0.f || b[1] != 0.f || b[2] != 0.f || b[3] != 0.f || b[4] != 0.f || b[5] != 0.f || b[6] != 0.f;
}

__global__ void __launch_bounds__(kDetThreads) det_assign_kernel(
    int n, int nv, int g, int nbins, const float *__restrict__ base, const float *__restrict__ vbase,
    const float *__restrict__ boxes, const int *__restrict__ labels, int *__restrict__ a_idx, float *__restrict__ a_box,
    float *__restrict__ pmask, float *__restrict__ nmask, float *__restrict__ cls_label, int *__restrict__ a_bin,
    float *__restrict__ a_res, float *__restrict__ off_t, float *__restrict__ vmask, float *__restrict__ vtarget)
{
    __shared__ Planes sp[kBoxTile], se[kBoxTile];
    __shared__ unsigned char sv[kBoxTile];
    const int s = blockIdx.x;
    const float *gb = boxes + (size_t)s * g * 7;
    const int npts = max(n, nv);
    for (int p0 = 0; p0 < npts; p0 += kDetThreads) {
        const int p = p0 + threadIdx.x;
        float q[3] = {0.f, 0.f, 0.f}, w[3] = {0.f, 0.f, 0.f};
        if (p < n) { const float *t = base + ((size_t)s * n + p) * 3; q[0] = t[0]; q[1] = t[2]; q[2] = t[1]; }
        if (p < nv) { const float *t = vbase + ((size_t)s * nv + p) * 3; w[0] = t[0]; w[1] = t[2]; w[2] = t[1]; }
        int first = -1, hit = -1, vhit = -1;
        for (int j0 = 0; j0 < g; j0 += kBoxTile) {
            const int tn = min(kBoxTile, g - j0);
            __syncthreads();
            for (int j = threadIdx.x; j < tn; j += blockDim.x) {
                const float *b = gb + (size_t)(j0 + j) * 7;
                const bool v = box_valid(b);
                sv[j] = v;
                if (v) {
                    double sd, cd;
                    sincos((double)b[6], &sd, &cd);
                    box_planes(b, 0.0f, (float)sd, (float)cd, sp[j]);
                    box_planes(b, kExpand, (float)sd, (float)cd, se[j]);
                }
            }
            __syncthreads();
            for (int j = 0; j < tn; j++) {
                if (!sv[j]) continue;                                           // padded rows (gt_sampler.py:199-201)
                if (first < 0) first = j0 + j;
                if (p < n && hit < 0 && inside(sp[j], q[0], q[1], q[2])) hit = j0 + j;
                if (p < nv && vhit < 0 && inside(se[j], w[0], w[1], w[2])) vhit = j0 + j;
            }
        }
        if (p < n) {
            const size_t r = (size_t)s * n + p;
            const int a = hit >= 0 ? hit : first;                              // np.argmax: first box that holds it
            float bx[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
            if (a >= 0)
                for (int k = 0; k < 7; k++) bx[k] = gb[(size_t)a * 7 + k];
            const float *t = base + r * 3;
            const float dx = __fsub_rn(t[0], bx[0]), dy = __fsub_rn(t[1], bx[1]), dz = __fsub_rn(t[2], bx[2]);
            const float dist = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
            const bool pos = hit >= 0 && dist <= kSampleRange;
            float label = 0.f;
            if (pos && labels[(size_t)s * g + a] == 1) {                       // one_hot(label - 1) of the one class
                // centre-ness (loss_builder.py:99-137) in double, rounded once
                const double ry = bx[6], c = cos(ry), sn = sin(ry);
                const double ex = (double)t[0] - bx[0], ey = (double)t[1] - bx[1], ez = (double)t[2] - bx[2];
                const double cx = c * ex - sn * ez, cy = ey, cz = sn * ex + c * ez;       // rotate_points(p, -ry)
                const double l2 = bx[3] / 2.0, h = bx[4], w2 = bx[5] / 2.0;
                const double fr = l2 - cx, bk = cx + l2, bo = -cy, tp = cy + h, le = w2 - cz, ri = cz + w2;
                const double cl = fmin(fr, bk) / fmax(fr, bk), cw = fmin(le, ri) / fmax(le, ri), ch = fmin(bo, tp) / fmax(bo, tp);
                label = (float)pow(fmax(cl * ch * cw, kCtrEps), 1.0 / 3.0);
            }
            int bin = 0;
            float res = 0.f;
            if (a >= 0) encode_angle(bx[6], nbins, bin, res);
            a_idx[r] = a >= 0 ? a : 0;
            for (int k = 0; k < 7; k++) a_box[r * 7 + k] = bx[k];
            pmask[r] = pos ? 1.f : 0.f;
            nmask[r] = hit < 0 ? 1.f : 0.f;
            cls_label[r] = label;
            a_bin[r] = bin;
            a_res[r] = res;
            float *o = off_t + r * 6;
            encode_offset(bx, t, o);
            if (a < 0) o[0] = o[1] = o[2] = 0.f;
        }
        if (p < nv) {
            const size_t r = (size_t)s * nv + p;
            const int a = vhit >= 0 ? vhit : first;
            const float *t = vbase + r * 3;
            float *o = vtarget + r * 3;
            vmask[r] = vhit >= 0 ? 1.f : 0.f;
            if (a >= 0) {                                                      // vote_targets_np (gt_sampler.py:55-57)
                const float *b = gb + (size_t)a * 7;
                o[0] = __fsub_rn(b[0], t[0]);
                o[1] = __fsub_rn(__fsub_rn(b[1], __fdiv_rn(b[4], 2.0f)), t[1]);
                o[2] = __fsub_rn(b[2], t[2]);
            } else {
                o[0] = o[1] = o[2] = 0.f;
            }
        }
    }
}

// ---- losses ----------------------------------------------------------------------------------------------------

struct LossIn {
    const float *base, *cls, *off, *acls, *ares, *vote;
    int ld_cls, ld_off, ld_acls, ld_ares, ld_vote;
    const float *box, *pmask, *nmask, *label, *res, *vmask, *vtarget;
    const int *bin;
};

// the regression target of a point from its assigned box and the live base_xyz, so that the loss is a function of the
// points it differentiates: the bits of det_assign's offset_target for the same points (pmask 0 where they differ)
__device__ __forceinline__ void target_of(const LossIn &in, size_t r, float *t)
{
    const float *bx = in.box + r * 7;
    encode_offset(bx, in.base + r * 3, t);
}

__device__ __forceinline__ double huber(double e)
{
    const double a = fabs(e), q = fmin(a, 1.0);
    return 0.5 * q * q + (a - q);
}
__device__ __forceinline__ double huber_grad(double e) { return fmin(fmax(e, -1.0), 1.0); }

__device__ __forceinline__ void corners8(double cx, double cy, double cz, double l, double h, double w, double c, double s,
                                         double X[8][3])
{
    const double sx[8] = {1, 1, -1, -1, 1, 1, -1, -1}, sz[8] = {1, -1, -1, 1, 1, -1, -1, 1};
#pragma unroll
    for (int i = 0; i < 8; i++) {                              // get_box3d_corners_helper (box_3d_utils.py:89-119)
        const double xc = sx[i] * l / 2.0, yc = i >= 4 ? -h : 0.0, zc = sz[i] * w / 2.0;
        X[i][0] = c * xc + s * zc + cx;
        X[i][1] = yc + cy;
        X[i][2] = -s * xc + c * zc + cz;
    }
}

// The box decode_dist_anchor_free makes from the offsets with the GT bin (single_stage_detector.py:173-177,
// anchor_decoder.py:86-112); lhw = max(2 * half, 0.1) in float32 as TF compares it, ties routed to 2 * half.
struct PredBox {
    double c[3], lhw[3], ang;
    bool pass[3];
};
__device__ __forceinline__ PredBox pred_box(const float *bx3, const float *o, float res, int bin, double interval)
{
    PredBox P;
    P.c[0] = (double)bx3[0] + o[0];
    P.c[1] = (double)bx3[1] + o[1] + o[4];
    P.c[2] = (double)bx3[2] + o[2];
    for (int k = 0; k < 3; k++) {
        const float two = __fmul_rn(o[3 + k], 2.0f);
        P.pass[k] = two >= 0.1f;
        P.lhw[k] = P.pass[k] ? (double)two : (double)0.1f;
    }
    P.ang = ((double)bin + res) * interval;
    return P;
}

__global__ void __launch_bounds__(kDetThreads) det_loss_partial_kernel(int n, int nv, int nbins, double interval, LossIn in,
                                                                       double *__restrict__ ws)
{
    __shared__ double red[9][kDetThreads];
    const int s = blockIdx.x;
    double acc[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};      // cls, offset, bin, res, corner, vote | cls_mask, pmask, vmask
    for (int p = threadIdx.x; p < n; p += blockDim.x) {
        const size_t r = (size_t)s * n + p;
        const double pm = in.pmask[r], cm = pm + in.nmask[r];
        const double x = in.cls[r * in.ld_cls], z = in.label[r];
        acc[0] += (fmax(x, 0.0) - x * z + log1p(exp(-fabs(x)))) * cm;            // sigmoid_cross_entropy_with_logits
        const float *o = in.off + r * in.ld_off;
        float t[6];
        target_of(in, r, t);
        double so = 0.0;
        for (int k = 0; k < 6; k++) so += huber((double)o[k] - t[k]);
        acc[1] += so * pm;
        const float *lg = in.acls + r * in.ld_acls;
        const int bin = in.bin[r];
        double mx = lg[0];
        for (int k = 1; k < nbins; k++) mx = fmax(mx, (double)lg[k]);
        double se = 0.0;
        for (int k = 0; k < nbins; k++) se += exp((double)lg[k] - mx);
        acc[2] += (mx + log(se) - lg[bin]) * pm;                                  // sparse softmax CE
        const float res = in.ares[r * in.ld_ares + bin];
        acc[3] += huber(((double)res - in.res[r]) * pm);
        const float *bx = in.box + r * 7;
        const PredBox P = pred_box(in.base + r * 3, o, res, bin, interval);
        double PC[8][3], GC[8][3];
        corners8(P.c[0], P.c[1], P.c[2], P.lhw[0], P.lhw[1], P.lhw[2], cos(P.ang), sin(P.ang), PC);
        corners8(bx[0], bx[1], bx[2], bx[3], bx[4], bx[5], cos((double)bx[6]), sin((double)bx[6]), GC);
        double sc = 0.0;
        for (int i = 0; i < 8; i++)
            for (int k = 0; k < 3; k++) sc += huber(PC[i][k] - GC[i][k]);
        acc[4] += sc * pm;
        acc[6] += cm;
        acc[7] += pm;
    }
    for (int p = threadIdx.x; p < nv; p += blockDim.x) {
        const size_t r = (size_t)s * nv + p;
        const double vm = in.vmask[r];
        const float *vo = in.vote + r * in.ld_vote, *vt = in.vtarget + r * 3;
        double sv = 0.0;
        for (int k = 0; k < 3; k++) sv += huber((double)vt[k] - vo[k]);
        acc[5] += sv * vm;
        acc[8] += vm;
    }
    for (int k = 0; k < 9; k++) red[k][threadIdx.x] = acc[k];
    for (int w = kDetThreads / 2; w > 0; w >>= 1) {                              // fixed-order tree
        __syncthreads();
        if (threadIdx.x < w)
            for (int k = 0; k < 9; k++) red[k][threadIdx.x] += red[k][threadIdx.x + w];
    }
    __syncthreads();
    if (threadIdx.x < 9) ws[(size_t)s * 9 + threadIdx.x] = red[threadIdx.x][0];
}

__global__ void det_loss_final_kernel(int b, const double *__restrict__ ws, float *__restrict__ loss, float *__restrict__ norm)
{
    __shared__ double tot[9];
    if (threadIdx.x < 9) {
        double a = 0.0;
        for (int s = 0; s < b; s++) a += ws[(size_t)s * 9 + threadIdx.x];
        tot[threadIdx.x] = a;
    }
    __syncthreads();
    if (threadIdx.x < 3) norm[threadIdx.x] = (float)fmax(1.0, tot[6 + threadIdx.x]);     // tf.maximum(1., sum(mask))
    if (threadIdx.x < 6) {
        const int which = threadIdx.x == 0 ? 6 : (threadIdx.x == 5 ? 8 : 7);
        loss[threadIdx.x] = (float)(tot[threadIdx.x] / fmax(1.0, tot[which]));
    }
}

__global__ void __launch_bounds__(kDetThreads) det_loss_grad_kernel(int b, int n, int nv, int nbins, double interval, LossIn in,
                                                                    const float *__restrict__ gl, const float *__restrict__ norm,
                                                                    float *__restrict__ gbase, float *__restrict__ gcls, int ldgc,
                                                                    float *__restrict__ goff, int ldgo, float *__restrict__ gacls,
                                                                    int ldga, float *__restrict__ gares, int ldgr,
                                                                    float *__restrict__ gvote)
{
    const long rows = (long)b * n, vrows = (long)b * nv;
    const long i = blockIdx.x * (long)blockDim.x + threadIdx.x;
    if (i < rows) {
        const size_t r = (size_t)i;
        const double pm = in.pmask[r], cm = pm + in.nmask[r];
        const double s_cls = (double)gl[0] / norm[0], s_off = (double)gl[1] / norm[1], s_bin = (double)gl[2] / norm[1],
                     s_res = (double)gl[3] / norm[1], s_cor = (double)gl[4] / norm[1];
        const double x = in.cls[r * in.ld_cls];
        gcls[r * ldgc] = cm != 0.0 ? (float)((1.0 / (1.0 + exp(-x)) - in.label[r]) * cm * s_cls) : 0.f;
        const float *o = in.off + r * in.ld_off;
        float t[6];
        target_of(in, r, t);
        const int bin = in.bin[r];
        const float *lg = in.acls + r * in.ld_acls;
        const float res = in.ares[r * in.ld_ares + bin];
        double d_off[6] = {0, 0, 0, 0, 0, 0}, d_base[3] = {0, 0, 0}, d_res = 0.0;
        if (pm != 0.0) {
            for (int k = 0; k < 6; k++) d_off[k] = huber_grad((double)o[k] - t[k]) * pm * s_off;
            // the target's translation is box - base_xyz (encoder_builder.py:57 -> anchor_encoder.py:172)
            for (int k = 0; k < 3; k++) d_base[k] = d_off[k];
            d_res = huber_grad(((double)res - in.res[r]) * pm) * pm * s_res;
            // corner loss through the decoded box
            const float *bx = in.box + r * 7;
            const PredBox P = pred_box(in.base + r * 3, o, res, bin, interval);
            const double c = cos(P.ang), sn = sin(P.ang);
            double PC[8][3], GC[8][3];
            corners8(P.c[0], P.c[1], P.c[2], P.lhw[0], P.lhw[1], P.lhw[2], c, sn, PC);
            corners8(bx[0], bx[1], bx[2], bx[3], bx[4], bx[5], cos((double)bx[6]), sin((double)bx[6]), GC);
            const double sx[8] = {1, 1, -1, -1, 1, 1, -1, -1}, sz[8] = {1, -1, -1, 1, 1, -1, -1, 1};
            double dc[3] = {0, 0, 0}, dl = 0, dh = 0, dw = 0, dang = 0;
            for (int q = 0; q < 8; q++) {
                const double gx = huber_grad(PC[q][0] - GC[q][0]) * pm * s_cor, gy = huber_grad(PC[q][1] - GC[q][1]) * pm * s_cor,
                             gz = huber_grad(PC[q][2] - GC[q][2]) * pm * s_cor;
                const double xc = sx[q] * P.lhw[0] / 2.0, zc = sz[q] * P.lhw[2] / 2.0;
                dc[0] += gx; dc[1] += gy; dc[2] += gz;
                dl += sx[q] / 2.0 * (c * gx - sn * gz);
                dw += sz[q] / 2.0 * (sn * gx + c * gz);
                if (q >= 4) dh -= gy;
                dang += gx * (-sn * xc + c * zc) + gz * (-c * xc - sn * zc);
            }
            for (int k = 0; k < 3; k++) { d_off[k] += dc[k]; d_base[k] += dc[k]; }
            d_off[4] += dc[1];                                                  // the centre moves down by the half height
            if (P.pass[0]) d_off[3] += 2.0 * dl;
            if (P.pass[1]) d_off[4] += 2.0 * dh;
            if (P.pass[2]) d_off[5] += 2.0 * dw;
            d_res += dang * interval;
        }
        for (int k = 0; k < 6; k++) goff[r * ldgo + k] = (float)d_off[k];
        for (int k = 0; k < 3; k++) gbase[r * 3 + k] = (float)d_base[k];
        double mx = lg[0];
        for (int k = 1; k < nbins; k++) mx = fmax(mx, (double)lg[k]);
        double se = 0.0;
        if (pm != 0.0)
            for (int k = 0; k < nbins; k++) se += exp((double)lg[k] - mx);
        for (int k = 0; k < nbins; k++) {
            gacls[r * ldga + k] = pm != 0.0 ? (float)((exp((double)lg[k] - mx) / se - (k == bin ? 1.0 : 0.0)) * pm * s_bin) : 0.f;
            gares[r * ldgr + k] = k == bin ? (float)d_res : 0.f;
        }
    }
    if (i < vrows) {
        const size_t r = (size_t)i;
        const double vm = in.vmask[r], s_v = (double)gl[5] / norm[2];
        const float *vo = in.vote + r * in.ld_vote, *vt = in.vtarget + r * 3;
        for (int k = 0; k < 3; k++) gvote[r * 3 + k] = vm != 0.0 ? (float)(-huber_grad((double)vt[k] - vo[k]) * vm * s_v) : 0.f;
    }
}

static double bin_interval(int nbins) { return (double)(float)(2.0 * M_PI / nbins); }   // the float32 constant of TF

}  // namespace ssd3d

using namespace ssd3d;

extern "C" int ssd3d_det_assign(int b, int n, int nv, int g, int angle_bins, const float *base_xyz, const float *vote_base,
                                const float *gt_boxes, const int *gt_labels, int *assigned_idx, float *assigned_box,
                                float *pmask, float *nmask, float *cls_label, int *angle_bin, float *angle_res,
                                float *offset_target, float *vote_mask, float *vote_target, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && n >= 0 && nv >= 0 && g >= 0 && angle_bins >= 1 && angle_bins <= kMaxBins,
                  "det_assign: bad shape b=%d n=%d nv=%d g=%d bins=%d", b, n, nv, g, angle_bins);
    if (b == 0 || (n == 0 && nv == 0)) return 0;
    SSD3D_REQUIRE((n == 0 || (base_xyz && assigned_idx && assigned_box && pmask && nmask && cls_label && angle_bin && angle_res &&
                              offset_target)) && (nv == 0 || (vote_base && vote_mask && vote_target)) &&
                  (g == 0 || (gt_boxes && gt_labels)), "det_assign: null pointer");
    det_assign_kernel<<<b, kDetThreads, 0, (cudaStream_t)stream>>>(n, nv, g, angle_bins, base_xyz, vote_base, gt_boxes, gt_labels,
                                                                   assigned_idx, assigned_box, pmask, nmask, cls_label, angle_bin,
                                                                   angle_res, offset_target, vote_mask, vote_target);
    SSD3D_LAUNCH_CHECK("det_assign_kernel");
}

extern "C" size_t ssd3d_det_loss_workspace(int b) { return (size_t)(b > 0 ? b : 0) * 9 * sizeof(double); }

static int det_loss_in(int n, int nv, int angle_bins, const float *base_xyz, const float *pred_cls, int ld_cls,
                       const float *pred_offset, int ld_offset, const float *pred_angle_cls, int ld_angle_cls,
                       const float *pred_angle_res, int ld_angle_res, const float *vote_offset, int ld_vote,
                       const float *assigned_box, const float *pmask, const float *nmask, const float *cls_label,
                       const int *angle_bin, const float *angle_res, const float *vote_mask,
                       const float *vote_target, LossIn &in)
{
    SSD3D_REQUIRE(angle_bins >= 1 && angle_bins <= kMaxBins && ld_cls >= 1 && ld_offset >= 6 && ld_angle_cls >= angle_bins &&
                  ld_angle_res >= angle_bins && ld_vote >= 3, "det_loss: bad row strides or bins=%d", angle_bins);
    SSD3D_REQUIRE(n == 0 || (base_xyz && pred_cls && pred_offset && pred_angle_cls && pred_angle_res && assigned_box && pmask &&
                             nmask && cls_label && angle_bin && angle_res), "det_loss: null pointer");
    SSD3D_REQUIRE(nv == 0 || (vote_offset && vote_mask && vote_target), "det_loss: null pointer");
    in = LossIn{base_xyz, pred_cls, pred_offset, pred_angle_cls, pred_angle_res, vote_offset, ld_cls, ld_offset, ld_angle_cls,
                ld_angle_res, ld_vote, assigned_box, pmask, nmask, cls_label, angle_res, vote_mask, vote_target,
                angle_bin};
    return 0;
}

extern "C" int ssd3d_det_loss(int b, int n, int nv, int angle_bins, const float *base_xyz, const float *pred_cls, int ld_cls,
                              const float *pred_offset, int ld_offset, const float *pred_angle_cls, int ld_angle_cls,
                              const float *pred_angle_res, int ld_angle_res, const float *vote_offset, int ld_vote,
                              const float *assigned_box, const float *pmask, const float *nmask, const float *cls_label,
                              const int *angle_bin, const float *angle_res, const float *vote_mask,
                              const float *vote_target, void *workspace, float *loss, float *norm, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 1 && n >= 0 && nv >= 0, "det_loss: bad shape b=%d n=%d nv=%d", b, n, nv);
    SSD3D_REQUIRE(workspace && loss && norm, "det_loss: null pointer");
    LossIn in;
    const int st = det_loss_in(n, nv, angle_bins, base_xyz, pred_cls, ld_cls, pred_offset, ld_offset, pred_angle_cls, ld_angle_cls,
                               pred_angle_res, ld_angle_res, vote_offset, ld_vote, assigned_box, pmask, nmask, cls_label, angle_bin,
                               angle_res, vote_mask, vote_target, in);
    if (st) return st;
    det_loss_partial_kernel<<<b, kDetThreads, 0, (cudaStream_t)stream>>>(n, nv, angle_bins, bin_interval(angle_bins), in,
                                                                         (double *)workspace);
    const int e = cuda_status(cudaGetLastError(), "det_loss_partial_kernel");
    if (e) return e;
    det_loss_final_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(b, (const double *)workspace, loss, norm);
    SSD3D_LAUNCH_CHECK("det_loss_final_kernel");
}

extern "C" int ssd3d_det_loss_grad(int b, int n, int nv, int angle_bins, const float *base_xyz, const float *pred_cls, int ld_cls,
                                   const float *pred_offset, int ld_offset, const float *pred_angle_cls, int ld_angle_cls,
                                   const float *pred_angle_res, int ld_angle_res, const float *vote_offset, int ld_vote,
                                   const float *assigned_box, const float *pmask, const float *nmask, const float *cls_label,
                                   const int *angle_bin, const float *angle_res, const float *vote_mask,
                                   const float *vote_target, const float *grad_loss, const float *norm,
                                   float *grad_base_xyz, float *grad_cls, int ldg_cls, float *grad_offset, int ldg_offset,
                                   float *grad_angle_cls, int ldg_angle_cls, float *grad_angle_res, int ldg_angle_res,
                                   float *grad_vote_offset, ssd3d_stream_t stream)
{
    SSD3D_REQUIRE(b >= 0 && n >= 0 && nv >= 0, "det_loss_grad: bad shape b=%d n=%d nv=%d", b, n, nv);
    SSD3D_REQUIRE(ldg_cls >= 1 && ldg_offset >= 6 && ldg_angle_cls >= angle_bins && ldg_angle_res >= angle_bins,
                  "det_loss_grad: bad gradient row strides");
    const long rows = (long)b * (n > nv ? n : nv);
    if (rows == 0) return 0;
    SSD3D_REQUIRE(grad_loss && norm && (n == 0 || (grad_base_xyz && grad_cls && grad_offset && grad_angle_cls && grad_angle_res)) &&
                  (nv == 0 || grad_vote_offset), "det_loss_grad: null pointer");
    LossIn in;
    const int st = det_loss_in(n, nv, angle_bins, base_xyz, pred_cls, ld_cls, pred_offset, ld_offset, pred_angle_cls, ld_angle_cls,
                               pred_angle_res, ld_angle_res, vote_offset, ld_vote, assigned_box, pmask, nmask, cls_label, angle_bin,
                               angle_res, vote_mask, vote_target, in);
    if (st) return st;
    det_loss_grad_kernel<<<ceil_div(rows, kDetThreads), kDetThreads, 0, (cudaStream_t)stream>>>(
        b, n, nv, angle_bins, bin_interval(angle_bins), in, grad_loss, norm, grad_base_xyz, grad_cls, ldg_cls, grad_offset, ldg_offset,
        grad_angle_cls, ldg_angle_cls, grad_angle_res, ldg_angle_res, grad_vote_offset);
    SSD3D_LAUNCH_CHECK("det_loss_grad_kernel");
}
