// box_geom.cuh -- box geometry shared by the target assignment (det_loss.cu), the evaluator (box_eval.cu), the
// augmentor (augment.cu) and the mixup paste (mixup.cu): the face planes of a box with the point-in-box test, the one
// pinned double sincos, and the float32 BEV corners and collision test of the noise search and the paste.
#pragma once
#include "common.cuh"

namespace ssd3d {

// The six face planes of a box in the frame check_inside_points uses (voxelnet_aug.py:318-342): point (x, z, y),
// box (x, z, y, l, w, h, ry), corners of center_to_corner_box3d(origin (0.5, 0.5, 1), axis 2), surfaces of
// corner_to_surfaces_3d_jit, plane (n, d) of surface_equ_3d_jit.  Every operation is one IEEE float32 op (no FMA
// contraction) in a fixed order, so that a numpy restatement gives the same bits.
struct Planes {
    float n[6][3];
    float d[6];
};

__device__ __forceinline__ void box_planes(const float *bx, float expand, float sn, float cs, Planes &P)
{
    const float c0 = bx[0], c1 = bx[2], c2 = bx[1];                          // centre in (x, z, y)
    const float dl = __fadd_rn(bx[3], expand), dw = __fadd_rn(bx[5], expand), dh = __fadd_rn(bx[4], expand);
    // corners_nd after its [0, 1, 3, 2, 4, 5, 7, 6] reordering, minus the origin (0.5, 0.5, 1.0)
    const float na[8] = {-0.5f, -0.5f, -0.5f, -0.5f, 0.5f, 0.5f, 0.5f, 0.5f};
    const float nb[8] = {-0.5f, -0.5f, 0.5f, 0.5f, -0.5f, -0.5f, 0.5f, 0.5f};
    const float nc[8] = {-1.0f, 0.0f, 0.0f, -1.0f, -1.0f, 0.0f, 0.0f, -1.0f};
    float C[8][3];
#pragma unroll
    for (int k = 0; k < 8; k++) {
        const float p0 = __fmul_rn(dl, na[k]), p1 = __fmul_rn(dw, nb[k]), p2 = __fmul_rn(dh, nc[k]);
        // rotation_3d_in_axis(axis=2): [p0, p1] @ [[cos, -sin], [sin, cos]]
        C[k][0] = __fadd_rn(__fadd_rn(__fmul_rn(p0, cs), __fmul_rn(p1, sn)), c0);
        C[k][1] = __fadd_rn(__fsub_rn(__fmul_rn(p1, cs), __fmul_rn(p0, sn)), c1);
        C[k][2] = __fadd_rn(p2, c2);
    }
    const int F[6][3] = {{0, 1, 2}, {7, 6, 5}, {0, 3, 7}, {1, 5, 6}, {0, 4, 5}, {3, 2, 6}};   // first 3 corners per face
#pragma unroll
    for (int f = 0; f < 6; f++) {
        const float *a = C[F[f][0]], *b = C[F[f][1]], *c = C[F[f][2]];
        const float u0 = __fsub_rn(a[0], b[0]), u1 = __fsub_rn(a[1], b[1]), u2 = __fsub_rn(a[2], b[2]);
        const float v0 = __fsub_rn(b[0], c[0]), v1 = __fsub_rn(b[1], c[1]), v2 = __fsub_rn(b[2], c[2]);
        const float n0 = __fsub_rn(__fmul_rn(u1, v2), __fmul_rn(u2, v1));
        const float n1 = __fsub_rn(__fmul_rn(u2, v0), __fmul_rn(u0, v2));
        const float n2 = __fsub_rn(__fmul_rn(u0, v1), __fmul_rn(u1, v0));
        P.n[f][0] = n0; P.n[f][1] = n1; P.n[f][2] = n2;
        P.d[f] = -__fadd_rn(__fadd_rn(__fmul_rn(n0, a[0]), __fmul_rn(n1, a[1])), __fmul_rn(n2, a[2]));
    }
}

// points_in_convex_polygon_3d_jit (voxelnet_aug.py:532-567): outside as soon as one face gives sign >= 0
__device__ __forceinline__ bool inside(const Planes &P, float q0, float q1, float q2)
{
#pragma unroll
    for (int f = 0; f < 6; f++) {
        const float s = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(q0, P.n[f][0]), __fmul_rn(q1, P.n[f][1])), __fmul_rn(q2, P.n[f][2])),
                                  P.d[f]);
        if (s >= 0.0f) return false;
    }
    return true;
}

// ---- sincos ----------------------------------------------------------------------------------------------------------
// Cody-Waite reduction by pi/2, fdlibm's minimax polynomials with explicit fma: CUDA's sincos and glibc's differ in the
// last bit on some inputs, this recipe gives the same bits on both sides (the C twin of the test suite restates it).
__device__ __forceinline__ double k_sin(double r)
{
    const double z = __dmul_rn(r, r);
    double p = __fma_rn(z, 1.58969099521155010221e-10, -2.50507602534068634195e-08);
    p = __fma_rn(z, p, 2.75573137070700676789e-06);
    p = __fma_rn(z, p, -1.98412698298579493134e-04);
    p = __fma_rn(z, p, 8.33333333332248946124e-03);
    p = __fma_rn(z, p, -1.66666666666666324348e-01);
    return __fma_rn(__dmul_rn(r, z), p, r);
}

__device__ __forceinline__ double k_cos(double r)
{
    const double z = __dmul_rn(r, r);
    double p = __fma_rn(z, -1.13596475577881948265e-11, 2.08757232129817482790e-09);
    p = __fma_rn(z, p, -2.75573143513906633035e-07);
    p = __fma_rn(z, p, 2.48015872894767294178e-05);
    p = __fma_rn(z, p, -1.38888888888741095749e-03);
    p = __fma_rn(z, p, 4.16666666666666019037e-02);
    const double hz = __dmul_rn(0.5, z), w = __dsub_rn(1.0, hz);
    return __dadd_rn(w, __fma_rn(z, __dmul_rn(z, p), __dsub_rn(__dsub_rn(1.0, w), hz)));
}

__device__ __forceinline__ void eval_sincos(double x, double &s, double &c)
{
    const double n = rint(__dmul_rn(x, 0x1.45f306dc9c883p-1));          // x * 2/pi, to the nearest integer
    double r = __fma_rn(-n, 0x1.921fb54442d18p+0, x);                   // x - n * pi/2, pi/2 in two parts
    r = __fma_rn(-n, 0x1.1a62633145c07p-54, r);
    const double sr = k_sin(r), cr = k_cos(r);
    switch (((long long)n) & 3) {
        case 0: s = sr; c = cr; break;
        case 1: s = cr; c = -sr; break;
        case 2: s = -sr; c = -cr; break;
        default: s = -cr; c = sr; break;
    }
}

__device__ __forceinline__ void sincos32(double a, float &s, float &c)
{
    double sd, cd;
    eval_sincos(a, sd, cd);
    s = (float)sd;
    c = (float)cd;
}

// ---- BEV rectangles (voxelnet_aug.py) ----------------------------------------------------------------------------------
// A padded GT row is all zeros.
__device__ __forceinline__ bool box_is_valid(const float *b)
{
    return b[0] != 0.f || b[1] != 0.f || b[2] != 0.f || b[3] != 0.f || b[4] != 0.f || b[5] != 0.f || b[6] != 0.f;
}

// box2d_to_corner_jit (voxelnet_aug.py:510-529) of one BEV box (x, z, l, w) whose dims the caller has already grown,
// float32 op by op: corners_norm * (l, w) @ [[cos, -sin], [sin, cos]] + (x, z)
__device__ __forceinline__ void bev_corners(float x, float z, float dl, float dw, float sn, float cs, float (*c)[2])
{
    const float na[4] = {-0.5f, -0.5f, 0.5f, 0.5f}, nb[4] = {-0.5f, 0.5f, 0.5f, -0.5f};
    for (int k = 0; k < 4; k++) {
        const float a = __fmul_rn(dl, na[k]), bb = __fmul_rn(dw, nb[k]);
        c[k][0] = __fadd_rn(__fadd_rn(__fmul_rn(a, cs), __fmul_rn(bb, sn)), x);
        c[k][1] = __fadd_rn(__fsub_rn(__fmul_rn(bb, cs), __fmul_rn(a, sn)), z);
    }
}

__device__ __forceinline__ bool ccw_gt(const float *A, const float *B, const float *C)   // (C1-A1)(B0-A0) > (B1-A1)(C0-A0)
{
    return __fmul_rn(__fsub_rn(C[1], A[1]), __fsub_rn(B[0], A[0])) > __fmul_rn(__fsub_rn(B[1], A[1]), __fsub_rn(C[0], A[0]));
}

// every corner of q strictly inside the clockwise rectangle a (box_collision_test's containment, clockwise=True)
__device__ __forceinline__ bool holds(const float (*a)[2], const float (*q)[2])
{
    for (int l = 0; l < 4; l++)
        for (int k = 0; k < 4; k++) {
            const int k1 = (k + 1) & 3;
            const float v0 = __fsub_rn(a[k1][0], a[k][0]), v1 = __fsub_rn(a[k1][1], a[k][1]);
            const float cr = __fsub_rn(__fmul_rn(v1, __fsub_rn(a[k][0], q[l][0])), __fmul_rn(v0, __fsub_rn(a[k][1], q[l][1])));
            if (cr >= 0.0f) return false;
        }
    return true;
}

// box_collision_test (voxelnet_aug.py:632-712) of one pair of BEV rectangles, float32 op by op
static __device__ bool collide(const float (*a)[2], const float (*q)[2])
{
    float amin0 = a[0][0], amax0 = a[0][0], amin1 = a[0][1], amax1 = a[0][1];
    float qmin0 = q[0][0], qmax0 = q[0][0], qmin1 = q[0][1], qmax1 = q[0][1];
    for (int k = 1; k < 4; k++) {
        amin0 = fminf(amin0, a[k][0]); amax0 = fmaxf(amax0, a[k][0]); amin1 = fminf(amin1, a[k][1]); amax1 = fmaxf(amax1, a[k][1]);
        qmin0 = fminf(qmin0, q[k][0]); qmax0 = fmaxf(qmax0, q[k][0]); qmin1 = fminf(qmin1, q[k][1]); qmax1 = fmaxf(qmax1, q[k][1]);
    }
    if (!(__fsub_rn(fminf(amax0, qmax0), fmaxf(amin0, qmin0)) > 0.0f)) return false;
    if (!(__fsub_rn(fminf(amax1, qmax1), fmaxf(amin1, qmin1)) > 0.0f)) return false;
    for (int k = 0; k < 4; k++) {
        const float *A = a[k], *B = a[(k + 1) & 3];
        for (int l = 0; l < 4; l++) {
            const float *C = q[l], *D = q[(l + 1) & 3];
            if (ccw_gt(A, C, D) != ccw_gt(B, C, D) && ccw_gt(A, B, C) != ccw_gt(A, B, D)) return true;
        }
    }
    return holds(a, q) || holds(q, a);
}

}  // namespace ssd3d
