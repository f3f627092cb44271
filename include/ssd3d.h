/*
 * ssd3d.h -- C ABI of libssd3d.so, the H100 (sm_90a) implementation of the set-abstraction
 * operators of dvlab-research/3DSSD.
 *
 * Drop-in boundary (SURVEY.md section 8b, seam iii): the reference's TF custom ops call free C++
 * "Launcher" functions that take plain ints and raw device pointers; each entry point below
 * replaces one of them with the same argument list, plus a CUDA stream and an int status
 * (0 = cudaSuccess, otherwise a cudaError_t or SSD3D_ERR_*).  Citations are file:line under
 * /root/reference/lib/utils/tf_ops/ (declaration in the .cpp that the TF op binds, definition at
 * the tail of the matching *_g.cu).
 *
 * Conventions, identical to the reference: dense row-major tensors, batch-major; fp32 values,
 * int32 indices; every pointer is a DEVICE pointer owned by the caller; the library allocates
 * nothing, keeps no state between calls, never synchronises the host, and is CUDA-graph
 * capturable.  `stream` is a cudaStream_t passed as void* (NULL = legacy default stream).
 */
#ifndef SSD3D_H_
#define SSD3D_H_

#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SSD3D_ERR_INVALID_ARGUMENT (-1) /* mirrors the reference's OP_REQUIRES -> InvalidArgument */
#define SSD3D_ERR_UNSUPPORTED      (-2)

typedef void *ssd3d_stream_t;

/* ABI version of this header (bumped on any signature change). */
int ssd3d_version(void);   /* 2 since round 2 (explicit-placement *_ex entry points, last_scale_nonneg) */
/* Human-readable description of the last non-zero status returned on this thread. */
const char *ssd3d_last_error(void);

/* ---- sampling ------------------------------------------------------------------------------ */

/* replaces farthestpointsamplingLauncher(b,n,c,m,inp,temp,out)
 *   sampling/tf_sampling.cpp:131 (decl), sampling/tf_sampling_g.cu:392-394 (def), kernel :124-178.
 * D-FPS over inp[b,n,c] (any c; c==3 takes the on-chip cluster kernel).  out[b,m] int32.
 * temp[b,n] fp32 scratch is only touched by the large-n fallback; it may be NULL when
 * ssd3d_fps_needs_temp(n,c)==0.  Bit-exact, including the reference's tie-break (value desc,
 * k mod 1024 asc, k asc). */
int ssd3d_farthest_point_sample(int b, int n, int c, int m, const float *inp, float *temp, int *out,
                                ssd3d_stream_t stream);
int ssd3d_fps_needs_temp(int n, int c);

/* The same operator with explicit placement -- what lets an SA layer run its sampling without any copy / add /
 * concat kernels around it (lib/utils/layers_util.py:84-111):
 *   in_stride   floats between consecutive scenes of inp (>= n*c): a [:, a:b] slice of a dense [b,N,c] tensor;
 *   ldo         ints between consecutive rows of out (>= m): a column block of the concatenated fps_idx tensor;
 *   idx_offset  added to every stored index (the `+ last_fps_end_index` of :109);
 *   j0, j1      run only rounds [j0, j1) of 0..m; the running state travels through temp[b, E] between the launches
 *               (required when the range is partial), E = ssd3d_fps_temp_elems(n, c, m, flags) floats per scene.  A
 *               sample is final as soon as its round is done, so work on the first samples can overlap the remaining
 *               rounds.  Partial ranges need ssd3d_fps_supports_rounds(n, c);
 *   cluster     CTAs per scene: 0 = heuristic, 1/2/4/8/16 = exactly that, negative = heuristic capped at -cluster
 *               (FPS is latency-bound: fewer CTAs cost little time and leave SMs to concurrent work);
 *   flags       bit 0: use the general cluster kernel (coordinates travel in the packets) even where the
 *               resident-scene kernel applies; bit 1: never / bit 2: always (64 <= n <= 16384) take the single-CTA
 *               kernel with spatial pruning (csrc/fps_bucket.cu) that c == 3 scenes of 8192 < n <= 16384 points and
 *               m >= 256 get by default -- points grouped into spatially compact buckets of 32, a round updates only
 *               the buckets whose bounding box lies closer to the new sample than their largest running distance
 *               (the others provably keep every distance), so one SM per scene suffices; `cluster` is ignored there.
 * No state is kept in the library: every choice is an argument. */
int ssd3d_farthest_point_sample_ex(int b, int n, int c, int m, const float *inp, long long in_stride, float *temp,
                                   int *out, int ldo, int idx_offset, int j0, int j1, int cluster, int flags,
                                   ssd3d_stream_t stream);
int ssd3d_fps_supports_rounds(int n, int c);
long ssd3d_fps_temp_elems(int n, int c, int m, int flags);

/* replaces farthestpointsamplingwithdistLauncher(b,n,m,inp,temp,out)
 *   sampling/tf_sampling.cpp:164, sampling/tf_sampling_g.cu:396-398, kernel :181-230.
 * F-FPS over a precomputed distance matrix dist[b,n,n]. */
int ssd3d_farthest_point_sample_with_distance(int b, int n, int m, const float *dist, float *temp, int *out,
                                              ssd3d_stream_t stream);
/* ... with explicit output placement and cluster request (see ssd3d_farthest_point_sample_ex). */
int ssd3d_farthest_point_sample_with_distance_ex(int b, int n, int m, const float *dist, float *temp, int *out, int ldo,
                                                 int idx_offset, int cluster, ssd3d_stream_t stream);

/* The F-FPS branch of the SA layer in one call (lib/utils/layers_util.py:94-96 and :102-104):
 *   farthest_point_sample_with_distance(m, calc_square_dist(concat[fa, fb]))
 * without materialising the [b,n,n] matrix -- each round evaluates the picked point's matrix row on the fly from
 * feature rows kept on chip.  fa[b,n,ca] (xyz, ca = 3 in the model), fb[b,n,cb] (features; may be NULL when cb = 0).
 * Same indices as the two-call route (same pinned fp32 arithmetic as ssd3d_calc_square_dist).  Covers
 * ca+cb <= 68 with n <= 4096 and ca+cb <= 132 with n <= 2048 (ssd3d_ffps_supported); other shapes return
 * SSD3D_ERR_UNSUPPORTED and the caller takes the two-call route. */
int ssd3d_farthest_point_sample_features(int b, int n, int ca, int cb, int m, const float *fa, const float *fb,
                                         int *out, ssd3d_stream_t stream);
/* ... with scene strides of fa / fb in floats, explicit output placement and a range of rounds [j0, j1) with the
 * running distances in temp[b,n] (see ssd3d_farthest_point_sample_ex; temp may be NULL for the full range). */
int ssd3d_farthest_point_sample_features_ex(int b, int n, int ca, int cb, int m, const float *fa, long long fa_stride,
                                            const float *fb, long long fb_stride, float *temp, int *out, int ldo,
                                            int idx_offset, int j0, int j1, ssd3d_stream_t stream);
/* ... with a cluster request: 0 = as _ex, < 0 = CTAs per scene capped at -cluster (-1, -2, -4, -8 or -16).  A cap below
 * what _ex uses runs a full-range call with 2048 < n <= 4096, 3 <= ca+cb <= 68 on 4 CTAs per scene with bucket
 * pruning (same indices; fewer SMs per scene for throughput); partial ranges and other shapes run as _ex. */
int ssd3d_farthest_point_sample_features_cl(int b, int n, int ca, int cb, int m, const float *fa, long long fa_stride,
                                            const float *fb, long long fb_stride, float *temp, int *out, int ldo,
                                            int idx_offset, int j0, int j1, int cluster, ssd3d_stream_t stream);
int ssd3d_ffps_supported(int n, int c);

/* replaces gatherpointLauncher(b,n,m,c,inp,idx,out)
 *   sampling/tf_sampling.cpp:235, sampling/tf_sampling_g.cu:403-407, kernel :320-331.
 * out[b,m,c] = inp[b, idx[b,m], c] */
int ssd3d_gather_point(int b, int n, int m, int c, const float *inp, const int *idx, float *out,
                       ssd3d_stream_t stream);
/* ... reading idx rows ld_idx ints apart (a column block of a wider [b, L] index tensor). */
int ssd3d_gather_point_ex(int b, int n, int m, int c, const float *inp, const int *idx, int ld_idx, float *out,
                          ssd3d_stream_t stream);

/* ---- grouping ------------------------------------------------------------------------------ */

/* replaces queryBallPointLauncher(b,n,m,radius,nsample,xyz1,xyz2,idx,pts_cnt)
 *   grouping/tf_grouping.cpp:270, grouping/tf_grouping_g.cu:461-464, kernel :215-255.
 * idx[b,m,nsample], pts_cnt[b,m].  Rows with pts_cnt==0 are written as zeros (the reference leaves
 * them uninitialised and its caller masks them, lib/utils/layers_util.py:157-159). */
int ssd3d_query_ball_point(int b, int n, int m, float radius, int nsample, const float *xyz1, const float *xyz2,
                           int *idx, int *pts_cnt, ssd3d_stream_t stream);

/* replaces queryBallPointDilatedLauncher(b,n,m,min_radius,max_radius,nsample,xyz1,xyz2,idx,pts_cnt)
 *   grouping/tf_grouping.cpp:363, grouping/tf_grouping_g.cu:465-468, kernel :308-357. */
int ssd3d_query_ball_point_dilated(int b, int n, int m, float min_radius, float max_radius, int nsample,
                                   const float *xyz1, const float *xyz2, int *idx, int *pts_cnt,
                                   ssd3d_stream_t stream);

/* Fast path used by pointnet_sa_module_msg: up to 4 (min_r,max_r,nsample) queries over the same
 * (xyz1,xyz2) answered in ONE pass over the candidates (the reference scans once per radius,
 * lib/utils/layers_util.py:134-147).  dilated!=0 selects the :308-357 predicate, else the :215-255 one
 * (min_radius ignored).  idx[s] / pts_cnt[s] are per-query outputs as above. */
int ssd3d_query_ball_point_multi(int b, int n, int m, int nqueries, int dilated, const float *min_radius,
                                 const float *max_radius, const int *nsample, const float *xyz1, const float *xyz2,
                                 int *const *idx, int *const *pts_cnt, ssd3d_stream_t stream);
/* The same search with spatial culling (csrc/ball_query_grid.cu) for large candidate sets: `workspace` is caller-owned
 * scratch of ssd3d_query_ball_point_workspace(b, n) bytes (16-byte aligned; 0 = this size has no culled kernel).  One
 * small kernel bins the candidates of every scene into a uniform 2-D grid with cells >= r_max, the search then visits
 * only the 3x3 cell neighbourhood of a query and restores "first nsample hits in ascending index" through a per-shell
 * bitmap over candidate indices.  Same outputs, bit for bit, non-finite coordinates included.  workspace == NULL
 * falls through to ssd3d_query_ball_point_multi.
 * units (optional, host array of nqueries device pointers, entries may be NULL): per-shell UNIT LISTS for the grouped MLP.
 * units[s] holds 1 + b*m*ceil(nsample[s]/8) ints: [0] = number of units, [1 + u] = (group << 4) | j naming rows 8j..8j+7
 * of neighbour list `group` (= scene*m + query).  A group with cnt hits gets ceil(cnt/8) units -- slots beyond cnt repeat
 * the first hit (tf_grouping_g.cu:245-248) and cannot change the max-pool that follows (layers_util.py:178), so the
 * grouped MLP needs only these rows (ssd3d_sa_mlp_fused*, ssd3d_linear_tc*_units).  The list order is unspecified.
 * Without a workspace the list is built from the finished counts by one more small kernel. */
size_t ssd3d_query_ball_point_workspace(int b, int n);
int ssd3d_query_ball_point_multi_ws(int b, int n, int m, int nqueries, int dilated, const float *min_radius,
                                    const float *max_radius, const int *nsample, const float *xyz1, const float *xyz2,
                                    int *const *idx, int *const *pts_cnt, int *const *units, void *workspace,
                                    size_t workspace_bytes, ssd3d_stream_t stream);
/* The same with a unit width per shell: unit_rows (host array of nqueries ints, NULL = all 8) gives shell s units of
 * W = unit_rows[s] rows, 8 or 4: [1 + u] = (group << 4) | j then names rows Wj..Wj+W-1, a group with cnt hits gets
 * ceil(cnt/W) units and units[s] holds 1 + b*m*ceil(nsample[s]/W) ints.  j has 4 bits, so W = 4 needs nsample <= 64
 * (W = 8: nsample <= 128).  The consumers of a list take the same width (the *_ex / *_units_ex calls below). */
int ssd3d_query_ball_point_multi_ws_ex(int b, int n, int m, int nqueries, int dilated, const float *min_radius,
                                       const float *max_radius, const int *nsample, const float *xyz1, const float *xyz2,
                                       int *const *idx, int *const *pts_cnt, int *const *units, void *workspace,
                                       size_t workspace_bytes, ssd3d_stream_t stream, const int *unit_rows);

/* replaces groupPointLauncher(b,n,c,m,nsample,points,idx,out)
 *   grouping/tf_grouping.cpp:446, grouping/tf_grouping_g.cu:476-479, kernel :362-379.
 * out[b,m,nsample,c] = points[b, idx[b,m,nsample], c]; idx==-1 -> 0 */
int ssd3d_group_point(int b, int n, int c, int m, int nsample, const float *points, const int *idx, float *out,
                      ssd3d_stream_t stream);

/* ---- interpolation ------------------------------------------------------------------------- */

/* replaces ThreeNNLauncher(b,n,m,xyz1,xyz2,dist,idx)
 *   interpolation/tf_interpolate.cpp:215, interpolation/tf_interpolate_g.cu:191-195, kernel :24-84. */
int ssd3d_three_nn(int b, int n, int m, const float *xyz1, const float *xyz2, float *dist, int *idx,
                   ssd3d_stream_t stream);

/* replaces ThreeInterpolateLauncher(b,m,c,n,points,idx,weight,out)
 *   interpolation/tf_interpolate.cpp:285, interpolation/tf_interpolate_g.cu:198-200, kernel :87-113. */
int ssd3d_three_interpolate(int b, int m, int c, int n, const float *points, const int *idx, const float *weight,
                            float *out, ssd3d_stream_t stream);

/* The operand of an FP layer's first conv in one pass (pointnet_fp_module, lib/utils/layers_util.py:206-214): for every
 * unknown point of xyz1[b,n,3] the three nearest of xyz2[b,m,3] (as ssd3d_three_nn), the weights w_k = inv_k / norm
 * with inv_k = 1 / max(d_k, 1e-10) and norm = (inv_0 + inv_1) + inv_2 (fp32, one rounding per operation), and the row
 * [three_interpolate(points2[b,m,c2]) | points1[b,n,c1]] written split into out_hi / out_lo [b*n, kp] bf16 (hi = bf16(x),
 * lo = bf16(x - hi), zero beyond c2 + c1; the operand of ssd3d_linear_tc).  m >= 1, kp % 16 == 0, kp >= c2 + c1,
 * points1 may be null when c1 == 0, outputs 16-byte aligned.  Bit for bit the split of the concatenation of
 * ssd3d_three_interpolate's output with points1. */
int ssd3d_fp_interp_split(int b, int n, int m, int c2, int c1, const float *xyz1, const float *xyz2, const float *points2,
                          const float *points1, void *out_hi, void *out_lo, int kp, ssd3d_stream_t stream);

/* ---- dense parts of the SA layer (TF stock ops in the reference) ---------------------------- */

/* model_util.calc_square_dist(a, a, norm=False)  (lib/utils/model_util.py:144-160) for a[b,n,c]:
 * out[b,i,j] = (|a_i|^2 + |a_j|^2) - 2 a_i.a_j, fp32, channel sums as sequential fma chains
 * (order pinned so the oracle can be bit-exact; the reference's cuBLAS order is unspecified). */
int ssd3d_calc_square_dist(int b, int n, int c, const float *a, float *out, ssd3d_stream_t stream);

/* Fused gather + concat of lib/utils/layers_util.py:160-165:
 *   x[b,m,k,:] = concat( points[b, idx[b,m,k], 0:c],  xyz[b, idx[b,m,k], :] - new_xyz[b,m,:] )
 * written with row stride ldx (>= c+3; columns c+3..ldx-1 are zero-filled). */
int ssd3d_group_concat(int b, int n, int c, int m, int nsample, const float *xyz, const float *points,
                       const float *new_xyz, const int *idx, float *x, int ldx, ssd3d_stream_t stream);

/* One tf_util.conv2d/conv1d 1x1 layer at inference (lib/utils/tf_util.py:51-201, BN :424-444) with
 * bias and BatchNorm pre-folded by the caller into per-channel (scale, shift):
 *   y[r, o] = act( (sum_k x[r,k] * w[k,o]) * scale[o] + shift[o] ),  act = relu or identity.
 * x[rows, ldx] (first cin columns used), w[cin, cout] (the TF kernel [1,1,cin,cout]), y[rows, ldy].
 * pool > 1: instead of y, write ymax[rows/pool, cout] = max over each run of `pool` consecutive rows
 * (tf.reduce_max(axis=2), layers_util.py:178) times rowmask[rows/pool] when rowmask != NULL (:180). */
int ssd3d_linear_bn_relu(long rows, int cin, int cout, const float *x, int ldx, const float *w,
                         const float *scale, const float *shift, int relu, int pool, const int *rowmask,
                         float *y, int ldy, ssd3d_stream_t stream);

/* ---- tensor-core (wgmma) path of the same layer -------------------------------------------------
 * fp32 operands travel as TWO bf16 matrices (x = hi + lo, 16 mantissa bits); the product is evaluated as
 * hi.hi + lo.hi + hi.lo with fp32 accumulation (error ~2^-16, inside the 1e-3 parity budget).
 *   a_hi/a_lo [rows, kp] bf16 row-major (kp % 16 == 0, zero padded); b_hi/b_lo [n, kp] bf16 = W^T split;
 *   outputs (any subset): out_f32 [rows or rows/pool, ld_f32] and/or out_hi/out_lo [.., ld_split] bf16 for the
 *   next layer (columns n..ld_split-1 are written as zeros when pool == 1).  pool / rowmask as above. */
int ssd3d_linear_tc(long rows, int kp, int n, const void *a_hi, const void *a_lo, const void *b_hi, const void *b_lo,
                    const float *scale, const float *shift, int relu, int pool, const int *rowmask, float *out_f32,
                    int ld_f32, void *out_hi, void *out_lo, int ld_split, ssd3d_stream_t stream);
/* ssd3d_linear_tc for the FIRST layer of an SA scale with the gather fused into the operand load: the A operand
 * x[b,m,k,:] = concat(points[b, idx[b,m,k], :], xyz[b, idx[b,m,k], :] - new_xyz[b,m,:]) (layers_util.py:160-165) is
 * built in shared memory by producer warps instead of being materialised in HBM.  b_hi/b_lo [nout, round16(c+3)]. */
int ssd3d_linear_tc_gather(int b, int n, int c, int m, int nsample, const float *xyz, const float *points,
                           const float *new_xyz, const int *idx, int nout, const void *b_hi, const void *b_lo,
                           const float *scale, const float *shift, int relu, int pool, const int *rowmask,
                           float *out_f32, int ld_f32, void *out_hi, void *out_lo, int ld_split, ssd3d_stream_t stream);

/* "Hoisted first layer": with the first conv of an SA scale split by input rows, W1 = [Wf ; Wx],
 *   relu((concat(f_j, x_j - c_i) . W1) * s1 + t1) = relu(z[j] + (x_j - c_i) . (Wx * s1)),   z = (f . Wf) * s1 + t1,
 * the feature part is one small per-POINT GEMM (ssd3d_linear_tc on the [b*n, c] features, no ReLU) instead of a
 * per-grouped-row one, and this call runs the SECOND conv of the scale with its operand rebuilt on the fly from z
 * (z[b,n,ldz], this scale's n1 columns start at the pointer; wx = Wx*s1 as [3][n1]).  Replaces conv #1 and #2 of
 * layers_util.py:167-176 plus the grouping of :157-165; outputs as ssd3d_linear_tc. */
int ssd3d_linear_tc_hoisted(int b, int n, int n1, int m, int nsample, const float *xyz, const float *z, int ldz,
                            const float *wx, const float *new_xyz, const int *idx, int nout, const void *b_hi,
                            const void *b_lo, const float *scale, const float *shift, int relu, int pool,
                            const int *rowmask, float *out_f32, int ld_f32, void *out_hi, void *out_lo, int ld_split,
                            ssd3d_stream_t stream);
/* The operand of ssd3d_linear_tc_hoisted materialised instead of built inside the GEMM: hi/lo[b*m*nsample, kp] bf16 =
 * split(relu(z[idx] + (xyz[idx] - new_xyz) . wx)), zero padded to kp.  For wide layers (K >= 256) an elementwise pass at
 * memory speed + the plain TMA-fed ssd3d_linear_tc beats in-kernel production (lib/utils/layers_util.py:160-176). */
int ssd3d_hoist_expand_split(int b, int n, int n1, int m, int nsample, const float *xyz, const float *z, int ldz,
                             const float *wx, const float *new_xyz, const int *idx, void *hi, void *lo, int kp,
                             ssd3d_stream_t stream);
/* UNIT-LIST forms of the three calls above (units: ssd3d_query_ball_point_multi_ws).  The grouped matrix then has
 * units[0] * 8 rows: compact row 8u + e is neighbour slot 8j + e of the group unit u names, and the buffers keep their
 * full capacity (rows / b*m*nsample rows).  ssd3d_hoist_expand_split_units and ssd3d_linear_tc_hoisted_units look their
 * source rows up through the list; ssd3d_linear_tc_units consumes compact rows.  unit_pool != 0 (last conv of a scale,
 * layers_util.py:176-180): every 8-row unit is max-pooled and combined into out_f32[group, :] with atomicMax -- requires
 * relu != 0 (values >= 0), no split output, and out_f32 ZERO-FILLED by the caller (which also is the cnt == 0 mask). */
int ssd3d_hoist_expand_split_units(int b, int n, int n1, int m, int nsample, const float *xyz, const float *z, int ldz,
                                   const float *wx, const float *new_xyz, const int *idx, const int *units, void *hi,
                                   void *lo, int kp, ssd3d_stream_t stream);
int ssd3d_linear_tc_units(long rows, int kp, int n, const void *a_hi, const void *a_lo, const void *b_hi, const void *b_lo,
                          const float *scale, const float *shift, int relu, const int *units, int unit_pool,
                          float *out_f32, int ld_f32, void *out_hi, void *out_lo, int ld_split, ssd3d_stream_t stream);
int ssd3d_linear_tc_hoisted_units(int b, int n, int n1, int m, int nsample, const float *xyz, const float *z, int ldz,
                                  const float *wx, const float *new_xyz, const int *idx, const int *units, int nout,
                                  const void *b_hi, const void *b_lo, const float *scale, const float *shift, int relu,
                                  int unit_pool, float *out_f32, int ld_f32, void *out_hi, void *out_lo, int ld_split,
                                  ssd3d_stream_t stream);
/* The three unit-list calls for lists of unit_rows-row units (8 or 4, as the list was built with
 * ssd3d_query_ball_point_multi_ws_ex; nsample a multiple of it and <= 16 * unit_rows): the matrix has units[0] * unit_rows
 * rows, compact row Wu + e is neighbour slot Wj + e, and unit_pool pools every W-row unit.  Otherwise as above. */
int ssd3d_hoist_expand_split_units_ex(int b, int n, int n1, int m, int nsample, const float *xyz, const float *z, int ldz,
                                      const float *wx, const float *new_xyz, const int *idx, const int *units, void *hi,
                                      void *lo, int kp, ssd3d_stream_t stream, int unit_rows);
int ssd3d_linear_tc_units_ex(long rows, int kp, int n, const void *a_hi, const void *a_lo, const void *b_hi,
                             const void *b_lo, const float *scale, const float *shift, int relu, const int *units,
                             int unit_pool, float *out_f32, int ld_f32, void *out_hi, void *out_lo, int ld_split,
                             ssd3d_stream_t stream, int unit_rows);
int ssd3d_linear_tc_hoisted_units_ex(int b, int n, int n1, int m, int nsample, const float *xyz, const float *z, int ldz,
                                     const float *wx, const float *new_xyz, const int *idx, const int *units, int nout,
                                     const void *b_hi, const void *b_lo, const float *scale, const float *shift, int relu,
                                     int unit_pool, float *out_f32, int ld_f32, void *out_hi, void *out_lo, int ld_split,
                                     ssd3d_stream_t stream, int unit_rows);
/* Same idea for a scale that fits the fused kernel (ssd3d_sa_mlp_fused): the stack passed here starts at the scale's
 * SECOND conv, the first operand row is relu(z[idx] + (xyz[idx] - new_xyz) . wx), built during the gather. */
int ssd3d_sa_mlp_fused_hoisted(int b, int n, int n1, int m, int nsample, const float *xyz, const float *z, int ldz,
                               const float *wx, const float *new_xyz, const int *idx, const int *pts_cnt, const int *units,
                               int nl, const int *nout, const void *w_blob, const float *ss_blob, int last_scale_nonneg,
                               float *out_f32, int ld_f32, void *out_hi, void *out_lo, int ld_split, ssd3d_stream_t stream);
/* ... for a list of unit_rows-row units (8, or 4 with nsample <= 64; ignored without a list) */
int ssd3d_sa_mlp_fused_hoisted_ex(int b, int n, int n1, int m, int nsample, const float *xyz, const float *z, int ldz,
                                  const float *wx, const float *new_xyz, const int *idx, const int *pts_cnt,
                                  const int *units, int nl, const int *nout, const void *w_blob, const float *ss_blob,
                                  int last_scale_nonneg, float *out_f32, int ld_f32, void *out_hi, void *out_lo,
                                  int ld_split, ssd3d_stream_t stream, int unit_rows);
/* hi/lo[row, 0:kp] = split(x[row, 0:c]), zero padded (kp % 8 == 0). */
int ssd3d_split_rows(long rows, int c, const float *x, int ldx, void *hi, void *lo, int kp, ssd3d_stream_t stream);
/* ssd3d_group_concat fused with the split: hi/lo [b*m*nsample, kp] bf16. */
int ssd3d_group_concat_split(int b, int n, int c, int m, int nsample, const float *xyz, const float *points,
                             const float *new_xyz, const int *idx, void *hi, void *lo, int kp, ssd3d_stream_t stream);

/* A whole SA scale in one kernel (gather + concat + up to 3 conv/BN/ReLU layers + max-pool + mask,
 * lib/utils/layers_util.py:157-180) for layer stacks whose weights fit in shared memory.
 * ssd3d_sa_fused_smem returns the shared-memory bytes needed, or 0 if the stack does not fit (use the per-layer
 * path then).  w_blob / ss_blob are the pre-swizzled split weights and folded scale/shift built by the host
 * (3dssd_b200/params.py: FusedStack).  Outputs as ssd3d_linear_tc with pool = nsample.
 * last_scale_nonneg != 0: the caller guarantees scale >= 0 in the LAST layer (fold the sign of a negative BatchNorm
 * gamma into that layer's weight column -- FusedStack does); the kernel then max-pools the raw accumulators and applies
 * scale / shift / ReLU to the pooled values only (exactly the same result: the affine map is monotone).
 * units != NULL: the unit list of this scale from ssd3d_query_ball_point_multi_ws.  The kernel then convolves only the
 * listed 8-row units instead of all nsample rows of every group -- the rows it skips repeat a group's first neighbour and
 * cannot change the max-pool -- and combines the units of a group with atomicMax on out_f32, which the caller must have
 * ZERO-FILLED (zero is also the masked result of a group without neighbours); out_hi / out_lo must be NULL.  Identical
 * results; the work shrinks from b*m*nsample rows to 8 * sum(ceil(cnt / 8)), or with a list of 4-row units
 * (ssd3d_sa_mlp_fused_ex, unit_rows = 4, nsample <= 64) to 4 * sum(ceil(cnt / 4)). */
size_t ssd3d_sa_fused_smem(int c, int nl, const int *nout);
int ssd3d_sa_mlp_fused(int b, int n, int c, int m, int nsample, const float *xyz, const float *points,
                       const float *new_xyz, const int *idx, const int *pts_cnt, const int *units, int nl,
                       const int *nout, const void *w_blob, const float *ss_blob, int last_scale_nonneg, float *out_f32,
                       int ld_f32, void *out_hi, void *out_lo, int ld_split, ssd3d_stream_t stream);
int ssd3d_sa_mlp_fused_ex(int b, int n, int c, int m, int nsample, const float *xyz, const float *points,
                          const float *new_xyz, const int *idx, const int *pts_cnt, const int *units, int nl,
                          const int *nout, const void *w_blob, const float *ss_blob, int last_scale_nonneg, float *out_f32,
                          int ld_f32, void *out_hi, void *out_lo, int ld_split, ssd3d_stream_t stream, int unit_rows);

/* ---- backward operators (training graphs) ---------------------------------------------------
 * Each zero-fills its output first, as the reference's TF ops do with cudaMemset before the launcher. */

/* replaces scatteraddpointLauncher(b,n,m,c,out_g,idx,inp_g)
 *   sampling/tf_sampling.cpp:261 (decl, memset :286), sampling/tf_sampling_g.cu:408-410, kernel :335-346.
 * inp_g[b, idx[b,j], :] += out_g[b,j,:] */
int ssd3d_gather_point_grad(int b, int n, int m, int c, const float *out_g, const int *idx, float *inp_g,
                            ssd3d_stream_t stream);

/* replaces groupPointGradLauncher(b,n,c,m,nsample,grad_out,idx,grad_points)
 *   grouping/tf_grouping.cpp:479 (memset :510), grouping/tf_grouping_g.cu:480-484, kernel :383-398 (idx == -1 skipped). */
int ssd3d_group_point_grad(int b, int n, int c, int m, int nsample, const float *grad_out, const int *idx,
                           float *grad_points, ssd3d_stream_t stream);

/* replaces ThreeInterpolateGradLauncher(b,n,c,m,grad_out,idx,weight,grad_points)
 *   interpolation/tf_interpolate.cpp:363 (memset :398), interpolation/tf_interpolate_g.cu:202-206, kernel :115-140. */
int ssd3d_three_interpolate_grad(int b, int n, int c, int m, const float *grad_out, const int *idx,
                                 const float *weight, float *grad_points, ssd3d_stream_t stream);

/* Per-scene greedy BEV NMS on the GPU: replaces box_3d_to_anchor + project_to_bev + tf.image.non_max_suppression
 * of lib/builder/postprocessor.py:76-88 (one class per call).  boxes [b,n,7] = (x,y,z,l,h,w,ry), scores [b,n];
 * candidates in descending score order (ties: lower index), dropped when axis-aligned BEV IoU with a kept box is
 * > iou_threshold, at most max_output kept.  out_block [b,max_output,9] = (box7, score, class) zero padded,
 * out_cnt [b] = number kept.  n <= 16384 (PointRCNN's RPN keeps every point a candidate); max_output is bounded only
 * by the shared memory of min(n, max_output) kept boxes next to the sort keys.  Rectangles and IoU by the float32 recipe of DESIGN.md section 3.5 (cos / sin
 * in double, every operation rounded on its own); -0 and +0 scores are equal.  NaN scores are outside the contract. */
int ssd3d_bev_nms(int b, int n, const float *boxes, const float *scores, float iou_threshold, int max_output,
                  int cls_id, float *out_block, int *out_cnt, ssd3d_stream_t stream);
/* ssd3d_bev_nms over the first n_valid[s] candidates of each scene s only (DEVICE int32 [b], clamped to [0, n]); the
 * rest are padding and never kept.  With n_valid[s] == n it is ssd3d_bev_nms bit for bit (the same kernel body).
 * PointRCNN's stage 2, whose proposal rows at or past the RPN's count are padding (DESIGN.md section 3.16). */
int ssd3d_bev_nms_counted(int b, int n, const float *boxes, const float *scores, const int *n_valid, float iou_threshold,
                          int max_output, int cls_id, float *out_block, int *out_cnt, ssd3d_stream_t stream);

/* The most classes of the multi-class entry points: the eight KITTI class names of the reference
 * (g_type_mean_size, lib/utils/model_util.py:19-26), and the portable thread-block cluster size. */
#define SSD3D_MAX_CLASSES 8
/* Per-class BEV NMS of postprocessor.py:49-120 in one launch (DESIGN.md section 3.17): for every class c < cls_num
 * (1..SSD3D_MAX_CLASSES) the NMS of ssd3d_bev_nms on scores[b, n, cls_num] column c over the shared boxes [b, n, 7],
 * at most max_output boxes per class.  out_block [b, cls_num * max_output, 9] holds class 0's kept rows in kept order,
 * then class 1's, and so on, column 8 = c; out_cnt [b] = rows kept over all classes; rows at or past it are zero.  Each
 * class's rows are the bits ssd3d_bev_nms(..., cls_id = c) writes on that column, so at cls_num = 1 the block is
 * ssd3d_bev_nms's.  One thread-block cluster of cls_num CTAs per scene; fails before launching when such a cluster
 * (each CTA with the shared memory of ssd3d_bev_nms at n, max_output) cannot be placed on the device. */
int ssd3d_bev_nms_classes(int b, int n, int cls_num, const float *boxes, const float *scores, float iou_threshold,
                          int max_output, float *out_block, int *out_cnt, ssd3d_stream_t stream);

/* ---- PointRCNN's region pool (DESIGN.md section 3.16) -------------------------------------------- */

/* query_boxes_3d_points (lib/utils/tf_ops/grouping/tf_grouping_g.cu:27-94, queryBoxes3dPointsLauncher :447-449):
 * for every bottom-centred box proposals[b,m,7] = (x, y_bottom, z, l, h, w, ry) the first nsample points of xyz[b,n,3]
 * inside it, in index order, by point_inside_box_3d's arithmetic; idx[b,m,nsample] is padded with the first hit and
 * pts_cnt[b,m] = hits (<= nsample).  Rows without a hit get idx 0 (the reference leaves them unwritten; its pooler
 * zeroes them, points_pooler.py:125-126).  Indices and counts equal the reference kernel's bit for bit. */
int ssd3d_query_boxes_3d_points(int b, int n, int m, int nsample, const float *xyz, const float *proposals, int *idx,
                                int *pts_cnt, ssd3d_stream_t stream);
/* Dynamic shared memory of ssd3d_region_pool: the scene's xyz plus the conv and the index lists (<= 227 KiB). */
size_t ssd3d_region_pool_smem(int n, int nsample, int c_info);
/* PointsPooler.region_pool (lib/builder/points_pooler.py:40-61, :119-170) at inference in one launch.  Proposal r of
 * scene s is row proposals[s, r, 0:7] (row stride ld_proposals floats, e.g. 9 for the NMS block); rows r >= count[s]
 * (DEVICE int32 [b]; null: none) are padding and pool nothing.  Each real proposal grows by `context` in l, h and w
 * (expand_proposals_context, the bottom centre kept) and collects its points as ssd3d_query_boxes_3d_points
 * (idx [b,p,nsample], pts_cnt [b,p]; pool_mask = pts_cnt > 0, rows without a hit use point 0).  Per pooled point k:
 * canonical = rotate_points(xyz[k] - box[0:3], -ry), mask = point_score[s,k] >= mask_thresh, dist = |xyz[k]|, and
 * out_xyz [b*p, nsample, 3] = canonical, out_features [b*p, nsample, c_info + c_feat] =
 * [relu((canonical | mask | dist) @ info_w[5, c_info] * info_scale + info_shift) | features[s,k,0:c_feat]]
 * (roi_pool/conv0 folded as params.FoldedConv).  c_feat, c_info multiples of 4, features / out_features 16-byte
 * aligned, ssd3d_region_pool_smem(n, nsample, c_info) <= 227 KiB (n <= 16384 at nsample 512, c_info 128). */
int ssd3d_region_pool(int b, int n, int p, int nsample, int c_feat, int c_info, const float *xyz, const float *features,
                      const float *point_score, const float *proposals, int ld_proposals, const int *count, float context,
                      float mask_thresh, const float *info_w, const float *info_scale, const float *info_shift, int *idx,
                      int *pts_cnt, float *out_xyz, float *out_features, ssd3d_stream_t stream);

/* ymax[g, 0:c] = max over rows g*pool .. g*pool+pool-1 of y[., 0:c] (times rowmask[g] != 0): the
 * tf.reduce_max(axis=2) * mask of layers_util.py:178-180 for nsample values the fused epilogue of
 * ssd3d_linear_bn_relu does not cover (pool must divide 128 there). */
int ssd3d_rowgroup_max(long groups, int pool, int c, const float *y, int ldy, const int *rowmask, float *out,
                       ssd3d_stream_t stream);

/* Training-mode BatchNorm + activation of one conv output (lib/utils/tf_util.py:424-444 with is_training=True:
 * tf.contrib.layers.batch_norm(decay, updates_collections=None, fused=False), epsilon 0.001 passed as `eps`):
 * batch mean / population variance of x[rows, c] over the rows, out = act(x * inv + (beta - mean * inv)) with
 * inv = gamma * rsqrt(var + eps), and -- when moving_mean / moving_var are given -- their in-place update
 * v -= (v - batch) * (1 - decay).  scale / shift [c] receive (inv, beta - mean*inv): the folded form the inference
 * kernels take.  batch_mean / batch_var [c] are optional outputs.  workspace: ssd3d_bn_train_workspace(c) bytes.
 * x and out may alias.  Statistics couple all rows: a batch sharded over GPUs reduces them with ssd3d_bn_train_sync. */
size_t ssd3d_bn_train_workspace(int c);
int ssd3d_bn_train(long rows, int c, const float *x, int ldx, const float *gamma, const float *beta, float *moving_mean,
                   float *moving_var, float decay, float eps, void *workspace, float *scale, float *shift,
                   float *batch_mean, float *batch_var, int relu, float *out, int ldo, ssd3d_stream_t stream);

/* ---- backward of the training-mode layers (csrc/train_grad.cu, csrc/bn.cu; DESIGN.md "Backward") ----------------
 * The data gradient of a conv, grad_x = dz . W^T, needs no entry point of its own: it is ssd3d_linear_tc with the
 * split of W^T as its weight (scale 1, shift 0, no ReLU). */

/* Weight gradient of a 1x1 conv: grad_w[cin, cout] = sum_r x[r, 0:cin]^T dz[r, 0:cout], grad_b[cout] = sum_r dz[r, :]
 * (grad_b may be NULL).  x [rows, ldx], dz [rows, lddz] fp32 row-major.  Tensor cores with the bf16 hi/lo split of
 * ssd3d_linear_tc (hi.hi + lo.hi + hi.lo, fp32 accumulation), split over row ranges; the partial tiles are reduced in a
 * fixed order through the workspace (ssd3d_linear_wgrad_workspace(rows, cin, cout) bytes, 8-byte aligned), so the
 * result is the same bits from run to run. */
size_t ssd3d_linear_wgrad_workspace(long rows, int cin, int cout);
int ssd3d_linear_wgrad(long rows, int cin, int cout, const float *x, int ldx, const float *dz, int lddz, void *workspace,
                       size_t workspace_bytes, float *grad_w, float *grad_b, ssd3d_stream_t stream);
/* Backward of ssd3d_bn_train (+ its activation): x is the forward's input (the pre-BN conv output), scale / shift /
 * batch_mean / batch_var its outputs.  The ReLU mask is the forward's decision fma(x, scale, shift) > 0.
 * grad_beta = sum g, grad_gamma = sum g x^, grad_x = gamma r / N (N g - sum g - x^ sum g x^), r = rsqrt(var + eps),
 * x^ = (x - mean) r; sums in double.  grad_gamma / grad_beta may be NULL.  The moving statistics are not touched.
 * workspace: ssd3d_bn_train_grad_workspace(c) bytes, 8-byte aligned. */
size_t ssd3d_bn_train_grad_workspace(int c);
int ssd3d_bn_train_grad(long rows, int c, const float *x, int ldx, const float *grad_out, int ldg, const float *scale,
                        const float *shift, const float *batch_mean, const float *batch_var, const float *gamma, float eps,
                        int relu, void *workspace, float *grad_gamma, float *grad_beta, float *grad_x, int ldgx,
                        ssd3d_stream_t stream);
/* Backward of ssd3d_rowgroup_max: grad_y[g*pool + r, o] = (ind / num) * (grad_out[g, o] * (rowmask[g] != 0)) with
 * ind = (y == max of the group), num = number of tied maxima (TF's reduce_max gradient); rowmask may be NULL.
 * grad_out [groups, c] dense. */
int ssd3d_rowgroup_max_grad(long groups, int pool, int c, const float *y, int ldy, const int *rowmask, const float *grad_out,
                            float *grad_y, int ldgy, ssd3d_stream_t stream);
/* Backward of ssd3d_group_concat from grad_x [b, m, nsample, ldx]: grad_points [b, n, c] (columns 0:c scattered through
 * idx), grad_xyz [b, n, 3] (columns c:c+3 scattered), grad_new_xyz [b, m, 3] = -sum over the nsample rows of columns
 * c:c+3.  Any output may be NULL; the scattered ones are zero-filled first and summed with fp32 atomics. */
int ssd3d_group_concat_grad(int b, int n, int c, int m, int nsample, const int *idx, const float *grad_x, int ldx,
                            float *grad_points, float *grad_xyz, float *grad_new_xyz, ssd3d_stream_t stream);
/* Backward of ssd3d_vote_translate w.r.t. the offsets: grad_offsets[r, l] = grad_out[r, l] where
 * min_l <= offsets[r, l] <= -min_l (both bounds inclusive, as tf.maximum / tf.minimum route ties), else 0.
 * grad_out / grad_offsets [rows, 3]. */
int ssd3d_vote_translate_grad(long rows, const float *offsets, int ld_offsets, const float *grad_out, float min_x, float min_y,
                              float min_z, float *grad_offsets, ssd3d_stream_t stream);

/* ---- the small elementwise stages of the path (csrc/misc.cu) --------------------------------- */

/* points[rows, c] -> xyz[rows, 3], feat[rows, c-3]: the tf.slice pair of
 * lib/modeling/single_stage_detector.py:116-117.  feat may be NULL when c == 3. */
int ssd3d_split_points(long rows, int c, const float *points, float *xyz, float *feat, ssd3d_stream_t stream);
/* x[0:count] = 0 (fp32): the zero fill the unit-list mode of ssd3d_sa_mlp_fused needs, as a kernel of this library. */
int ssd3d_fill_zero(float *x, long count, ssd3d_stream_t stream);
/* out[s*ldo + j] = start + j, s < b, j < m: tf.tile(tf.range(npoint)) of lib/utils/layers_util.py:91-92, :100-101. */
int ssd3d_iota_idx(int b, int m, int start, int *out, int ldo, ssd3d_stream_t stream);
/* out[b,n,ca+cb] = concat(a[b,n,ca], bsrc[b,n,cb]) with scene strides in floats: tf.concat([xyz, points], -1) in
 * front of calc_square_dist (lib/utils/layers_util.py:94, :102). */
int ssd3d_concat_cols(int b, int n, int ca, int cb, const float *a, long long a_stride, const float *bsrc,
                      long long b_stride, float *out, ssd3d_stream_t stream);
/* out[b, sum(m), c] = concat along axis 1 of parts src[i][b, m[i], c] (i < parts <= 8; src / m are HOST arrays of
 * device pointers / row counts): joins the per-part results of an SA layer whose sampling was consumed in parts. */
int ssd3d_concat_rows(int b, int parts, const float *const *src, const int *m, int c, float *out, ssd3d_stream_t stream);
/* out[r, 0:3] = xyz[r, 0:3] + min(max(offsets[r, 0:3], min_xyz), -min_xyz): the clamp + add of vote_layer,
 * lib/utils/layers_util.py:20-23 (min_xyz = MODEL.MAX_TRANSLATE_RANGE, negative). */
int ssd3d_vote_translate(long rows, const float *xyz, const float *offsets, int ld_offsets, float min_x, float min_y,
                         float min_z, float *out, ssd3d_stream_t stream);
/* decode_dist_anchor_free + decode_class2angle + the score sigmoid (lib/utils/anchor_decoder.py:86-112, :6-14,
 * lib/modeling/single_stage_detector.py:210-211) in one pass.  pred_reg[rows, ld_reg] = [6 face distances |
 * angle_bins logits | angle_bins residuals], pred_cls[rows, ld_cls] (column 0 = the class logit), center_xyz[rows,3]
 * -> boxes[rows,7] = (x, y, z, l, h, w, ry), scores[rows]. */
int ssd3d_decode_dist_anchor_free(long rows, int angle_bins, const float *center_xyz, const float *pred_reg, int ld_reg,
                                  const float *pred_cls, int ld_cls, float *boxes, float *scores, ssd3d_stream_t stream);
/* ssd3d_decode_dist_anchor_free with cls_num (1..SSD3D_MAX_CLASSES, <= ld_cls) sigmoid scores per row:
 * scores[rows, cls_num], column c from pred_cls column c as the single-class form computes column 0; the same boxes. */
int ssd3d_decode_dist_anchor_free_classes(long rows, int angle_bins, int cls_num, const float *center_xyz, const float *pred_reg,
                                          int ld_reg, const float *pred_cls, int ld_cls, float *boxes, float *scores,
                                          ssd3d_stream_t stream);
/* decode_bin_anchor on the anchors of generate_3d_anchors_by_point_tf + the score sigmoid (lib/utils/anchor_decoder.py:
 * 115-164, lib/utils/generate_anchors.py:33-65; PointRCNN's 'Bin-Anchor' regression, one anchor size per point).
 * pred_reg[rows, ld_reg] = [x_bin | x_res | z_bin | z_res (bin_num each) | y_res | 3 size residuals | angle_bins logits |
 * angle_bins residuals], pred_cls[rows, ld_cls] (column 0), center_xyz[rows,3], anchor_lhw = host float[3] ->
 * boxes[rows,7] = (x, y, z, l, h, w, ry), scores[rows].  TF's fp32 operation order, one rounding per operation; argmax
 * ties to the first index. */
int ssd3d_decode_bin_anchor(long rows, int bin_num, float half_bin_search_range, int angle_bins, const float *center_xyz,
                            const float *pred_reg, int ld_reg, const float *pred_cls, int ld_cls, const float *anchor_lhw,
                            float *boxes, float *scores, ssd3d_stream_t stream);
/* decode_bin_anchor against per-row anchors (lib/utils/anchor_decoder.py:115-164 as PointRCNN's stage 2 calls it,
 * double_stage_detector.py:298-337): anchors[rows, ld_anchors] = the bottom-centred proposals (x, y, z, l, h, w, ry),
 * pred_reg as ssd3d_decode_bin_anchor, y = anchor y + y_res, sizes = anchor size + residual (>= 0.1), ry = anchor ry +
 * the decoded angle; scores[rows] = softmax(pred_cls[r, 0:2])[1] (in double, rounded once) times (pool_cnt[r] > 0)
 * (pool_cnt may be null: no mask).  TF's fp32 operation order; argmax ties to the first index. */
int ssd3d_decode_bin_anchor_rows(long rows, int bin_num, float half_bin_search_range, int angle_bins, const float *anchors,
                                 int ld_anchors, const float *pred_reg, int ld_reg, const float *pred_cls, int ld_cls,
                                 const int *pool_cnt, float *boxes, float *scores, ssd3d_stream_t stream);

/* ---- training targets and detection losses (csrc/det_loss.cu, DESIGN.md section 3.8) -------- */

/* 'Mask' target assignment and vote targets of the shipped 3DSSD configuration in one launch, one CTA per scene:
 * TargetAssigner.assign + mask_assign_targets_anchors_np + vote_targets_np (lib/builder/target_assigner.py:147,
 * lib/np_functions/gt_sampler.py:168-259, :28-61) with the encode step of the regression targets.
 * gt_boxes [b, g, 7] (x, y, z, l, h, w, ry; a row of seven zeros is padding and is skipped, any g >= 0),
 * gt_labels [b, g] int32.  For each candidate point base_xyz [b, n, 3]:
 *   inside        the face-plane test of check_inside_points (lib/utils/voxelnet_aug.py:318-342, :532-567): a point
 *                 is outside a box as soon as one face gives sign >= 0, so a point on a face is outside;
 *   assigned_idx  [b, n] int32: the first valid box that contains the point, else the first valid box;
 *   assigned_box  [b, n, 7]: that box;
 *   pmask [b, n]  inside && |base_xyz - box[:3]| <= 10;  nmask [b, n] = !inside (inside but beyond 10 m: neither);
 *   cls_label     [b, n]: the centre-ness label (lib/builder/loss_builder.py:99-137) of a positive whose box has
 *                 label 1, else 0 (the label one_hot(label - 1) * centre-ness of the one class);
 *   angle_bin     [b, n] int32, angle_res [b, n]: encode_angle2class of the box's ry with float32 floor-mods
 *                 (lib/utils/anchor_encoder.py:9-33; a bin that rounds to angle_bins is clamped to angle_bins - 1);
 *   offset_target [b, n, 6]: encode_dist_anchor_free (anchor_encoder.py:151-173): box centre moved up by h/2 minus
 *                 base_xyz, then l/2, h/2, w/2.
 * For each vote base point vote_base [b, nv, 3], against the boxes grown by 0.1 in l, h and w (gt_sampler.py:28-61):
 *   vote_mask [b, nv], vote_target [b, nv, 3] = (x, y - h/2, z) of the first (unexpanded) box whose expansion holds the
 *   point, else of the first valid box, minus the point.
 * A scene without a valid box: every point is a negative, assigned_idx / assigned_box / cls_label / angle_bin /
 * angle_res / offset_target / vote_mask / vote_target are 0.  float32 targets made of + - * / are the bits of the
 * reference's float32 numpy / TF arithmetic; the centre-ness label is evaluated in double and rounded once. */
int ssd3d_det_assign(int b, int n, int nv, int g, int angle_bins, const float *base_xyz, const float *vote_base,
                     const float *gt_boxes, const int *gt_labels, int *assigned_idx, float *assigned_box, float *pmask,
                     float *nmask, float *cls_label, int *angle_bin, float *angle_res, float *offset_target, float *vote_mask,
                     float *vote_target, ssd3d_stream_t stream);
/* ssd3d_det_assign for cls_num classes (1..SSD3D_MAX_CLASSES; labels 1..cls_num): every target but cls_label is the
 * class-agnostic one of ssd3d_det_assign, bit for bit.  cls_label [b, n, cls_num]: column c is the centre-ness label of
 * a positive whose box has label c + 1, else 0 (one_hot(label - 1, cls_num) * centre-ness, loss_builder.py:58-96); a
 * label outside 1..cls_num gives a zero row and stays a regression positive. */
int ssd3d_det_assign_classes(int b, int n, int nv, int g, int angle_bins, int cls_num, const float *base_xyz,
                             const float *vote_base, const float *gt_boxes, const int *gt_labels, int *assigned_idx,
                             float *assigned_box, float *pmask, float *nmask, float *cls_label, int *angle_bin, float *angle_res,
                             float *offset_target, float *vote_mask, float *vote_target, ssd3d_stream_t stream);
/* The six losses of LossBuilder.forward (loss_builder.py) for 'Center-ness' sigmoid classification, 'Dist-Anchor-free'
 * regression, the corner loss and the vote loss, from the head outputs read in place through row strides
 * (pred_cls [b, n, ld_cls] column 0, pred_offset [.., ld_offset] columns 0:6, pred_angle_cls / pred_angle_res columns
 * 0:angle_bins), the raw vote offsets vote_offset [b, nv, ld_vote] and the targets of ssd3d_det_assign.  The
 * regression target is encoded again from assigned_box and base_xyz (the bits of offset_target for the same points), so
 * the loss is a function of the base_xyz it differentiates.
 * loss[6] = cls, offset, angle bin, angle residual, corner, vote; norm[3] = max(1, sum) of the classification mask
 * (pmask + nmask), of pmask and of vote_mask over the whole batch.  The corner loss decodes the predicted box with the
 * GT angle bin (single_stage_detector.py:173-177).  Each term is summed per scene, then over the scenes in order, in
 * double; transcendentals and loss arithmetic run in double and each result is rounded once.
 * workspace: ssd3d_det_loss_workspace(b) bytes, 8-byte aligned. */
size_t ssd3d_det_loss_workspace(int b);
int ssd3d_det_loss(int b, int n, int nv, int angle_bins, const float *base_xyz, const float *pred_cls, int ld_cls,
                   const float *pred_offset, int ld_offset, const float *pred_angle_cls, int ld_angle_cls,
                   const float *pred_angle_res, int ld_angle_res, const float *vote_offset, int ld_vote,
                   const float *assigned_box, const float *pmask, const float *nmask, const float *cls_label,
                   const int *angle_bin, const float *angle_res, const float *vote_mask, const float *vote_target,
                   void *workspace, float *loss, float *norm, ssd3d_stream_t stream);
/* ssd3d_det_loss for cls_num sigmoid classes (1..SSD3D_MAX_CLASSES): pred_cls columns 0:cls_num (ld_cls >= cls_num),
 * cls_label [b, n, cls_num] of ssd3d_det_assign_classes.  The classification term of a row is the mean over the classes
 * of the sigmoid cross-entropy, summed over the classes in order in double; the other five losses are ssd3d_det_loss's.
 * At cls_num = 1 it is ssd3d_det_loss bit for bit. */
int ssd3d_det_loss_classes(int b, int n, int nv, int angle_bins, int cls_num, const float *base_xyz, const float *pred_cls,
                           int ld_cls, const float *pred_offset, int ld_offset, const float *pred_angle_cls, int ld_angle_cls,
                           const float *pred_angle_res, int ld_angle_res, const float *vote_offset, int ld_vote,
                           const float *assigned_box, const float *pmask, const float *nmask, const float *cls_label,
                           const int *angle_bin, const float *angle_res, const float *vote_mask, const float *vote_target,
                           void *workspace, float *loss, float *norm, ssd3d_stream_t stream);
/* Backward of ssd3d_det_loss from grad_loss[6] (device) and the norm[3] it wrote: grad_base_xyz [b, n, 3] (through the
 * offset target and the corner loss's decoded box; none through the centre-ness label, which TF stops),
 * grad_cls / grad_offset / grad_angle_cls / grad_angle_res with row strides ldg_* (the residual gradient only at the
 * GT bin; lhw = max(2 * half, 0.1) routes a tie to 2 * half), grad_vote_offset [b, nv, 3].  Rows no term touches get
 * exactly 0.  One thread per row, no atomics. */
int ssd3d_det_loss_grad(int b, int n, int nv, int angle_bins, const float *base_xyz, const float *pred_cls, int ld_cls,
                        const float *pred_offset, int ld_offset, const float *pred_angle_cls, int ld_angle_cls,
                        const float *pred_angle_res, int ld_angle_res, const float *vote_offset, int ld_vote,
                        const float *assigned_box, const float *pmask, const float *nmask, const float *cls_label,
                        const int *angle_bin, const float *angle_res, const float *vote_mask, const float *vote_target,
                        const float *grad_loss, const float *norm, float *grad_base_xyz,
                        float *grad_cls, int ldg_cls, float *grad_offset, int ldg_offset, float *grad_angle_cls,
                        int ldg_angle_cls, float *grad_angle_res, int ldg_angle_res, float *grad_vote_offset,
                        ssd3d_stream_t stream);
/* Backward of ssd3d_det_loss_classes: grad_cls columns 0:cls_num (ldg_cls >= cls_num) = (sigmoid(x_c) - label_c) *
 * cls_mask * grad_loss[0] / norm[0] / cls_num; every other gradient is ssd3d_det_loss_grad's.  At cls_num = 1 it is
 * ssd3d_det_loss_grad bit for bit. */
int ssd3d_det_loss_grad_classes(int b, int n, int nv, int angle_bins, int cls_num, const float *base_xyz, const float *pred_cls,
                                int ld_cls, const float *pred_offset, int ld_offset, const float *pred_angle_cls, int ld_angle_cls,
                                const float *pred_angle_res, int ld_angle_res, const float *vote_offset, int ld_vote,
                                const float *assigned_box, const float *pmask, const float *nmask, const float *cls_label,
                                const int *angle_bin, const float *angle_res, const float *vote_mask, const float *vote_target,
                                const float *grad_loss, const float *norm, float *grad_base_xyz,
                                float *grad_cls, int ldg_cls, float *grad_offset, int ldg_offset, float *grad_angle_cls,
                                int ldg_angle_cls, float *grad_angle_res, int ldg_angle_res, float *grad_vote_offset,
                                ssd3d_stream_t stream);

/* ---- sharded step: exchange over NVLink peer memory ---------------------------------------- */

/* All-gather of one slice per rank as ONE kernel (csrc/peer_gather.cu): no reference counterpart (the reference's
 * inference is single-GPU, lib/core/evaluator.py:145-147); replaces the ncclAllGather of the per-scene detection blocks at
 * the end of a sharded step.  peer_base: DEVICE array [world] with the base address of every rank's symmetric buffer as
 * mapped in this process (e.g. torch.distributed._symmetric_memory buffer_ptrs); inside it, for parity q in {0,1}:
 * recv_off<q> = world slices of slice_bytes, flag_off<q> = world int32 flags, all zero before the first call.  The call
 * stores src into slot `rank` of every peer's receive area, publishes replay number s (kept in state[0], so a captured
 * launch needs no changing argument; state = 3 zero-initialised ints owned by this exchange) with release semantics at
 * system scope, waits for the peers' flags and copies the received slices to out[world][slice_bytes].  Every rank must
 * make the same sequence of calls; two parities make reuse safe without acknowledgements.  A wait of ~4 s gives up and
 * increments state[2] instead of hanging the GPU. */
int ssd3d_peer_allgather(const void *src, size_t slice_bytes, void *const *peer_base, int world, int rank,
                         size_t recv_off0, size_t recv_off1, size_t flag_off0, size_t flag_off1, int *state, void *out,
                         ssd3d_stream_t stream);

/* ---- data-parallel training: the per-step gradient exchange (csrc/grad_exchange.cu, DESIGN.md section 3.9) ---------
 * The reference's towers (lib/core/trainer.py:143-154, lib/utils/trainer_utils.py:23-46) with pinned arithmetic:
 * clip each rank's gradient, average the clipped gradients in rank order, apply every rank's BatchNorm statistics.
 * None allocates, uses float atomics or synchronises the host; all are CUDA-graph capturable. */

/* Global norm and clip scale of one rank's flat gradient grad[n]: *norm = float32(sqrt(sum grad^2)), the sum in double
 * over a fixed tree (256 blocks of 256 threads, each thread in index order, then a halving tree in the block and over
 * the block partials), so the same bits every run; *scale = rn(clip_norm * minimum(rn(1 / use_norm), rn(1 / clip_norm)))
 * with use_norm = *norm when finite, else NaN (tf.clip_by_global_norm in float32; the NaN propagates).  norm and scale
 * are device floats.  workspace: ssd3d_grad_clip_scale_workspace(n) bytes, 8-byte aligned. */
size_t ssd3d_grad_clip_scale_workspace(long n);
int ssd3d_grad_clip_scale(const float *grad, long n, float clip_norm, void *workspace, float *norm, float *scale,
                          ssd3d_stream_t stream);
/* Mean of the ranks' clipped gradients, written back into every rank's grad[n] (16-byte aligned):
 * grad[i] = float32((sum over r = 0..world-1 of (double) rn(grad_r[i] * scale_r)) / world), scale = this rank's device
 * scalar of ssd3d_grad_clip_scale.  ONE launch of `ctas` CTAs: reduce-scatter plus all-gather over the symmetric
 * buffers (peer_base as in ssd3d_peer_allgather).  Rank p owns floats [p*chunk, (p+1)*chunk), cut into sub-slices of
 * `sub` floats, one per CTA (chunk and sub multiples of 4, chunk*world >= n, sub*ctas >= chunk).  Inside every rank's
 * symmetric buffer, per parity q in {0,1}: r1_off<q> and r2_off<q> = world*chunk floats, f1_off<q> and f2_off<q> =
 * world*ctas int32 flags, all zero before the first call.  state = 3 zero-initialised ints owned by this exchange
 * ([0] replays done, [2] waits that gave up after ~4 s; a CTA whose wait gave up writes NaN into its part of grad).
 * All `ctas` CTAs must be co-resident on the device: at most
 * ssd3d_peer_allreduce_resident_ctas() less whatever else runs there.  Every rank makes the same sequence of calls. */
int ssd3d_peer_allreduce_resident_ctas(void);
int ssd3d_peer_allreduce_mean(float *grad, size_t n, const float *scale, void *const *peer_base, int world, int rank, int ctas,
                              size_t chunk, size_t sub, size_t r1_off0, size_t r1_off1, size_t r2_off0, size_t r2_off1,
                              size_t f1_off0, size_t f1_off1, size_t f2_off0, size_t f2_off1, int *state,
                              ssd3d_stream_t stream);
/* The BatchNorm moving-average update of `world` ranks, in rank order: for r = 0..world-1,
 * stats[i] = rn(stats[i] - rn(rn(stats[i] - batch[r*ld_batch + i]) * rn(1 - decay))), the update of ssd3d_bn_train.
 * stats[n] and each rank's batch[.., n] hold means and variances at the same offsets. */
int ssd3d_bn_moving_update_ranks(float *stats, long n, const float *batch, long ld_batch, int world, float decay,
                                 ssd3d_stream_t stream);

/* SyncBN (csrc/bn.cu, DESIGN.md section 3.18): ssd3d_bn_train / ssd3d_bn_train_grad of a batch sharded over `world` ranks.
 * Each is the same partial kernel, then ONE exchange-and-finalize launch of ceil(c / 128) CTAs, then the same apply
 * kernel.  The exchange adds every rank's per-channel (rows, sum, sum of squares) -- backward: (rows, sum g, sum g x^) --
 * in rank order in double, so the statistics (and the backward's coef) are those of all ranks' rows and every rank holds
 * the same bits; with world = 1 the results equal the plain calls bit for bit.  The moving statistics are updated in
 * place with the global statistics; grad_gamma / grad_beta stay this rank's own sums.
 * peer_base: DEVICE array [world] of every rank's symmetric allocation as mapped here; area_off (16-byte multiple): the
 * byte offset, in every rank's allocation, of this (scope, direction)'s area of ssd3d_bn_sync_area_bytes(world, c)
 * bytes, zero-initialised; state: int32 [>= 3] zero-initialised, owned by this (scope, direction): [0] replays,
 * [2] waits that gave up after ~4 s (that CTA's channels then come out NaN).  Every rank makes the same sequence of
 * calls per area; the world's exchange CTAs of one call must be co-resident (ssd3d_bn_sync_resident_ctas per device).
 * Capturable: no host sync, no allocation, no float atomics. */
size_t ssd3d_bn_sync_area_bytes(int world, int c);
int ssd3d_bn_sync_resident_ctas(void);
int ssd3d_bn_train_sync(long rows, int c, const float *x, int ldx, const float *gamma, const float *beta, float *moving_mean,
                        float *moving_var, float decay, float eps, void *workspace, float *scale, float *shift,
                        float *batch_mean, float *batch_var, int relu, float *out, int ldo, void *const *peer_base, int world,
                        int rank, size_t area_off, int *state, ssd3d_stream_t stream);
int ssd3d_bn_train_grad_sync(long rows, int c, const float *x, int ldx, const float *grad_out, int ldg, const float *scale,
                             const float *shift, const float *batch_mean, const float *batch_var, const float *gamma, float eps,
                             int relu, void *workspace, float *grad_gamma, float *grad_beta, float *grad_x, int ldgx,
                             void *const *peer_base, int world, int rank, size_t area_off, int *state, ssd3d_stream_t stream);

/* ---- the solver: Adam, Momentum and the weight operands (csrc/solver.cu, DESIGN.md sections 3.11, 3.19) -------------
 * The updates of tf.train.AdamOptimizer and tf.train.MomentumOptimizer (lib/core/trainer.py:72-75) under the
 * learning-rate schedule of tf.train.piecewise_constant (lib/core/trainer_utils.py:7-13), with every float32 operation
 * rounded once.  No entry allocates, uses float atomics or synchronises the host; all are CUDA-graph capturable. */

/* One Adam step over flat buffers param, m, v (updated in place) and grad [n], all 16-byte aligned, in ONE launch.
 * state: the caller's 32-byte, 8-byte aligned device block { int64 global_step; float beta1_power; float beta2_power;
 * float lr_used; uint32 done; uint32 reserved[2] }, initialised to { 0, beta1, beta2, 0, 0, 0, 0 }; `done` is the
 * launch's own block counter and is 0 between launches.  boundaries [nb] (increasing, nb <= 8) and values [nb + 1] are
 * HOST arrays copied into the launch.  With the state as it was BEFORE the launch:
 *   lr    = values[k], k = number of boundaries < global_step   (values[0] while global_step <= boundaries[0])
 *   alpha = rn(rn(lr * rn(sqrt(rn(1 - beta2_power)))) / rn(1 - beta1_power))
 *   m = rn(m + rn(rn(g - m) * rn(1 - beta1)));  v = rn(v + rn(rn(rn(g * g) - v) * rn(1 - beta2)))
 *   param = rn(param - rn(rn(m * alpha) / rn(rn(sqrt(v)) + epsilon)))
 * and, once every element is done: beta1_power = rn(beta1_power * beta1), beta2_power likewise, global_step += 1,
 * lr_used = lr.  Non-finite gradients propagate. */
int ssd3d_adam_step(float *param, const float *grad, float *m, float *v, long n, void *state, float beta1, float beta2,
                    float epsilon, int nb, const long long *boundaries, const float *values, ssd3d_stream_t stream);
/* One step of tf.train.MomentumOptimizer(lr, momentum), use_nesterov=False (TF's ApplyMomentum), over flat buffers param
 * and accum (updated in place) and grad [n], all 16-byte aligned, in ONE launch.  state, boundaries, values and the
 * launch protocol are those of ssd3d_adam_step; momentum is in [0, 1] and accum starts at 0.  With lr read from the
 * state as it was BEFORE the launch:
 *   accum = rn(rn(accum * momentum) + g);  param = rn(param - rn(accum * lr))
 * and, once every element is done: global_step += 1, lr_used = lr.  beta1_power and beta2_power are not touched.
 * Non-finite gradients propagate. */
int ssd3d_momentum_step(float *param, const float *grad, float *accum, long n, void *state, float momentum, int nb,
                        const long long *boundaries, const float *values, ssd3d_stream_t stream);
/* The split-bf16 tensor-core operands of nw conv weights, rebuilt from the flat parameter buffer in ONE launch.
 * table: DEVICE int64 [nw][8], row = { offset of W [cin, cout] in param (floats), cin, cout, then offsets in arena (bf16
 * elements, multiples of 8) of fwd_hi, fwd_lo [cout, round16(cin)] = split of W^T and of bwd_hi, bwd_lo
 * [cin, round16(cout)] = split of W, then tile_start }.  hi = bf16_rne(w), lo = bf16_rne(w - float(hi)); padding
 * columns are +0.  A weight takes ceil(round16(cin) / 32) * ceil(round16(cout) / 32) tiles; tile_start is the running
 * sum over the rows before it and `tiles` the total.  arena: 16-byte aligned. */
int ssd3d_weight_operands(const float *param, const long long *table, int nw, long tiles, void *arena,
                          ssd3d_stream_t stream);

/* ---- KITTI evaluation (csrc/box_eval.cu, DESIGN.md section 3.10; evaluation/evaluate.cpp, tf_evaluate.cpp) ----------
 * Boxes are (x, y, z, l, h, w, ry), camera frame, origin at the bottom-face centre.  Overlaps are computed in double by
 * the recipe of DESIGN.md section 3.10; a pair whose union area or volume is <= 0 has overlap 0.
 * calc_iou (tf_evaluate.cpp:35-48): iou_bev, iou_3d [b, n, m] = rotated BEV / 3-D IoU of dets [b, n, 7] x gts [b, m, 7]. */
int ssd3d_box_iou(int b, int n, int m, const float *dets, const float *gts, float *iou_bev, float *iou_3d,
                  ssd3d_stream_t stream);
/* calc_iou_match (tf_evaluate.cpp:50-63): iou_bev[i], iou_3d[i] of dets[i] [n, 7] against gts[i] [n, 7]. */
int ssd3d_box_iou_matched(long n, const float *dets, const float *gts, float *iou_bev, float *iou_3d, ssd3d_stream_t stream);
/* The Evaluate op (tf_evaluate.cpp:14-33) in three launches.  Frames are CSR-packed: dets [N, 14] float rows (class, x1,
 * y1, x2, y2, alpha, t1, t2, t3, h, w, l, ry, score) with frame f at rows det_off[f] .. det_off[f+1]-1; labels [R, 15]
 * DOUBLE rows (the 15 fields of a KITTI label line, the type replaced by 0 Car, 1 Pedestrian, 2 Cyclist, 3 Van,
 * 4 Person_sitting, 5 DontCare, 6 other) indexed by label_off; pair_off [frames] int64 = sum over earlier frames of
 * (detections * label rows).  Every frame holds at most max_dets <= 1024 detections and max_labels <= 256 label rows.
 * Cases are numbered metric * 9 + class * 3 + difficulty (metric: image, ground, 3-D).
 * Workspace of ssd3d_eval_overlaps: ssd3d_eval_workspace(total pairs) bytes, 8-byte aligned. */
size_t ssd3d_eval_workspace(long pairs);
int ssd3d_eval_overlaps(int frames, int max_dets, int max_labels, const float *dets, const int *det_off,
                        const double *labels, const int *label_off, const long *pair_off, void *workspace,
                        ssd3d_stream_t stream);
/* First pass of computeStatistics (evaluate.cpp:649-830, no false positives counted), all 27 cases in one launch:
 * tp_scores[case * label_rows + label_off[f] + k] for k < tp_count[case * frames + f]; n_gt[case * frames + f]. */
int ssd3d_eval_first_pass(int frames, int max_dets, int max_labels, const float *dets, const int *det_off,
                          const double *labels, const int *label_off, const long *pair_off, const void *workspace,
                          long label_rows, double *tp_scores, int *tp_count, int *n_gt, ssd3d_stream_t stream);
/* Counting pass at each case's score thresholds (thresholds [27, 41] double, n_thresholds [27] <= 41, from getThresholds,
 * evaluate.cpp:539-572): counts [27, 41, 3] int = tp, fp, fn summed over the frames (cleared here first). */
int ssd3d_eval_count(int frames, int max_dets, int max_labels, const float *dets, const int *det_off,
                     const double *labels, const int *label_off, const long *pair_off, const void *workspace,
                     const double *thresholds, const int *n_thresholds, int *counts, ssd3d_stream_t stream);

/* ---- training-scene augmentation (csrc/augment.cu, DESIGN.md section 3.12) -----------------------------------------
 * DataAugmentor.kitti_forward of 3dssd.yaml after the mixup paste (flip, per-object noise, global rotation and scale,
 * the context filter) and the point choice of kitti_dataloader.py:137-147, on ragged scenes: points [T, 4] (x, y, z,
 * intensity) with scene s at rows offsets[s] .. offsets[s+1]-1 (DEVICE int32 [b+1]), gt_boxes [b, g, 7] (x, y, z, l, h, w,
 * ry) zero-padded, gt_labels [b, g].  Limits: g <= 256, 1 <= points per scene <= max_n <= 131072, num_points <= 16384.
 * Every random number comes from the draw block: scene_u [b, 6] (flip, c0, c1, c2, rotation, scale), loc_noise
 * [b, g, 100, 2] standard normals (x, z), rot_u [b, g, 100] uniforms, keys [T] and refill [b, num_points] uint32.  The
 * same draws give the same bits; nothing synchronises the host.  Workspace: ssd3d_augment_workspace(b, g) bytes,
 * 256-byte aligned, written by ssd3d_augment_boxes and read by ssd3d_augment_points. */
size_t ssd3d_augment_workspace(int b, int g);
/* sem_labels [T] = class of the first valid box grown by 0.1 that holds the point, else 0 (kitti_dataloader.py:211-219). */
int ssd3d_augment_sem_labels(int b, int g, int max_n, const float *points, const int *offsets, const float *gt_boxes,
                             const int *gt_labels, int *sem_labels, ssd3d_stream_t stream);
/* Flip, noise search, box transforms, global rotation and scale, context-filter dims: out_boxes [b, g, 7];
 * chosen_try [b, g] = the try a box took, -1 when all 100 collided (the box keeps the identity transform) or padded. */
int ssd3d_augment_boxes(int b, int g, const float *gt_boxes, const double *scene_u, const double *loc_noise,
                        const double *rot_u, float *out_boxes, int *chosen_try, void *workspace, ssd3d_stream_t stream);
/* out_points [T, 4] transformed; sort_keys [T] = keys << 32 | index in the scene for a survivor of the context filter,
 * all ones for a dropped point; survivors [b] counts (cleared here); moved_by [T] (may be NULL) = the box that moved the
 * point or -1.  A negative semantic label marks a slot that holds no point (a dropped object of the mixup layout): it
 * is not moved, its sort key is all ones, it is not a survivor, moved_by is -1 and its output is zeros. */
int ssd3d_augment_points(int b, int g, int max_n, const float *points, const int *offsets, const int *sem_labels,
                         const unsigned *keys, const void *workspace, float *out_points, unsigned long long *sort_keys,
                         int *survivors, int *moved_by, ssd3d_stream_t stream);
/* out [b, num_points, 4]: with N = survivors[s], the min(N, num_points) survivors of smallest sort key in key order, then
 * for slot t >= N the survivor at rank (refill[s, t] * N) >> 32.  A scene without survivors gets zeros. */
int ssd3d_augment_choose(int b, int num_points, const float *points, const int *offsets, const unsigned long long *sort_keys,
                         const int *survivors, const unsigned *refill, float *out, ssd3d_stream_t stream);

/* ---- mixup paste and its object database (csrc/mixup.cu, DESIGN.md section 3.13) ------------------------------------
 * Scenes as for the augmentation: points [T, 4], DEVICE offsets [b + 1], gt_boxes [b, g, 7] zero-padded, gt_labels [b, g].
 * Database: db_points [P, 4] with object o at rows db_offsets[o] .. db_offsets[o+1]-1 (int64), db_boxes [O, 7],
 * db_classes [O].  Limits: g + s <= 256, points per scene before and after the paste <= 131072.  Nothing synchronises the
 * host; the same inputs give the same bits. */
/* counts [b, g] (cleared here) = the points of each frame inside each valid row grown by 0.1 on (l, h, w). */
int ssd3d_mixup_db_count(int b, int g, int max_n, const float *points, const int *offsets, const float *gt_boxes,
                         int *counts, ssd3d_stream_t stream);
/* out_points rows object_offsets[o] .. object_offsets[o+1]-1 = the points of frame objects[o, 0] inside its row
 * objects[o, 1] grown by 0.1, in frame order (object_offsets from the counts of ssd3d_mixup_db_count). */
int ssd3d_mixup_db_write(int g, int n_objects, const float *points, const int *offsets, const float *gt_boxes,
                         const int *objects, const long long *object_offsets, float *out_points, ssd3d_stream_t stream);
/* box_3d_collision_test of the s drawn objects ids [b, s] (-1: none) against each scene: drawn box i with (l, w) grown by
 * 0.5 is kept iff it collides with no valid scene row and no kept drawn box k < i; a kept box stands on the scene's plane
 * planes [b, 4] float64 (a, b, c, d), y -= y - (-d - a x - c z) / b.  out_boxes [b, g + s, 7] / out_labels [b, g + s] = the
 * valid scene rows in order, the kept boxes in draw order (label db_classes[id]), zero rows; accepted [b, s] 0 / 1. */
int ssd3d_mixup_paste_boxes(int b, int g, int s, const float *gt_boxes, const int *gt_labels, const int *ids,
                            const float *db_boxes, const int *db_classes, const double *planes, float *out_boxes,
                            int *out_labels, int *accepted, ssd3d_stream_t stream);
/* Scene s's output slots out_offsets[s] .. out_offsets[s+1]-1 (DEVICE int32 [b + 1]): its points with their semantic
 * labels, then drawn object i at slots slot_start[s, i] .. slot_start[s, i+1]-1 (DEVICE int32 [b, s + 1], slot_start[s, 0]
 * = the scene's point count): the database points with y moved as the box when accepted (label db_classes[id]), else
 * zeros with label -1.  max_slots = the largest scene after the paste. */
int ssd3d_mixup_paste_points(int b, int s, int max_slots, const float *points, const int *offsets, const int *sem_labels,
                             const int *ids, const float *db_points, const long long *db_offsets, const float *db_boxes,
                             const int *db_classes, const double *planes, const int *accepted, const int *out_offsets,
                             const int *slot_start, float *out_points, int *out_sem_labels, ssd3d_stream_t stream);

/* ---- KITTI preprocessing (csrc/prepare.cu, DESIGN.md section 3.14) --------------------------------------------------
 * A batch of b raw velodyne frames: points [total, 4] float32 (x, y, z, intensity) packed frame after frame, DEVICE
 * offsets [b + 1] int32, calib [b, 33] float64 per frame (Tr_velo_to_cam V [3, 4], R0_rect R [3, 3], P2 P [3, 4], each
 * row-major), image_hw [b, 2] int32 (H, W > 0), extents [6] float64 (x0, x1, y0, y1, z0, z1 of the rect frame).  Limits:
 * b <= 4096 frames, max_n (the largest frame) <= 262144 points, total <= 16777216 points.  In float64, every product,
 * sum and quotient rounded once and the inputs widened exactly from float32:
 *   ref_j  = ((x V[j,0] + y V[j,1]) + z V[j,2]) + V[j,3]
 *   rect_i = (R[i,0] ref_0 + R[i,1] ref_1) + R[i,2] ref_2
 *   h_k    = ((rect_0 P[k,0] + rect_1 P[k,1]) + rect_2 P[k,2]) + P[k,3],   u = h_0 / h_2,  v = h_1 / h_2
 * a point is kept iff 0 <= u < W, 0 <= v < H, rect_2 >= 0 and x0 < rect_0 < x1, y0 < rect_1 < y1, z0 < rect_2 < z1 (a NaN
 * fails every test).  out_points [total, 4] float64: rows out_offsets[s] .. out_offsets[s+1]-1 (DEVICE int32 [b + 1], an
 * exclusive scan of the kept counts) hold frame s's kept points (rect_0, rect_1, rect_2, intensity) in input order; rows
 * from out_offsets[b] on are not written.  No atomics, nothing synchronises the host; the same inputs give the same bits.
 * Workspace: ssd3d_prepare_workspace(b, max_n) bytes (0 when a limit is exceeded). */
#define SSD3D_PREPARE_MAX_FRAMES 4096
#define SSD3D_PREPARE_MAX_FRAME_POINTS 262144
#define SSD3D_PREPARE_MAX_BATCH_POINTS 16777216
size_t ssd3d_prepare_workspace(int b, int max_n);
int ssd3d_prepare_points(int b, int max_n, int total, const float *points, const int *offsets, const double *calib,
                         const int *image_hw, const double *extents, void *workspace, double *out_points, int *out_offsets,
                         ssd3d_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* SSD3D_H_ */
