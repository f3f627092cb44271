"""The reference's `tf_ops` operator surface on torch CUDA tensors.

Same function names, argument orders and error behaviour as
  /root/reference/lib/utils/tf_ops/sampling/tf_sampling.py      (:24 gather_point, :43 farthest_point_sample,
                                                                  :54 farthest_point_sample_with_distance)
  /root/reference/lib/utils/tf_ops/grouping/tf_grouping.py      (:53 query_ball_point, :68 query_ball_point_dilated,
                                                                  :114 group_point)
  /root/reference/lib/utils/tf_ops/interpolation/tf_interpolate.py (:8 three_nn, :21 three_interpolate)
with the TF custom-op layer replaced by ctypes calls into libssd3d.so (include/ssd3d.h).  Shape / attribute
checks mirror the reference's OP_REQUIRES (InvalidArgument -> ValueError); outputs are allocated here, like
TF's allocate_output, and the kernels run on torch's current stream (CUDA-graph capturable).
"""
import ctypes
import math

import numpy as np
import torch

from ._lib import check, lib
from .params import BN_EPS, FoldedConv, round16


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _req(t, name, dtype, rank=None, last=None, copy=True):
    """The one operand check: a CUDA tensor of `dtype`, of rank `rank` (None: any) and last dimension `last` (None: any).
    copy=True: an input, returned contiguous (copied if it is not); copy=False: used in place (caller-supplied outputs,
    workspaces, state updated in place), so it must already be contiguous; copy=None: returned as it is, for callers
    that read its strides."""
    if not isinstance(t, torch.Tensor):
        raise ValueError("%s must be a torch.Tensor" % name)
    if not t.is_cuda:
        raise ValueError("%s must be a CUDA tensor (there is no CPU path)" % name)
    if t.dtype != dtype:
        raise ValueError("%s must be %s, got %s" % (name, dtype, t.dtype))
    if rank is not None and t.dim() != rank:
        raise ValueError("%s must have rank %d, got shape %s" % (name, rank, tuple(t.shape)))
    if last is not None and t.shape[-1] != last:
        raise ValueError("%s must have last dimension %d, got shape %s" % (name, last, tuple(t.shape)))
    if copy is None or t.is_contiguous():
        return t
    if not copy:
        raise ValueError("%s is written or kept in place and must be contiguous" % name)
    return t.contiguous()


def _vec(t, name, c):
    """A per-channel float32 vector of length c, read or updated in place."""
    t = _req(t, name, torch.float32, 1, copy=False)
    if t.shape[0] != c:
        raise ValueError("%s must have shape (%d,), got %s" % (name, c, tuple(t.shape)))
    return t


def _scene_strided(t, name):
    """A float32 CUDA tensor (b, n, c) whose rows are dense but whose scenes may be strided (a [:, a:b] slice of a
    dense tensor): returns (tensor, scene stride in floats) without copying; anything else is made contiguous."""
    t = _req(t, name, torch.float32, 3, copy=None)
    b, n, c = t.shape
    if c > 0 and n > 0 and t.stride(2) == 1 and t.stride(1) == c and (b <= 1 or t.stride(0) >= n * c):
        return t, (t.stride(0) if b > 1 else n * c)
    return t.contiguous(), n * c


def _idx_out(out, b, npoint, device):
    """Resolve the optional (buffer, column) output placement of the sampling ops -> (tensor to return, ptr, ldo)."""
    if out is None:
        o = torch.empty((b, npoint), dtype=torch.int32, device=device)
        return o, o.data_ptr(), npoint
    buf, col = out
    buf = _req(buf, "out", torch.int32, 2, copy=False)
    if buf.shape[0] != b or col < 0 or col + npoint > buf.shape[1]:
        raise ValueError("out must be (int32 contiguous (b, >= col + npoint) buffer, col)")
    return buf[:, col:col + npoint], buf.data_ptr() + 4 * col, buf.shape[1]


def _temp(temp, elems):
    """The caller's FPS state buffer: contiguous float32 of at least `elems` elements, used in place."""
    temp = _req(temp, "temp", torch.float32, copy=False)
    if temp.numel() < elems:
        raise ValueError("temp must hold at least %d elements, got %d" % (elems, temp.numel()))
    return temp


def _fps_flags(packet_kernel, bucket_kernel):
    return (1 if packet_kernel else 0) | (0 if bucket_kernel is None else (4 if bucket_kernel else 2))


def fps_temp_elems(n, c=3, npoint=0, packet_kernel=False, bucket_kernel=None):
    """float32 elements per scene of the `temp` buffer farthest_point_sample(..., rounds=...) carries its state in."""
    return int(lib().ssd3d_fps_temp_elems(int(n), int(c), int(npoint), _fps_flags(packet_kernel, bucket_kernel)))


def farthest_point_sample(npoint, inp, *, out=None, idx_offset=0, rounds=None, temp=None, cluster=0, packet_kernel=False,
                          bucket_kernel=None):
    """inp: (batch, ndataset, c) float32 -> (batch, npoint) int32.  tf_sampling.py:43-51; shape check
    tf_sampling.cpp:142 (rank 3).

    Keyword extensions (include/ssd3d.h, ssd3d_farthest_point_sample_ex; none changes the sampled indices):
      out=(buffer, col)   write into columns [col, col+npoint) of an int32 (batch, L) buffer and return that view;
      idx_offset          added to every index (segment offset of a fusion-sampling layer, layers_util.py:109);
      rounds=(j0, j1), temp   run only rounds [j0, j1); `temp` (batch, fps_temp_elems(n, c, npoint)) float32 carries the
                          running state between the calls (j0 == 0 starts fresh); the output must be the same buffer in
                          every call;
      cluster             CTAs per scene: 0 heuristic, >0 exact, <0 heuristic capped at -cluster;
      packet_kernel       use the general cluster kernel even where the resident-scene one applies (tests);
      bucket_kernel       None: automatic (xyz scenes of 8192 < n <= 16384 points take the single-CTA kernel with spatial
                          pruning, csrc/fps_bucket.cu), True / False: force (64 <= n <= 16384) / forbid it."""
    inp, stride = _scene_strided(inp, "inp")
    npoint = int(npoint)
    if npoint < 0:
        raise ValueError("npoint must be non-negative")
    b, n, c = inp.shape
    o, optr, ldo = _idx_out(out, b, npoint, inp.device)
    j0, j1 = (0, npoint) if rounds is None else (int(rounds[0]), int(rounds[1]))
    flags = _fps_flags(packet_kernel, bucket_kernel)
    elems = int(lib().ssd3d_fps_temp_elems(n, c, npoint, flags))
    if temp is None and (lib().ssd3d_fps_needs_temp(n, c) or (j0, j1) != (0, npoint)):
        if (j0, j1) != (0, npoint):
            raise ValueError("a partial range of rounds needs the caller's temp (batch, fps_temp_elems(...)) float32 buffer")
        temp = torch.empty((b, elems), dtype=torch.float32, device=inp.device)
    if temp is not None:
        temp = _temp(temp, b * elems)
    check(lib().ssd3d_farthest_point_sample_ex(b, n, c, npoint, _p(inp), stride, _p(temp), ctypes.c_void_p(optr), ldo,
                                               int(idx_offset), j0, j1, int(cluster), flags, _stream()),
          "farthest_point_sample")
    return o


furthest_point_sample = farthest_point_sample  # spelling used by BASELINE.json's north star


def fps_supports_rounds(n, c=3):
    """True when farthest_point_sample(..., rounds=...) is available for n points of c channels."""
    return bool(lib().ssd3d_fps_supports_rounds(int(n), int(c)))


def farthest_point_sample_with_distance(npoint, dist, *, out=None, idx_offset=0, cluster=0):
    """dist: (batch, n, n) float32 distance matrix -> (batch, npoint) int32.  tf_sampling.py:54-62; the
    square-matrix check is tf_sampling.cpp:175.  Keyword extensions as farthest_point_sample."""
    dist = _req(dist, "dist", torch.float32, 3)
    b, n, n2 = dist.shape
    if n != n2:
        raise ValueError("FarthestPointSampleWithDistance expects (batch_size,num_points,num_points) inp shape")
    npoint = int(npoint)
    o, optr, ldo = _idx_out(out, b, npoint, dist.device)
    temp = torch.empty((b, n), dtype=torch.float32, device=dist.device) if n > 65536 else None
    check(lib().ssd3d_farthest_point_sample_with_distance_ex(b, n, npoint, _p(dist), _p(temp), ctypes.c_void_p(optr), ldo,
                                                             int(idx_offset), int(cluster), _stream()),
          "farthest_point_sample_with_distance")
    return o


def ffps_supported(n, c):
    """True when the matrix-free F-FPS kernel covers n points with c concatenated channels."""
    return bool(lib().ssd3d_ffps_supported(int(n), int(c)))


def farthest_point_sample_features(npoint, xyz, points=None, *, out=None, idx_offset=0, rounds=None, temp=None,
                                   cluster=None):
    """F-FPS on concat[xyz, points] without the distance matrix: the same indices as
    farthest_point_sample_with_distance(npoint, calc_square_dist(concat[xyz, points])) (layers_util.py:94-96).
    Keyword extensions as farthest_point_sample (out, idx_offset, rounds + temp); cluster < 0 caps the CTAs per scene
    at -cluster where a kernel allows it (a full range of 2048 < n <= 4096 points of <= 68 channels then runs on 4 CTAs
    with bucket pruning), cluster=None or 0 leaves the choice to the library."""
    xyz, sa = _scene_strided(xyz, "xyz")
    b, n, ca = xyz.shape
    cb, sb = 0, 0
    if points is not None and points.shape[-1] > 0:
        points, sb = _scene_strided(points, "points")
        if points.shape[:2] != (b, n):
            raise ValueError("points must be (batch, n, c) like xyz")
        cb = points.shape[2]
    else:
        points = None
    npoint = int(npoint)
    o, optr, ldo = _idx_out(out, b, npoint, xyz.device)
    j0, j1 = (0, npoint) if rounds is None else (int(rounds[0]), int(rounds[1]))
    if (j0, j1) != (0, npoint):
        if temp is None:
            raise ValueError("a partial range of rounds needs a contiguous float32 temp buffer of batch * n elements")
        temp = _temp(temp, b * n)
    args = (b, n, ca, cb, npoint, _p(xyz), sa, _p(points), sb, _p(temp), ctypes.c_void_p(optr), ldo, int(idx_offset), j0, j1)
    if cluster is None:
        rc = lib().ssd3d_farthest_point_sample_features_ex(*args, _stream())
    else:
        rc = lib().ssd3d_farthest_point_sample_features_cl(*args, int(cluster), _stream())
    check(rc, "farthest_point_sample_features")
    return o


def _gather_point_fwd(inp, idx):
    b, n, c = inp.shape
    m = idx.shape[1]
    out = torch.empty((b, m, c), dtype=torch.float32, device=inp.device)
    # idx may be a column block of a wider contiguous (b, L) tensor: read in place
    check(lib().ssd3d_gather_point_ex(b, n, m, c, _p(inp), _p(idx), idx.stride(0) if b > 1 else m, _p(out), _stream()),
          "gather_point")
    return out


def gather_point_grad(inp, idx, out_g):
    """Gradient of gather_point w.r.t. inp (tf_sampling.py:38-42 _gather_point_grad): scatter-add of out_g."""
    idx = _req(idx, "idx", torch.int32, 2)
    out_g = _req(out_g, "out_g", torch.float32, 3)
    b, n, c = inp.shape
    inp_g = torch.empty((b, n, c), dtype=torch.float32, device=out_g.device)
    check(lib().ssd3d_gather_point_grad(b, n, idx.shape[1], c, _p(out_g), _p(idx), _p(inp_g), _stream()), "gather_point_grad")
    return inp_g


class _GatherPoint(torch.autograd.Function):
    @staticmethod
    def forward(ctx, inp, idx):
        ctx.save_for_backward(idx)
        ctx.shape = inp.shape
        return _gather_point_fwd(inp, idx)

    @staticmethod
    def backward(ctx, out_g):
        (idx,) = ctx.saved_tensors
        return gather_point_grad(torch.empty(ctx.shape, device="meta"), idx, out_g.contiguous()), None


def gather_point(inp, idx):
    """inp (batch, ndataset, c) float32, idx (batch, npoints) int32 -> (batch, npoints, c).  tf_sampling.py:24-32.
    Differentiable w.r.t. inp (the reference registers GatherPoint's gradient, tf_sampling.py:37-42)."""
    inp = _req(inp, "inp", torch.float32, 3)
    idx = _req(idx, "idx", torch.int32, 2, copy=None)
    if not (idx.stride(1) == 1 and idx.stride(0) >= idx.shape[1]):
        idx = idx.contiguous()
    if idx.shape[0] != inp.shape[0]:
        raise ValueError("GatherPoint expects (batch_size,num_result) idx shape")
    if inp.requires_grad and torch.is_grad_enabled():
        return _GatherPoint.apply(inp, idx)
    return _gather_point_fwd(inp, idx)


def _bq_shapes(xyz1, xyz2):
    xyz1 = _req(xyz1, "xyz1", torch.float32, 3, 3)   # tf_grouping.cpp:283
    xyz2 = _req(xyz2, "xyz2", torch.float32, 3, 3)   # tf_grouping.cpp:288
    if xyz1.shape[0] != xyz2.shape[0]:
        raise ValueError("xyz1 and xyz2 must share the batch dimension")
    return xyz1, xyz2


def _query_ball(op, min_radius, max_radius, nsample, xyz1, xyz2, dilated):
    """The body of query_ball_point (dilated=False, min_radius unused) and query_ball_point_dilated; op names the
    reference op in the error texts."""
    xyz1, xyz2 = _bq_shapes(xyz1, xyz2)
    if not max_radius > 0:
        raise ValueError("%s expects positive radius" % op)      # tf_grouping.cpp:275
    if not int(nsample) > 0:
        raise ValueError("%s expects positive nsample" % op)     # tf_grouping.cpp:278
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    if n >= BQ_GRID_MIN_N and lib().ssd3d_query_ball_point_workspace(b, n):
        i, c = query_ball_point_multi([min_radius], [max_radius], [nsample], xyz1, xyz2, dilated)
        return i[0], c[0]
    idx = torch.empty((b, m, int(nsample)), dtype=torch.int32, device=xyz1.device)
    cnt = torch.empty((b, m), dtype=torch.int32, device=xyz1.device)
    tail = (int(nsample), _p(xyz1), _p(xyz2), _p(idx), _p(cnt), _stream())
    if dilated:
        check(lib().ssd3d_query_ball_point_dilated(b, n, m, float(min_radius), float(max_radius), *tail), "query_ball_point_dilated")
    else:
        check(lib().ssd3d_query_ball_point(b, n, m, float(max_radius), *tail), "query_ball_point")
    return idx, cnt


def query_ball_point(radius, nsample, xyz1, xyz2):
    """xyz1 (batch, ndataset, 3), xyz2 (batch, npoint, 3) -> idx (batch, npoint, nsample) int32,
    pts_cnt (batch, npoint) int32.  tf_grouping.py:53-65."""
    return _query_ball("QueryBallPoint", 0.0, radius, nsample, xyz1, xyz2, False)


def query_ball_point_dilated(min_radius, max_radius, nsample, xyz1, xyz2):
    """Shell query  d == 0 or min_radius <= d < max_radius.  tf_grouping.py:68-81."""
    return _query_ball("QueryBallPointDilated", min_radius, max_radius, nsample, xyz1, xyz2, True)


BQ_GRID_MIN_N = 2048     # candidate sets at least this large take the spatially culled kernel (csrc/ball_query_grid.cu)


def query_ball_point_multi(min_radius_list, max_radius_list, nsample_list, xyz1, xyz2, dilated, grid=None, return_units=False):
    """All radius shells of one SA layer in a single pass over the candidates (fast path; same results
    as calling query_ball_point[_dilated] once per shell).  Returns lists (idx_list, pts_cnt_list).
    grid: None = automatic (the culled kernel for ndataset >= BQ_GRID_MIN_N), True / False = force / forbid it;
    the outputs are identical either way.
    return_units: also return, per shell, the UNIT LIST of the grouped MLP (int32 tensor, include/ssd3d.h
    ssd3d_query_ball_point_multi_ws), or None for nsample > 128: (idx_list, pts_cnt_list, units_list)."""
    xyz1, xyz2 = _bq_shapes(xyz1, xyz2)
    nq = len(max_radius_list)
    if not (len(nsample_list) == nq and len(min_radius_list) == nq and 1 <= nq <= 4):
        raise ValueError("query_ball_point_multi takes 1..4 shells with matching list lengths")
    for r, k in zip(max_radius_list, nsample_list):
        if not r > 0:
            raise ValueError("QueryBallPoint expects positive radius")
        if not int(k) > 0:
            raise ValueError("QueryBallPoint expects positive nsample")
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    idx = [torch.empty((b, m, int(k)), dtype=torch.int32, device=xyz1.device) for k in nsample_list]
    cnt = [torch.empty((b, m), dtype=torch.int32, device=xyz1.device) for _ in nsample_list]
    lo = (ctypes.c_float * nq)(*[float(v) for v in min_radius_list])
    hi = (ctypes.c_float * nq)(*[float(v) for v in max_radius_list])
    ks = (ctypes.c_int * nq)(*[int(v) for v in nsample_list])
    pi = (ctypes.c_void_p * nq)(*[t.data_ptr() for t in idx])
    pc = (ctypes.c_void_p * nq)(*[t.data_ptr() for t in cnt])
    ws_bytes = int(lib().ssd3d_query_ball_point_workspace(b, n)) if (b and m) else 0
    use_grid = ws_bytes > 0 and (n >= BQ_GRID_MIN_N if grid is None else bool(grid))
    if grid and not use_grid and b and m:
        raise ValueError("the culled ball query covers ndataset <= 16384, got %d" % n)
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=xyz1.device) if use_grid else None
    units = [None] * nq
    pu = ctypes.c_void_p(0)
    if return_units and all(int(k) <= 128 for k in nsample_list):
        units = [torch.empty((1 + b * m * ((int(k) + 7) // 8),), dtype=torch.int32, device=xyz1.device) for k in nsample_list]
        parr = (ctypes.c_void_p * nq)(*[t.data_ptr() for t in units])
        pu = ctypes.cast(parr, ctypes.c_void_p)
    check(lib().ssd3d_query_ball_point_multi_ws(b, n, m, nq, 1 if dilated else 0, ctypes.cast(lo, ctypes.c_void_p),
                                                ctypes.cast(hi, ctypes.c_void_p), ctypes.cast(ks, ctypes.c_void_p),
                                                _p(xyz1), _p(xyz2), ctypes.cast(pi, ctypes.c_void_p),
                                                ctypes.cast(pc, ctypes.c_void_p), pu, _p(ws), ws_bytes if use_grid else 0,
                                                _stream()), "query_ball_point_multi")
    if return_units:
        return idx, cnt, units
    return idx, cnt


def _group_point_fwd(points, idx):
    b, n, c = points.shape
    _, m, ns = idx.shape
    out = torch.empty((b, m, ns, c), dtype=torch.float32, device=points.device)
    check(lib().ssd3d_group_point(b, n, c, m, ns, _p(points), _p(idx), _p(out), _stream()), "group_point")
    return out


def group_point_grad(points, idx, grad_out):
    """Gradient of group_point w.r.t. points (tf_grouping.py:123-128 _group_point_grad)."""
    idx = _req(idx, "idx", torch.int32, 3)
    grad_out = _req(grad_out, "grad_out", torch.float32, 4)
    b, n, c = points.shape
    _, m, ns = idx.shape
    g = torch.empty((b, n, c), dtype=torch.float32, device=grad_out.device)
    check(lib().ssd3d_group_point_grad(b, n, c, m, ns, _p(grad_out), _p(idx), _p(g), _stream()), "group_point_grad")
    return g


class _GroupPoint(torch.autograd.Function):
    @staticmethod
    def forward(ctx, points, idx):
        ctx.save_for_backward(idx)
        ctx.shape = points.shape
        return _group_point_fwd(points, idx)

    @staticmethod
    def backward(ctx, grad_out):
        (idx,) = ctx.saved_tensors
        return group_point_grad(torch.empty(ctx.shape, device="meta"), idx, grad_out.contiguous()), None


def group_point(points, idx):
    """points (batch, ndataset, channel) float32, idx (batch, npoint, nsample) int32 ->
    (batch, npoint, nsample, channel); idx == -1 gives zeros.  tf_grouping.py:114-122; differentiable w.r.t. points."""
    points = _req(points, "points", torch.float32, 3)
    idx = _req(idx, "idx", torch.int32, 3)
    if idx.shape[0] != points.shape[0]:
        raise ValueError("GroupPoint expects (batch_size, npoints, nsample) idx shape")
    if points.requires_grad and torch.is_grad_enabled():
        return _GroupPoint.apply(points, idx)
    return _group_point_fwd(points, idx)


def three_nn(xyz1, xyz2):
    """xyz1 (b,n,3) unknown, xyz2 (b,m,3) known -> dist (b,n,3) float32 (squared), idx (b,n,3) int32.
    tf_interpolate.py:8-19."""
    xyz1 = _req(xyz1, "xyz1", torch.float32, 3, 3)   # tf_interpolate.cpp:222
    xyz2 = _req(xyz2, "xyz2", torch.float32, 3, 3)   # tf_interpolate.cpp:227
    if xyz1.shape[0] != xyz2.shape[0]:
        raise ValueError("xyz1 and xyz2 must share the batch dimension")
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    dist = torch.empty((b, n, 3), dtype=torch.float32, device=xyz1.device)
    idx = torch.empty((b, n, 3), dtype=torch.int32, device=xyz1.device)
    check(lib().ssd3d_three_nn(b, n, m, _p(xyz1), _p(xyz2), _p(dist), _p(idx), _stream()), "three_nn")
    return dist, idx


def three_interpolate(points, idx, weight):
    """points (b,m,c), idx (b,n,3) int32, weight (b,n,3) -> (b,n,c).  tf_interpolate.py:21-31."""
    points = _req(points, "points", torch.float32, 3)
    idx = _req(idx, "idx", torch.int32, 3, 3)
    weight = _req(weight, "weight", torch.float32, 3, 3)
    b, m, c = points.shape
    n = idx.shape[1]
    if idx.shape[0] != b or weight.shape != idx.shape:
        raise ValueError("ThreeInterpolate expects (b,n,3) idx and weight shapes")
    if points.requires_grad and torch.is_grad_enabled():
        return _ThreeInterpolate.apply(points, idx, weight)
    return _three_interpolate_fwd(points, idx, weight)


def _three_interpolate_fwd(points, idx, weight):
    b, m, c = points.shape
    n = idx.shape[1]
    out = torch.empty((b, n, c), dtype=torch.float32, device=points.device)
    check(lib().ssd3d_three_interpolate(b, m, c, n, _p(points), _p(idx), _p(weight), _p(out), _stream()),
          "three_interpolate")
    return out


def three_interpolate_grad(points, idx, weight, grad_out):
    """Gradient of three_interpolate w.r.t. points (tf_interpolate.py:32-37 _three_interpolate_grad)."""
    grad_out = _req(grad_out, "grad_out", torch.float32, 3)
    b, m, c = points.shape
    n = idx.shape[1]
    g = torch.empty((b, m, c), dtype=torch.float32, device=grad_out.device)
    check(lib().ssd3d_three_interpolate_grad(b, n, c, m, _p(grad_out), _p(idx), _p(weight), _p(g), _stream()),
          "three_interpolate_grad")
    return g


class _ThreeInterpolate(torch.autograd.Function):
    @staticmethod
    def forward(ctx, points, idx, weight):
        ctx.save_for_backward(idx, weight)
        ctx.shape = points.shape
        return _three_interpolate_fwd(points, idx, weight)

    @staticmethod
    def backward(ctx, grad_out):
        idx, weight = ctx.saved_tensors
        return three_interpolate_grad(torch.empty(ctx.shape, device="meta"), idx, weight, grad_out.contiguous()), None, None


# ---- dense pieces that are stock TF ops in the reference -------------------------------------------------

def calc_square_dist(a):
    """model_util.calc_square_dist(a, a, norm=False) (/root/reference/lib/utils/model_util.py:144-160)."""
    a = _req(a, "a", torch.float32, 3)
    b, n, c = a.shape
    out = torch.empty((b, n, n), dtype=torch.float32, device=a.device)
    check(lib().ssd3d_calc_square_dist(b, n, c, _p(a), _p(out), _stream()), "calc_square_dist")
    return out


def _grouping(xyz, points, new_xyz, idx, cnt=None):
    """The operands of a grouping kernel: xyz (b, n, 3), points (b, n, c) or None, new_xyz (b, m, 3), idx (b, m, nsample)
    int32 and, when given, cnt (b, m) int32 -> (xyz, points, new_xyz, idx, b, n, c, m, nsample)."""
    xyz = _req(xyz, "xyz", torch.float32, 3, 3)
    new_xyz = _req(new_xyz, "new_xyz", torch.float32, 3, 3)
    idx = _req(idx, "idx", torch.int32, 3)
    b, n, _ = xyz.shape
    _, m, ns = idx.shape
    if tuple(new_xyz.shape) != (b, m, 3) or idx.shape[0] != b:
        raise ValueError("new_xyz %s and idx %s must be (b, m, 3) and (b, m, nsample) with xyz %s"
                         % (tuple(new_xyz.shape), tuple(idx.shape), tuple(xyz.shape)))
    c = 0
    if points is not None:
        points = _req(points, "points", torch.float32, 3)
        c = points.shape[2]
        if points.shape[:2] != (b, n):
            raise ValueError("points %s must be (b, n, c) like xyz %s" % (tuple(points.shape), tuple(xyz.shape)))
    if cnt is not None and tuple(_req(cnt, "cnt", torch.int32, 2, copy=False).shape) != (b, m):
        raise ValueError("cnt must be (%d, %d), got %s" % (b, m, tuple(cnt.shape)))
    return xyz, points, new_xyz, idx, b, n, c, m, ns


def _hoisted_table(z, zoff, wx, b, n):
    """The per-point table of a hoisted first conv: z (b, n, ldz) fp32 whose columns [zoff, zoff + n1) belong to this
    scale, wx (3, n1) fp32 -> (pointer to column zoff, ldz, wx, n1)."""
    z = _req(z, "z", torch.float32, 3)
    wx = _req(wx, "wx", torch.float32, 2)
    n1 = wx.shape[1]
    if z.shape[:2] != (b, n) or wx.shape[0] != 3 or zoff < 0 or zoff + n1 > z.shape[2]:
        raise ValueError("z must be (b, n, ldz) with zoff + n1 <= ldz and wx (3, n1)")
    return ctypes.c_void_p(z.data_ptr() + 4 * zoff), z.shape[2], wx, n1


def _placed(out, name, dtype, lead, n):
    """A caller's output slot for n columns, (buffer, col) or (hi, lo, col): contiguous `dtype` buffers (*lead, ld) with
    0 <= col and col + n <= ld -> ([buffers], [pointers to their column col], ld)."""
    buf, col = out[:-1], int(out[-1])
    bufs = [_req(t, name, dtype, copy=False) for t in buf]
    ld = bufs[0].shape[-1]
    if any(tuple(t.shape) != tuple(lead) + (ld,) for t in bufs) or col < 0 or col + n > ld:
        raise ValueError("%s must be (%s buffer (%s, ld), col) with 0 <= col and col + %d <= ld, got shape %s and col %d"
                         % (name, dtype, ", ".join(map(str, lead)), n, tuple(bufs[0].shape), col))
    return bufs, [ctypes.c_void_p(t.data_ptr() + t.element_size() * col) for t in bufs], ld


def _outputs(lead, n, dev, want_f32, want_split, out_f32, out_split, pooled):
    """The fp32 and split-bf16 outputs of the tensor-core and fused kernels: the caller's (buffer, col) /
    (hi, lo, col) slots, else fresh tensors (*lead, n) / (*lead, round16(n)) when wanted.  A pooled split output is
    zero-filled so that its padding columns are 0.  -> (y, (hi, lo) or None, [pf, ldf, phi, plo, lds])."""
    y, sp = None, None
    pf, ldf = ctypes.c_void_p(0), 0
    if out_f32 is not None:
        (y,), (pf,), ldf = _placed(out_f32, "out_f32", torch.float32, lead, n)
    elif want_f32:
        y = torch.empty(lead + (n,), dtype=torch.float32, device=dev)
        pf, ldf = _p(y), n
    ph = pl = ctypes.c_void_p(0)
    lds = 0
    if out_split is not None:
        sp, (ph, pl), lds = _placed(out_split, "out_split", torch.bfloat16, lead, n)
        sp = tuple(sp)
    elif want_split:
        lds = round16(n)
        alloc = torch.zeros if (pooled and lds != n) else torch.empty
        sp = tuple(alloc(lead + (lds,), dtype=torch.bfloat16, device=dev) for _ in range(2))
        ph, pl = _p(sp[0]), _p(sp[1])
    return y, sp, [pf, ldf, ph, pl, lds]


def _units_check(units, unit_pool, pool=1, rowmask=None, relu=True, out_f32=None, out_split=None, want_split=False):
    """A unit list (query_ball_point_multi(return_units=True)) replaces pool / rowmask; with unit_pool the listed 8-row
    units are max-pooled into the caller's zero-filled out_f32 by atomicMax, so there is no split output."""
    if units is None:
        if unit_pool:
            raise ValueError("unit_pool needs a unit list")
        return
    _req(units, "units", torch.int32, copy=False)
    if int(pool) != 1 or rowmask is not None:
        raise ValueError("a unit list replaces pool / rowmask (unit_pool=True pools the listed 8-row units)")
    if unit_pool and (not relu or out_f32 is None or out_split is not None or want_split):
        raise ValueError("a pooled unit list needs relu, out_f32=(zero-filled buffer, col_offset) and no split output")


def _pool(pool, group):
    """The max-pool width of a tensor-core kernel: 1, or the group size `group` when that is one of TC_POOL_WIDTHS."""
    pool = int(pool)
    if pool > 1 and (pool != group or pool not in TC_POOL_WIDTHS):
        raise ValueError("pool must equal nsample (the second-to-last dimension) and be one of %s" % (TC_POOL_WIDTHS,))
    return pool


def _rowmask(rowmask, groups):
    """A pooled output's mask: int32 with one entry per pooled group, or None."""
    if rowmask is None:
        return None
    rowmask = _req(rowmask, "rowmask", torch.int32)
    if rowmask.numel() != groups:
        raise ValueError("rowmask must hold one entry per group (%d), got shape %s" % (groups, tuple(rowmask.shape)))
    return rowmask


def group_concat(xyz, points, new_xyz, idx, ldx=None):
    """concat[group_point(points, idx), group_point(xyz, idx) - new_xyz] (layers_util.py:160-165) in one kernel.
    Returns x (b, m, nsample, ldx) with zero padding beyond c+3."""
    xyz, points, new_xyz, idx, b, n, c, m, ns = _grouping(xyz, points, new_xyz, idx)
    ldx = c + 3 if ldx is None else int(ldx)
    x = torch.empty((b, m, ns, ldx), dtype=torch.float32, device=xyz.device)
    check(lib().ssd3d_group_concat(b, n, c, m, ns, _p(xyz), _p(points), _p(new_xyz), _p(idx), _p(x), ldx, _stream()),
          "group_concat")
    return x


def linear_bn_relu(x, w, scale, shift, relu=True, pool=1, rowmask=None, cin=None):
    """act((x[..., :cin] @ w) * scale + shift) over the last axis; pool > 1 max-pools runs of `pool` rows and
    multiplies by rowmask != 0 (layers_util.py:178-180).  x (..., ldx), w (cin, cout)."""
    x = _req(x, "x", torch.float32)
    w = _req(w, "w", torch.float32, 2)
    wcin, cout = w.shape
    cin = wcin if cin is None else cin
    ldx = x.shape[-1]
    if cin != wcin or ldx < cin:
        raise ValueError("linear_bn_relu: x last dim %d / cin %d do not match w %s" % (ldx, cin, tuple(w.shape)))
    rows = x.numel() // ldx
    pool = int(pool)
    lead = tuple(x.shape[:-1])
    if pool > 1 and lead[-1] != pool:
        raise ValueError("pool must equal the second-to-last dimension of x")
    olead = lead[:-1] if pool > 1 else lead
    rowmask = _rowmask(rowmask, math.prod(olead))
    y = torch.empty(olead + (cout,), dtype=torch.float32, device=x.device)
    if pool > 1 and 128 % pool != 0:
        r = linear_bn_relu(x, w, scale, shift, relu, 1, None, cin)
        check(lib().ssd3d_rowgroup_max(rows // pool, pool, cout, _p(r), cout, _p(rowmask), _p(y), _stream()), "rowgroup_max")
        return y
    check(lib().ssd3d_linear_bn_relu(rows, cin, cout, _p(x), ldx, _p(w), _p(scale), _p(shift), 1 if relu else 0, pool,
                                     _p(rowmask), _p(y), cout, _stream()), "linear_bn_relu")
    return y


# ---- tensor-core (wgmma) path of the MLP: operands split in two bf16 terms ---------------------------------

TC_POOL_WIDTHS = (8, 16, 32, 64, 128)   # group sizes the max-pool epilogue of the tensor-core kernels covers


def split_rows(x, kp=None):
    """fp32 (..., c) -> (hi, lo) bf16 (..., kp) with hi + lo ~= x (16 mantissa bits), zero padded to kp."""
    x = _req(x, "x", torch.float32)
    c = x.shape[-1]
    kp = round16(c) if kp is None else int(kp)
    rows = x.numel() // c
    hi = torch.empty(tuple(x.shape[:-1]) + (kp,), dtype=torch.bfloat16, device=x.device)
    lo = torch.empty_like(hi)
    check(lib().ssd3d_split_rows(rows, c, _p(x), c, _p(hi), _p(lo), kp, _stream()), "split_rows")
    return hi, lo


def group_concat_split(xyz, points, new_xyz, idx, kp=None):
    """group_concat + split in one kernel: (hi, lo) bf16 (b, m, nsample, kp)."""
    xyz, points, new_xyz, idx, b, n, c, m, ns = _grouping(xyz, points, new_xyz, idx)
    kp = round16(c + 3) if kp is None else int(kp)
    hi = torch.empty((b, m, ns, kp), dtype=torch.bfloat16, device=xyz.device)
    lo = torch.empty_like(hi)
    check(lib().ssd3d_group_concat_split(b, n, c, m, ns, _p(xyz), _p(points), _p(new_xyz), _p(idx), _p(hi), _p(lo), kp,
                                         _stream()), "group_concat_split")
    return hi, lo


def _tc_epilogue(f, relu, pool, rowmask, lead, ns, dev, want_f32, want_split, out_f32, out_split, units, unit_pool):
    """Checks and output placement shared by the linear_tc* wrappers, for an operand of leading shape `lead` in groups
    of ns rows -> (y, (hi, lo) or None, pool, rowmask, the layer's arguments, the output arguments)."""
    _units_check(units, unit_pool, pool, rowmask, relu, out_f32, out_split, want_split)
    pool = _pool(pool, ns)
    pooled = pool > 1 or unit_pool
    olead = lead[:-1] if pooled else lead
    rowmask = _rowmask(rowmask, math.prod(olead))
    y, sp, out = _outputs(olead, f.cout, dev, want_f32, want_split, out_f32, out_split, pooled)
    return y, sp, pool, rowmask, [_p(f.b_hi), _p(f.b_lo), _p(f.scale), _p(f.shift), 1 if relu else 0], out


def linear_tc(a_hi, a_lo, f, relu=True, pool=1, rowmask=None, want_f32=True, want_split=False, out_f32=None,
              out_split=None, units=None, unit_pool=False):
    """One folded conv layer on the tensor cores.  a_hi/a_lo (..., kp) bf16; f: params.FoldedConv.
    Returns (y_f32 or None, (hi, lo) or None).  out_f32=(buffer, col_offset) / out_split=(hi_buf, lo_buf, col_offset)
    write into slices of preallocated (..., ld) buffers (the concat of the SA scales) instead of allocating.
    units: the operand holds COMPACT rows (8 per listed unit, include/ssd3d.h ssd3d_linear_tc_units) in its first
    units[0] * 8 rows; outputs are compact likewise, or -- unit_pool=True, the last conv of a scale -- every unit is
    max-pooled and combined into out_f32[group] by atomicMax (buffer zero-filled by the caller)."""
    a_hi, a_lo = _req(a_hi, "a_hi", torch.bfloat16), _req(a_lo, "a_lo", torch.bfloat16)
    if a_hi.shape != a_lo.shape:
        raise ValueError("a_hi / a_lo must be bfloat16 tensors of the same shape")
    kp = a_hi.shape[-1]
    if kp != f.kp:
        raise ValueError("operand K (%d) does not match the layer's padded K (%d)" % (kp, f.kp))
    lead = tuple(a_hi.shape[:-1])
    y, sp, pool, rowmask, head, out = _tc_epilogue(f, relu, pool, rowmask, lead, lead[-1] if lead else 1, a_hi.device,
                                                   want_f32, want_split, out_f32, out_split, units, unit_pool)
    args = [a_hi.numel() // kp, kp, f.cout, _p(a_hi), _p(a_lo)] + head
    if units is not None:
        check(lib().ssd3d_linear_tc_units(*args, _p(units), 1 if unit_pool else 0, *out, _stream()), "linear_tc_units")
    else:
        check(lib().ssd3d_linear_tc(*args, pool, _p(rowmask), *out, _stream()), "linear_tc")
    return y, sp


def linear_tc_gather(xyz, points, new_xyz, idx, f, relu=True, pool=1, rowmask=None, want_f32=False, want_split=True,
                     out_f32=None, out_split=None):
    """First conv layer of an SA scale with the gather / centre-subtract / concat of layers_util.py:160-165 fused
    into the tensor-core kernel's operand load (no [B,M,K,C] tensor in HBM).  Outputs as linear_tc, leading shape
    (b, m, nsample) or (b, m) when pooled."""
    xyz, points, new_xyz, idx, b, n, c, m, ns = _grouping(xyz, points, new_xyz, idx)
    if round16(c + 3) != f.kp or c + 3 != f.cin:
        raise ValueError("layer input width %d does not match c+3 = %d" % (f.cin, c + 3))
    y, sp, pool, rowmask, head, out = _tc_epilogue(f, relu, pool, rowmask, (b, m, ns), ns, xyz.device, want_f32,
                                                   want_split, out_f32, out_split, None, False)
    check(lib().ssd3d_linear_tc_gather(b, n, c, m, ns, _p(xyz), _p(points), _p(new_xyz), _p(idx), f.cout, *head, pool,
                                       _p(rowmask), *out, _stream()), "linear_tc_gather")
    return y, sp


def linear_tc_hoisted(xyz, z, zoff, wx, new_xyz, idx, f, relu=True, pool=1, rowmask=None, want_f32=False, want_split=True,
                      out_f32=None, out_split=None, units=None, unit_pool=False):
    """Second conv of an SA scale fed by the hoisted first conv (include/ssd3d.h, ssd3d_linear_tc_hoisted).
    z: (b, n, ldz) fp32 per-point table = (features . Wf) * s1 + t1 for all scales of the layer, this scale's
    columns start at zoff; wx: (3, n1) fp32 = Wx * s1; f: params.FoldedConv of the second conv (cin == n1).
    units / unit_pool: as linear_tc (the source rows are looked up through the list, outputs are compact)."""
    xyz, _, new_xyz, idx, b, n, _, m, ns = _grouping(xyz, None, new_xyz, idx)
    zp, ldz, wx, n1 = _hoisted_table(z, zoff, wx, b, n)
    if f.cin != n1:
        raise ValueError("second conv expects %d inputs, the hoisted first conv has %d outputs" % (f.cin, n1))
    y, sp, pool, rowmask, head, out = _tc_epilogue(f, relu, pool, rowmask, (b, m, ns), ns, xyz.device, want_f32,
                                                   want_split, out_f32, out_split, units, unit_pool)
    args = [b, n, n1, m, ns, _p(xyz), zp, ldz, _p(wx), _p(new_xyz), _p(idx)]
    if units is not None:
        check(lib().ssd3d_linear_tc_hoisted_units(*args, _p(units), f.cout, *head, 1 if unit_pool else 0, *out, _stream()),
              "linear_tc_hoisted_units")
    else:
        check(lib().ssd3d_linear_tc_hoisted(*args, f.cout, *head, pool, _p(rowmask), *out, _stream()), "linear_tc_hoisted")
    return y, sp


def hoist_expand_split(xyz, z, zoff, wx, new_xyz, idx, units=None):
    """The operand linear_tc_hoisted would build in its producer warps, materialised: (hi, lo) bf16 (b, m, nsample, kp) =
    split(relu(z[idx] + (xyz[idx] - new_xyz) . wx)).  Followed by the plain linear_tc this is the faster route for wide
    layers (K >= 256), where the resident operand of the in-kernel route leaves the weight ring two narrow stages.
    units: only the listed 8-row units are built, as compact rows at the start of the buffers."""
    xyz, _, new_xyz, idx, b, n, _, m, ns = _grouping(xyz, None, new_xyz, idx)
    zp, ldz, wx, n1 = _hoisted_table(z, zoff, wx, b, n)
    if zoff % 4 or ldz % 4:                         # the kernel reads the table in 16-byte vectors
        raise ValueError("z must be (b, n, ldz) with ldz, zoff multiples of 4, zoff + n1 <= ldz, and wx (3, n1)")
    _units_check(units, False)
    kp = round16(n1)
    hi = torch.empty((b, m, ns, kp), dtype=torch.bfloat16, device=xyz.device)
    lo = torch.empty_like(hi)
    args = [b, n, n1, m, ns, _p(xyz), zp, ldz, _p(wx), _p(new_xyz), _p(idx)]
    if units is not None:
        check(lib().ssd3d_hoist_expand_split_units(*args, _p(units), _p(hi), _p(lo), kp, _stream()), "hoist_expand_split_units")
    else:
        check(lib().ssd3d_hoist_expand_split(*args, _p(hi), _p(lo), kp, _stream()), "hoist_expand_split")
    return hi, lo


def _sa_fused(xyz, points, table, new_xyz, idx, cnt, stack, out_f32, out_split, units):
    """The body of sa_mlp_fused (points, table None) and sa_mlp_fused_hoisted (table = (z, zoff, wx)) up to the entry
    point -> (y, the entry point's arguments without the stream)."""
    _units_check(units, units is not None, out_f32=out_f32, out_split=out_split)
    xyz, points, new_xyz, idx, b, n, c, m, ns = _grouping(xyz, points, new_xyz, idx, cnt)
    if table is None:
        if c + 3 != stack.cin:
            raise ValueError("feature channels (%d) do not match the stack's input width (%d)" % (c, stack.cin - 3))
        src = [c, m, ns, _p(xyz), _p(points)]
    else:
        zp, ldz, wx, n1 = _hoisted_table(*table, b, n)
        if n1 != stack.cin:
            raise ValueError("hoisted width (%d) does not match the stack's input width (%d)" % (n1, stack.cin))
        src = [n1, m, ns, _p(xyz), zp, ldz, _p(wx)]
    y, _, out = _outputs((b, m), stack.nout[-1], xyz.device, out_split is None, False, out_f32, out_split, True)
    nout = (ctypes.c_int * len(stack.nout))(*stack.nout)
    return y, [b, n] + src + [_p(new_xyz), _p(idx), _p(cnt), _p(units), len(stack.nout), ctypes.cast(nout, ctypes.c_void_p),
                              _p(stack.w_blob), _p(stack.ss_blob), 1 if stack.last_scale_nonneg else 0] + out


def sa_mlp_fused(xyz, points, new_xyz, idx, cnt, stack, out_f32=None, out_split=None, units=None):
    """One SA scale in one kernel: gather + concat + conv stack + max-pool + mask (layers_util.py:157-180).
    stack: params.FusedStack.  out_f32=(buffer, col_offset) / out_split=(hi, lo, col_offset) as linear_tc;
    without them a fresh (b, m, C3) fp32 tensor is returned.
    units: the scale's unit list (query_ball_point_multi(return_units=True)): only the listed 8-row units are convolved
    -- the skipped rows repeat a group's first neighbour and cannot change the max-pool -- and results are combined with
    atomicMax into out_f32, which must be zero-filled (fill_zero)."""
    y, args = _sa_fused(xyz, points, None, new_xyz, idx, cnt, stack, out_f32, out_split, units)
    check(lib().ssd3d_sa_mlp_fused(*args, _stream()), "sa_mlp_fused")
    return y


def sa_mlp_fused_hoisted(xyz, z, zoff, wx, new_xyz, idx, cnt, stack, out_f32=None, out_split=None, units=None):
    """sa_mlp_fused with the scale's first conv hoisted into the per-point table z (see linear_tc_hoisted): `stack` is the
    params.FusedStack of the REMAINING convs (its input width == wx.shape[1]).  units: as sa_mlp_fused."""
    y, args = _sa_fused(xyz, None, (z, zoff, wx), new_xyz, idx, cnt, stack, out_f32, out_split, units)
    check(lib().ssd3d_sa_mlp_fused_hoisted(*args, _stream()), "sa_mlp_fused_hoisted")
    return y


def bev_nms(boxes, scores, iou_threshold, max_output, cls_id=0, out=None):
    """Greedy BEV NMS per scene (postprocessor.py:76-88): boxes (b,n,7) = (x,y,z,l,h,w,ry), scores (b,n) ->
    block (b,max_output,9) = (box7, score, class) zero padded, count (b,) int32.  out=(block, count) writes into
    preallocated contiguous tensors (the send buffer of the multi-GPU gather).  Descending score, ties (-0 and +0
    included) to the lower index; rectangles and IoU by the float32 recipe of DESIGN.md §3.5, which the CPU
    restatements of the test suite share decision for decision.  NaN scores are outside the contract."""
    boxes = _req(boxes, "boxes", torch.float32, 3, 7)
    scores = _req(scores, "scores", torch.float32, 2)
    b, n, _ = boxes.shape
    if scores.shape != (b, n):
        raise ValueError("scores must be (b, n)")
    if out is None:
        block = torch.empty((b, int(max_output), 9), dtype=torch.float32, device=boxes.device)
        cnt = torch.empty((b,), dtype=torch.int32, device=boxes.device)
    else:
        block, cnt = _req(out[0], "out block", torch.float32, 3, 9, copy=False), _req(out[1], "out count", torch.int32, 1, copy=False)
        if tuple(block.shape) != (b, int(max_output), 9) or tuple(cnt.shape) != (b,):
            raise ValueError("out must be (float32 (b, max_output, 9), int32 (b,)) contiguous tensors")
    check(lib().ssd3d_bev_nms(b, n, _p(boxes), _p(scores), float(iou_threshold), int(max_output), int(cls_id),
                              _p(block), _p(cnt), _stream()), "bev_nms")
    return block, cnt


# ---- KITTI evaluation (csrc/box_eval.cu, DESIGN.md section 3.10; evaluation/tf_evaluate.py) --------------------------

EVAL_MAX_DETS = 1024          # detections per frame
EVAL_MAX_LABELS = 256         # label rows per frame
EVAL_NSAMPLE = 41


def calc_iou(detections, groundtruths):
    """tf_evaluate.py:26-33: detections (bs, n, 7), groundtruths (bs, m, 7) as (x, y, z, l, h, w, ry) ->
    (iou_bev, iou_3d), each (bs, n, m) float32: rotated BEV and 3-D IoU computed in double."""
    d = _req(detections, "detections", torch.float32, 3, 7)
    g = _req(groundtruths, "groundtruths", torch.float32, 3, 7)
    if g.shape[0] != d.shape[0]:
        raise ValueError("groundtruths must be (bs, -1, 7) with bs = %d, got %s" % (d.shape[0], tuple(g.shape)))
    b, n, m = d.shape[0], d.shape[1], g.shape[1]
    bev = torch.empty((b, n, m), dtype=torch.float32, device=d.device)
    v3 = torch.empty((b, n, m), dtype=torch.float32, device=d.device)
    check(lib().ssd3d_box_iou(b, n, m, _p(d), _p(g), _p(bev), _p(v3), _stream()), "calc_iou")
    return bev, v3


def calc_iou_match(detections, groundtruths):
    """tf_evaluate.py:35-42: row i of detections (-1, 7) against row i of groundtruths (-1, 7) -> (iou_bev, iou_3d),
    each (-1,) float32."""
    d = _req(detections, "detections", torch.float32, 2, 7)
    g = _req(groundtruths, "groundtruths", torch.float32, 2, 7)
    if g.shape[0] != d.shape[0]:
        raise ValueError("groundtruths must be (%d, 7), got %s" % (d.shape[0], tuple(g.shape)))
    n = d.shape[0]
    bev = torch.empty((n,), dtype=torch.float32, device=d.device)
    v3 = torch.empty((n,), dtype=torch.float32, device=d.device)
    check(lib().ssd3d_box_iou_matched(n, _p(d), _p(g), _p(bev), _p(v3), _stream()), "calc_iou_match")
    return bev, v3


def evaluate(detections, names, numlist):
    """tf_evaluate.py:9-23: detections (n, 14) float32 rows as evaluate_map builds them, names (m,) KITTI label_2 file
    paths, numlist (m,) int32 detections per frame -> (precision_image, aos_image, precision_ground, aos_ground,
    precision_3d, aos_3d), each (3, 3, 41) float32 = [Car / Pedestrian / Cyclist, easy / moderate / hard, sample].
    A class is evaluated in a metric only when one of its detections has the fields the metric needs; its other entries,
    and every AOS entry (the reference never computes AOS), are -1."""
    from .evaluation import read_label_file
    names = [n.decode() if isinstance(n, bytes) else str(n) for n in names]
    nl = _req(numlist, "numlist", torch.int32, 1)
    if nl.shape[0] != len(names):
        raise ValueError("numlist must be (%d,) like names, got %s" % (len(names), tuple(nl.shape)))
    return evaluate_labels(detections, [read_label_file(n) for n in names], nl)


def _eval_frames(detections, labels, numlist):
    """Operand checks and CSR offsets of evaluate_labels, all before anything reaches the library."""
    import numpy as np
    det = _req(detections, "detections", torch.float32, 2, 14)
    nl = _req(numlist, "numlist", torch.int32, 1)
    labels = [np.asarray(x, np.float64) for x in labels]
    if any(x.ndim != 2 or x.shape[1] != 15 for x in labels):
        raise ValueError("labels must be one (rows, 15) float64 array per frame (evaluation.read_label_file)")
    if nl.shape[0] != len(labels):
        raise ValueError("numlist must be (%d,) like labels, got %s" % (len(labels), tuple(nl.shape)))
    counts = nl.cpu().numpy().astype(np.int64)
    lc = np.array([x.shape[0] for x in labels], np.int64)
    if (counts < 0).any() or counts.sum() != det.shape[0]:
        raise ValueError("numlist must be non-negative and sum to the %d detection rows" % det.shape[0])
    if len(counts) and counts.max() > EVAL_MAX_DETS:
        raise ValueError("evaluate: at most %d detections per frame (frame %d has %d)" %
                         (EVAL_MAX_DETS, int(counts.argmax()), int(counts.max())))
    if len(lc) and lc.max() > EVAL_MAX_LABELS:
        raise ValueError("evaluate: at most %d label rows per frame (frame %d has %d)" %
                         (EVAL_MAX_LABELS, int(lc.argmax()), int(lc.max())))
    return det, labels, counts, lc


def evaluate_labels(detections, labels, numlist):
    """evaluate() on label rows already read (one (rows, 15) float64 array per frame, evaluation.read_label_file)."""
    import numpy as np
    from .evaluation import eval_flags, get_thresholds, precision_curve
    det, labels, counts, lc = _eval_frames(detections, labels, numlist)
    dev = det.device
    frames = len(labels)
    out = np.full((6, 3, 3, EVAL_NSAMPLE), -1.0, np.float32)
    flags = eval_flags(det.cpu().numpy())
    if frames and any(any(f) for f in flags):
        rows = int(lc.sum())
        det_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
        label_off = np.concatenate([[0], np.cumsum(lc)]).astype(np.int32)
        pairs = counts * lc
        pair_off = np.concatenate([[0], np.cumsum(pairs)[:-1]]).astype(np.int64)
        up = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a)).to(dev, dt)
        d_det_off, d_label_off, d_pair_off = up(det_off, torch.int32), up(label_off, torch.int32), up(pair_off, torch.int64)
        d_lab = up(np.concatenate(labels, 0) if rows else np.zeros((0, 15)), torch.float64)
        ws = torch.empty((max(1, int(lib().ssd3d_eval_workspace(int(pairs.sum()))) // 8),), dtype=torch.float64, device=dev)
        md, ml = int(counts.max()), int(lc.max())
        args = (frames, md, ml, _p(det), _p(d_det_off), _p(d_lab), _p(d_label_off), _p(d_pair_off), _p(ws))
        check(lib().ssd3d_eval_overlaps(*args, _stream()), "evaluate")
        tp_scores = torch.empty((27, max(rows, 1)), dtype=torch.float64, device=dev)
        tp_count = torch.empty((27, frames), dtype=torch.int32, device=dev)
        n_gt = torch.empty((27, frames), dtype=torch.int32, device=dev)
        check(lib().ssd3d_eval_first_pass(*args, rows, _p(tp_scores), _p(tp_count), _p(n_gt), _stream()), "evaluate")
        # getThresholds on the host (float64, evaluate.cpp:539-572)
        scores, tpc, ngt = tp_scores.cpu().numpy(), tp_count.cpu().numpy(), n_gt.cpu().numpy()
        frame_of_row = np.repeat(np.arange(frames), lc)
        k_of_row = np.arange(rows) - label_off[:-1][frame_of_row]
        thr = np.zeros((27, EVAL_NSAMPLE), np.float64)
        nthr = np.zeros((27,), np.int32)
        for cs in range(27):
            if flags[cs // 9][(cs // 3) % 3]:
                t = get_thresholds(scores[cs, :rows][k_of_row < tpc[cs][frame_of_row]], int(ngt[cs].sum()))
                thr[cs, :len(t)], nthr[cs] = t, len(t)
        d_thr, d_nthr = up(thr, torch.float64), up(nthr, torch.int32)
        cnt = torch.empty((27, EVAL_NSAMPLE, 3), dtype=torch.int32, device=dev)
        check(lib().ssd3d_eval_count(*args, _p(d_thr), _p(d_nthr), _p(cnt), _stream()), "evaluate")
        cnt = cnt.cpu().numpy()
        for cs in range(27):
            m, c, d = cs // 9, (cs // 3) % 3, cs % 3
            if flags[m][c]:
                out[2 * m, c, d] = precision_curve(cnt[cs, :, 0], cnt[cs, :, 1], int(nthr[cs]))
    return tuple(torch.from_numpy(a.copy()).to(dev) for a in out)


# ---- the small elementwise stages (csrc/misc.cu): one kernel each, so a captured step holds no framework kernels ----

def fill_zero(t):
    """t[...] = 0 for a contiguous float32 CUDA tensor, as a kernel of this library."""
    t = _req(t, "t", torch.float32, copy=False)
    check(lib().ssd3d_fill_zero(_p(t), t.numel(), _stream()), "fill_zero")
    return t


def peer_allgather(send, peers, world, rank, slice_bytes, recv_off, flag_off, state, out):
    """All-gather of one slice per rank over NVLink peer memory (include/ssd3d.h, ssd3d_peer_allgather).
    send: uint8 [slice_bytes]; peers: int64 CUDA tensor [world] of the ranks' symmetric-buffer bases as mapped in THIS
    process; state: int32 [>= 3] zero-initialised, owned by this exchange (state[2] counts waits that timed out); out: uint8
    [world * slice_bytes]."""
    for name, t, dt in (("send", send, torch.uint8), ("peers", peers, torch.int64), ("state", state, torch.int32), ("out", out, torch.uint8)):
        _req(t, name, dt, copy=False)
    if send.numel() < slice_bytes or out.numel() < world * slice_bytes or peers.numel() < world or state.numel() < 3:
        raise ValueError("peer_allgather: buffers smaller than world=%d slices of %d bytes" % (world, slice_bytes))
    check(lib().ssd3d_peer_allgather(_p(send), int(slice_bytes), _p(peers), int(world), int(rank), int(recv_off[0]), int(recv_off[1]),
                                     int(flag_off[0]), int(flag_off[1]), _p(state), _p(out), _stream()), "peer_allgather")
    return out


# ---- data-parallel training: the gradient exchange (csrc/grad_exchange.cu, DESIGN.md section 3.9) -------------------

def grad_clip_scale(grad, norm, scale, clip_norm=5.0, workspace=None):
    """Global norm and tf.clip_by_global_norm scale of one rank's flat float32 gradient, written to the device floats
    norm[0] and scale[0] (include/ssd3d.h, ssd3d_grad_clip_scale).  workspace: optional uint8 buffer of
    ssd3d_grad_clip_scale_workspace bytes (allocated here when None)."""
    grad = _req(grad, "grad", torch.float32, copy=False)
    norm, scale = _req(norm, "norm", torch.float32, copy=False), _req(scale, "scale", torch.float32, copy=False)
    if grad.numel() == 0 or norm.numel() < 1 or scale.numel() < 1:
        raise ValueError("grad_clip_scale: grad must be non-empty and norm / scale hold one float each")
    if workspace is not None:
        workspace = _req(workspace, "workspace", torch.uint8, copy=False)
    ws_bytes = int(lib().ssd3d_grad_clip_scale_workspace(grad.numel()))
    if workspace is None:
        workspace = torch.empty((ws_bytes,), dtype=torch.uint8, device=grad.device)
    if workspace.numel() < ws_bytes:
        raise ValueError("grad_clip_scale: workspace must hold %d bytes" % ws_bytes)
    check(lib().ssd3d_grad_clip_scale(_p(grad), grad.numel(), float(clip_norm), _p(workspace), _p(norm), _p(scale), _stream()),
          "grad_clip_scale")
    return norm, scale


def peer_allreduce_resident_ctas():
    """CTAs of the allreduce kernel that fit co-resident on the current device (occupancy API)."""
    n = int(lib().ssd3d_peer_allreduce_resident_ctas())
    if n < 0:
        check(n, "peer_allreduce_resident_ctas")
    return n


def peer_allreduce_mean(grad, scale, peers, world, rank, layout, state):
    """Rank-ordered mean of the ranks' clipped gradients over NVLink peer memory, written back into grad (include/ssd3d.h,
    ssd3d_peer_allreduce_mean).  grad: float32 [n] 16-byte aligned; scale: this rank's device clip scale; peers: int64
    CUDA tensor [world] of the ranks' symmetric-buffer bases as mapped here; layout: dist.allreduce_layout(n, world,
    ctas) shifted to this exchange's share; state: int32 [>= 3] zero-initialised, owned by this exchange."""
    grad = _req(grad, "grad", torch.float32, copy=False)
    scale = _req(scale, "scale", torch.float32, copy=False)
    for name, t, dt in (("peers", peers, torch.int64), ("state", state, torch.int32)):
        _req(t, name, dt, copy=False)
    if grad.numel() == 0 or scale.numel() < 1 or peers.numel() < world or state.numel() < 3:
        raise ValueError("peer_allreduce_mean: grad must be non-empty, scale one float, peers >= world=%d, state >= 3" % world)
    if grad.numel() != layout.n or world != layout.world:
        raise ValueError("peer_allreduce_mean: layout is for n=%d world=%d, got n=%d world=%d"
                         % (layout.n, layout.world, grad.numel(), world))
    if grad.data_ptr() % 16:
        raise ValueError("peer_allreduce_mean: grad must be 16-byte aligned")
    check(lib().ssd3d_peer_allreduce_mean(_p(grad), grad.numel(), _p(scale), _p(peers), int(world), int(rank), int(layout.ctas),
                                          int(layout.chunk), int(layout.sub), int(layout.r1[0]), int(layout.r1[1]),
                                          int(layout.r2[0]), int(layout.r2[1]), int(layout.f1[0]), int(layout.f1[1]),
                                          int(layout.f2[0]), int(layout.f2[1]), _p(state), _stream()), "peer_allreduce_mean")
    return grad


def bn_moving_update_ranks(stats, batch, world, decay):
    """stats (float32 [n], in place) <- the BatchNorm moving-average update of `world` ranks in rank order from batch,
    float32 [world, ld >= n] (row r = rank r's batch means / variances at stats' offsets): ssd3d_bn_moving_update_ranks."""
    stats = _req(stats, "stats", torch.float32, copy=False)
    batch = _req(batch, "batch", torch.float32, 2, copy=None)
    n = stats.numel()
    if n == 0 or batch.shape[0] != world or batch.shape[1] < n or batch.stride(1) != 1 or batch.stride(0) < n:
        raise ValueError("bn_moving_update_ranks: batch %s (strides %s) must be [world=%d, >= %d] with unit column stride"
                         % (tuple(batch.shape), tuple(batch.stride()), world, n))
    if not 0.0 <= float(decay) <= 1.0:
        raise ValueError("bn_moving_update_ranks: decay=%g must be in [0, 1]" % decay)
    check(lib().ssd3d_bn_moving_update_ranks(_p(stats), n, _p(batch), batch.stride(0), int(world), float(decay), _stream()),
          "bn_moving_update_ranks")
    return stats


# ---- the solver: Adam and the weight operands (csrc/solver.cu, DESIGN.md section 3.11) -------------------------------

ADAM_STATE_INTS = 8           # the 32-byte state block as int32: [0:2] global_step, [2:5] float bits, [5] block counter


def adam_step(param, grad, m, v, state, boundaries, values, beta1=0.9, beta2=0.999, epsilon=1e-8):
    """One Adam step of the flat float32 buffers param / m / v (in place) from grad, in one launch (include/ssd3d.h,
    ssd3d_adam_step).  state: int32 CUDA [8], the device state block { global_step, beta1_power, beta2_power, lr_used };
    boundaries (<= 8 increasing ints) and values (one more float) are the piecewise-constant learning-rate schedule, read
    with the step before the increment."""
    bufs = [_req(t, name, torch.float32, 1, copy=False) for name, t in (("param", param), ("grad", grad), ("m", m), ("v", v))]
    state = _req(state, "state", torch.int32, 1, copy=False)
    n = bufs[0].numel()
    if n == 0 or any(t.numel() != n for t in bufs) or state.numel() < ADAM_STATE_INTS:
        raise ValueError("adam_step: param, grad, m, v must hold the same n > 0 floats and state %d int32" % ADAM_STATE_INTS)
    if any(t.data_ptr() % 16 for t in bufs) or state.data_ptr() % 8:
        raise ValueError("adam_step: param, grad, m, v must be 16-byte and state 8-byte aligned")
    nb = len(boundaries)
    if nb > 8 or len(values) != nb + 1:
        raise ValueError("adam_step: %d boundaries (at most 8) need %d values, got %d" % (nb, nb + 1, len(values)))
    bd = (ctypes.c_longlong * max(nb, 1))(*[int(b) for b in boundaries])
    vals = (ctypes.c_float * (nb + 1))(*[float(x) for x in values])
    check(lib().ssd3d_adam_step(*[_p(t) for t in bufs], n, _p(state), float(beta1), float(beta2), float(epsilon), nb,
                                ctypes.cast(bd, ctypes.c_void_p), ctypes.cast(vals, ctypes.c_void_p), _stream()), "adam_step")
    return param


def weight_operands(param, table, tiles, arena):
    """Rebuild the split-bf16 operands of every conv weight from the flat parameter buffer in one launch (include/ssd3d.h,
    ssd3d_weight_operands).  table: int64 CUDA [nw, 8] and tiles as laid out by params.operand_layout; arena: bfloat16."""
    param = _req(param, "param", torch.float32, 1, copy=False)
    table = _req(table, "table", torch.int64, 2, last=8, copy=False)
    arena = _req(arena, "arena", torch.bfloat16, 1, copy=False)
    if table.shape[0] == 0 or arena.data_ptr() % 16:
        raise ValueError("weight_operands: the table must have rows and the arena be 16-byte aligned")
    check(lib().ssd3d_weight_operands(_p(param), _p(table), table.shape[0], int(tiles), _p(arena), _stream()), "weight_operands")
    return arena


def split_points(points):
    """(b, n, 3 + c) -> xyz (b, n, 3), features (b, n, c): single_stage_detector.py:116-117."""
    points = _req(points, "points", torch.float32, 3)
    b, n, c = points.shape
    if c < 3:
        raise ValueError("points must have at least 3 channels")
    xyz = torch.empty((b, n, 3), dtype=torch.float32, device=points.device)
    feat = torch.empty((b, n, c - 3), dtype=torch.float32, device=points.device)
    check(lib().ssd3d_split_points(b * n, c, _p(points), _p(xyz), _p(feat) if c > 3 else ctypes.c_void_p(0), _stream()),
          "split_points")
    return xyz, feat


def iota_idx(b, npoint, device, *, out=None, start=0):
    """tf.tile(tf.range(npoint)) + start: the identity sampling of layers_util.py:91-92, :100-101."""
    o, optr, ldo = _idx_out(out, b, int(npoint), device)
    check(lib().ssd3d_iota_idx(b, int(npoint), int(start), ctypes.c_void_p(optr), ldo, _stream()), "iota_idx")
    return o


def concat_cols(a, bsrc):
    """tf.concat([a, bsrc], -1) for (b, n, ca) / (b, n, cb) float32 tensors whose scenes may be strided."""
    a, sa = _scene_strided(a, "a")
    bsrc, sb = _scene_strided(bsrc, "bsrc")
    b, n, ca = a.shape
    if bsrc.shape[:2] != (b, n):
        raise ValueError("concat_cols: leading shapes differ")
    cb = bsrc.shape[2]
    out = torch.empty((b, n, ca + cb), dtype=torch.float32, device=a.device)
    check(lib().ssd3d_concat_cols(b, n, ca, cb, _p(a), sa, _p(bsrc), sb, _p(out), _stream()), "concat_cols")
    return out


def vote_translate(xyz, offsets, min_range):
    """xyz + min(max(offsets, min_range), -min_range) (layers_util.py:20-23); offsets (b, n, >= 3)."""
    xyz = _req(xyz, "xyz", torch.float32, 3, 3)
    offsets = _req(offsets, "offsets", torch.float32, 3)
    if offsets.shape[:2] != xyz.shape[:2] or offsets.shape[2] < 3:
        raise ValueError("offsets must be (b, n, >= 3) like xyz")
    out = torch.empty_like(xyz)
    check(lib().ssd3d_vote_translate(xyz.shape[0] * xyz.shape[1], _p(xyz), _p(offsets), offsets.shape[2], float(min_range[0]),
                                     float(min_range[1]), float(min_range[2]), _p(out), _stream()), "vote_translate")
    return out


def decode_dist_anchor_free(center_xyz, pred_reg, pred_cls, angle_bins=12):
    """anchor_decoder.decode_dist_anchor_free + decode_class2angle + sigmoid in one kernel: center_xyz (b, n, 3),
    pred_reg (b, n, 6 + 2*angle_bins), pred_cls (b, n, >= 1) -> boxes (b, n, 7), scores (b, n)."""
    center_xyz = _req(center_xyz, "center_xyz", torch.float32, 3, 3)
    pred_reg = _req(pred_reg, "pred_reg", torch.float32, 3)
    pred_cls = _req(pred_cls, "pred_cls", torch.float32, 3)
    b, n, _ = center_xyz.shape
    if pred_reg.shape[:2] != (b, n) or pred_cls.shape[:2] != (b, n) or pred_reg.shape[2] < 6 + 2 * angle_bins:
        raise ValueError("pred_reg must be (b, n, >= 6 + 2*angle_bins) and pred_cls (b, n, >= 1)")
    boxes = torch.empty((b, n, 7), dtype=torch.float32, device=center_xyz.device)
    scores = torch.empty((b, n), dtype=torch.float32, device=center_xyz.device)
    check(lib().ssd3d_decode_dist_anchor_free(b * n, int(angle_bins), _p(center_xyz), _p(pred_reg), pred_reg.shape[2],
                                              _p(pred_cls), pred_cls.shape[2], _p(boxes), _p(scores), _stream()),
          "decode_dist_anchor_free")
    return boxes, scores


def concat_rows(parts):
    """tf.concat(parts, axis=1) for contiguous float32 (b, m_i, c) tensors (at most 8) in one kernel."""
    parts = [_req(t, "part", torch.float32, 3) for t in parts]
    if len(parts) == 1:
        return parts[0]
    if len(parts) > 8:
        raise ValueError("concat_rows joins at most 8 parts")
    b, _, c = parts[0].shape
    if any(t.shape[0] != b or t.shape[2] != c for t in parts):
        raise ValueError("concat_rows: parts must agree in batch and channel size")
    ms = [t.shape[1] for t in parts]
    out = torch.empty((b, sum(ms), c), dtype=torch.float32, device=parts[0].device)
    src = (ctypes.c_void_p * len(parts))(*[t.data_ptr() for t in parts])
    marr = (ctypes.c_int * len(parts))(*ms)
    check(lib().ssd3d_concat_rows(b, len(parts), ctypes.cast(src, ctypes.c_void_p), ctypes.cast(marr, ctypes.c_void_p), c,
                                  _p(out), _stream()), "concat_rows")
    return out


# ---- training-mode BatchNorm (SURVEY.md 8f row f3) -----------------------------------------------------------------

def bn_train(x, gamma, beta, moving_mean=None, moving_var=None, decay=0.9, relu=True, eps=BN_EPS, stats_out=None):
    """Batch-statistics BatchNorm + activation over the last axis of x (tf_util.py:424-444, is_training=True);
    moving_mean / moving_var (float32 CUDA tensors [c]) are updated IN PLACE like updates_collections=None does.
    Returns (y, scale, shift, batch_mean, batch_var); (scale, shift) is the folded per-channel form.
    stats_out: optional (mean, var) float32 CUDA tensors [c] that receive the batch statistics and are returned as
    batch_mean / batch_var (the BN record of data-parallel training writes them straight into its exchange buffer)."""
    x = _req(x, "x", torch.float32)
    c = x.shape[-1]
    rows = x.numel() // c
    for t, name in ((gamma, "gamma"), (beta, "beta"), (moving_mean, "moving_mean"), (moving_var, "moving_var")):
        if t is not None:
            _vec(t, name, c)
    if (moving_mean is None) != (moving_var is None):
        raise ValueError("moving_mean and moving_var go together")
    dev = x.device
    y = torch.empty_like(x)
    scale, shift = (torch.empty((c,), dtype=torch.float32, device=dev) for _ in range(2))
    if stats_out is None:
        bmean, bvar = (torch.empty((c,), dtype=torch.float32, device=dev) for _ in range(2))
    else:
        bmean, bvar = _vec(stats_out[0], "stats_out mean", c), _vec(stats_out[1], "stats_out var", c)
    ws = torch.empty((int(lib().ssd3d_bn_train_workspace(c)),), dtype=torch.uint8, device=dev)
    check(lib().ssd3d_bn_train(rows, c, _p(x), c, _p(gamma), _p(beta), _p(moving_mean), _p(moving_var), float(decay), float(eps),
                               _p(ws), _p(scale), _p(shift), _p(bmean), _p(bvar), 1 if relu else 0, _p(y), c, _stream()),
          "bn_train")
    return y, scale, shift, bmean, bvar


def rowgroup_max(y, pool, rowmask=None):
    """tf.reduce_max over runs of `pool` rows times (rowmask != 0) (layers_util.py:178-180): y (..., pool, c) -> (..., c)."""
    y = _req(y, "y", torch.float32)
    c, pool = y.shape[-1], int(pool)
    if y.shape[-2] != pool:
        raise ValueError("pool must equal the second-to-last dimension")
    rowmask = _rowmask(rowmask, y.numel() // (c * pool))
    out = torch.empty(tuple(y.shape[:-2]) + (c,), dtype=torch.float32, device=y.device)
    check(lib().ssd3d_rowgroup_max(y.numel() // (c * pool), pool, c, _p(y), c, _p(rowmask), _p(out), _stream()), "rowgroup_max")
    return out


# ---- backward of the training-mode layers (DESIGN.md "Backward") ---------------------------------------------------

def linear_wgrad(x, dz, want_bias=True):
    """Weight gradient of a 1x1 conv: x (..., cin), dz (..., cout) -> grad_w (cin, cout) = x^T dz over all rows and
    grad_b (cout,) = column sums of dz (None unless want_bias).  Tensor cores, fixed-order split-K: same bits every run."""
    x, dz = _req(x, "x", torch.float32), _req(dz, "dz", torch.float32)
    cin, cout = x.shape[-1], dz.shape[-1]
    rows = x.numel() // cin if cin else 0
    if cin == 0 or cout == 0 or dz.numel() // cout != rows or rows == 0:
        raise ValueError("linear_wgrad: x %s and dz %s must share their rows" % (tuple(x.shape), tuple(dz.shape)))
    ws_bytes = int(lib().ssd3d_linear_wgrad_workspace(rows, cin, cout))
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=x.device)
    gw = torch.empty((cin, cout), dtype=torch.float32, device=x.device)
    gb = torch.empty((cout,), dtype=torch.float32, device=x.device) if want_bias else None
    check(lib().ssd3d_linear_wgrad(rows, cin, cout, _p(x), cin, _p(dz), cout, _p(ws), ws_bytes, _p(gw), _p(gb), _stream()),
          "linear_wgrad")
    return gw, gb


def bn_train_grad(x, grad_out, scale, shift, batch_mean, batch_var, gamma, relu=True, eps=BN_EPS):
    """Backward of bn_train (+ ReLU) from its input x (the pre-BN conv output) and its outputs (scale, shift, batch_mean,
    batch_var) -> (grad_x, grad_gamma, grad_beta).  The moving statistics are not touched."""
    x, grad_out = _req(x, "x", torch.float32), _req(grad_out, "grad_out", torch.float32)
    if grad_out.shape != x.shape:
        raise ValueError("bn_train_grad: grad_out %s must have the shape of x %s" % (tuple(grad_out.shape), tuple(x.shape)))
    c = x.shape[-1]
    rows = x.numel() // c
    for t, name in ((scale, "scale"), (shift, "shift"), (batch_mean, "batch_mean"), (batch_var, "batch_var"), (gamma, "gamma")):
        _vec(t, name, c)
    dev = x.device
    gx = torch.empty_like(x)
    gg, gbeta = (torch.empty((c,), dtype=torch.float32, device=dev) for _ in range(2))
    ws = torch.empty((int(lib().ssd3d_bn_train_grad_workspace(c)),), dtype=torch.uint8, device=dev)
    check(lib().ssd3d_bn_train_grad(rows, c, _p(x), c, _p(grad_out), c, _p(scale), _p(shift), _p(batch_mean), _p(batch_var),
                                    _p(gamma), float(eps), 1 if relu else 0, _p(ws), _p(gg), _p(gbeta), _p(gx), c, _stream()),
          "bn_train_grad")
    return gx, gg, gbeta


def rowgroup_max_grad(y, grad_out, pool, rowmask=None):
    """Backward of rowgroup_max: y (..., pool, c), grad_out (..., c) -> grad_y (..., pool, c); the gradient of a group is
    split evenly among its tied maxima and multiplied by (rowmask != 0)."""
    y, grad_out = _req(y, "y", torch.float32), _req(grad_out, "grad_out", torch.float32)
    c, pool = y.shape[-1], int(pool)
    if y.dim() < 2 or y.shape[-2] != pool or tuple(grad_out.shape) != tuple(y.shape[:-2]) + (c,):
        raise ValueError("rowgroup_max_grad: y must be (..., pool, c) and grad_out (..., c)")
    groups = grad_out.numel() // c
    rowmask = _rowmask(rowmask, groups)
    gy = torch.empty_like(y)
    check(lib().ssd3d_rowgroup_max_grad(groups, pool, c, _p(y), c, _p(rowmask), _p(grad_out), _p(gy), c, _stream()),
          "rowgroup_max_grad")
    return gy


def group_concat_grad(grad_x, idx, n, c, want_points=True, want_xyz=True, want_new_xyz=True):
    """Backward of group_concat: grad_x (b, m, nsample, ldx) -> (grad_points (b, n, c), grad_xyz (b, n, 3),
    grad_new_xyz (b, m, 3)); an output not wanted is None."""
    grad_x = _req(grad_x, "grad_x", torch.float32, 4)
    idx = _req(idx, "idx", torch.int32, 3)
    b, m, ns, ldx = grad_x.shape
    if tuple(idx.shape) != (b, m, ns) or ldx < c + 3 or int(n) <= 0:
        raise ValueError("group_concat_grad: grad_x %s does not match idx %s with c = %d" % (tuple(grad_x.shape), tuple(idx.shape), c))
    dev = grad_x.device
    gp = torch.empty((b, n, c), dtype=torch.float32, device=dev) if (want_points and c > 0) else None
    gxyz = torch.empty((b, n, 3), dtype=torch.float32, device=dev) if want_xyz else None
    gnew = torch.empty((b, m, 3), dtype=torch.float32, device=dev) if want_new_xyz else None
    check(lib().ssd3d_group_concat_grad(b, int(n), int(c), m, ns, _p(idx), _p(grad_x), ldx, _p(gp), _p(gxyz), _p(gnew), _stream()),
          "group_concat_grad")
    return gp, gxyz, gnew


def vote_translate_grad(offsets, grad_out, min_range):
    """Backward of vote_translate w.r.t. the offsets (b, n, >= 3): grad_out (b, n, 3) where min <= offset <= -min
    (inclusive), else 0 -> (b, n, 3)."""
    offsets, grad_out = _req(offsets, "offsets", torch.float32, 3), _req(grad_out, "grad_out", torch.float32, 3, 3)
    if offsets.shape[:2] != grad_out.shape[:2] or offsets.shape[2] < 3:
        raise ValueError("offsets must be (b, n, >= 3) like grad_out")
    g = torch.empty_like(grad_out)
    check(lib().ssd3d_vote_translate_grad(grad_out.shape[0] * grad_out.shape[1], _p(offsets), offsets.shape[2], _p(grad_out),
                                          float(min_range[0]), float(min_range[1]), float(min_range[2]), _p(g), _stream()),
          "vote_translate_grad")
    return g


def linear_bn_train(x, f, gamma=None, beta=None, moving_mean=None, moving_var=None, bn=True, relu=True, decay=0.9,
                    stats_out=None):
    """Forward of one training-mode layer: split_rows -> linear_tc with the BN-less fold f (params.FoldedConv with
    scale = 1, shift = bias) -> bn_train (bn=True: batch statistics, moving statistics updated in place) -> ReLU.
    Returns (y, r): y the conv output before BatchNorm, r bn_train's (out, scale, shift, batch_mean, batch_var), or (y,)
    when bn=False.  stats_out: see bn_train."""
    hi, lo = split_rows(x)
    y, _ = linear_tc(hi, lo, f, relu=bool(relu and not bn), want_f32=True, want_split=False)
    if not bn:
        return y, (y,)
    extra = {} if stats_out is None else {"stats_out": stats_out}
    return y, bn_train(y, gamma, beta, moving_mean, moving_var, decay=decay, relu=relu, **extra)


class _ConvTrain(torch.autograd.Function):
    """conv (+bias) -> [training BatchNorm] -> [ReLU] of one layer (tf_util.conv2d / conv1d with is_training=True).
    Forward: linear_bn_train with a fold of the live weights, the sequence of the non-trainable training path.
    Backward: bn_train_grad -> split -> linear_tc with W^T (grad_x) and linear_wgrad (grad_w, grad_b).
    opts may end with operands = (forward fold, grad-x fold) prebuilt from the same weights (params.TrainableParams'
    operand cache): they are then used instead of building both folds here."""

    @staticmethod
    def forward(ctx, x, w, b, gamma, beta, opts):
        bn, relu, decay, moving, debug, stats_out = opts[:6]
        operands = opts[6] if len(opts) > 6 else None
        x = x if x.is_contiguous() else x.contiguous()
        if operands is None:
            f = FoldedConv(w.detach(), torch.ones((w.shape[1],), dtype=torch.float32, device=x.device), b.detach())
        else:
            f = operands[0]
        y, r = linear_bn_train(x, f, gamma.detach(), beta.detach(), moving[0], moving[1],
                               bn=bn, relu=relu, decay=decay, stats_out=stats_out)
        out = r[0]
        ctx.bn, ctx.relu = bn, relu
        ctx.wt = None if operands is None else operands[1]
        if bn:
            ctx.save_for_backward(x, w, y, *r[1:], gamma)       # scale, shift, batch_mean, batch_var
        else:
            ctx.save_for_backward(x, w, y)
        if debug is not None:
            debug.append((y, out))
        return out

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous()
        x, w, y = ctx.saved_tensors[:3]
        ggamma = gbeta = None
        if ctx.bn:
            scale, shift, bmean, bvar, gamma = ctx.saved_tensors[3:]
            dz, ggamma, gbeta = bn_train_grad(y, g, scale, shift, bmean, bvar, gamma, relu=ctx.relu)
        elif ctx.relu:
            dz = torch.where(y > 0, g, torch.zeros((), dtype=g.dtype, device=g.device))   # ReluGrad: output > 0
        else:
            dz = g
        cin, cout = w.shape
        gx = None
        if ctx.needs_input_grad[0]:
            d_hi, d_lo = split_rows(dz)
            wt = ctx.wt
            if wt is None:
                wt = FoldedConv(w.detach().t().contiguous(), torch.ones((cin,), dtype=torch.float32, device=dz.device),
                                torch.zeros((cin,), dtype=torch.float32, device=dz.device))
            gx, _ = linear_tc(d_hi, d_lo, wt, relu=False, want_f32=True, want_split=False)
        gw, gb = linear_wgrad(x, dz, want_bias=True)
        return gx, gw, gb, ggamma, gbeta, None


def conv_train(x, w, b, gamma=None, beta=None, moving_mean=None, moving_var=None, bn=True, relu=True, decay=0.9, debug=None,
               stats_out=None, operands=None):
    """Differentiable conv (+bias) -> training BatchNorm (bn=True; updates moving_mean / moving_var in place) -> ReLU of
    one layer over the last axis of x, with the forward bits of the non-trainable training path.  x (..., cin),
    w (cin, cout), b / gamma / beta (cout,).  debug: a list that receives (pre-BN conv output, layer output).
    stats_out: optional (mean, var) [cout] that receive the batch statistics (bn=True; kept for the backward).
    operands: optional (forward fold of w with scale 1 and shift b, grad-x fold of w^T with scale 1 and shift 0), current
    for w -- the caller's promise; both are otherwise built here on every call."""
    if not isinstance(x, torch.Tensor) or x.dtype != torch.float32:     # the device is checked by the kernels' wrappers
        raise ValueError("x must be a float32 tensor")
    if w.dim() != 2 or x.shape[-1] != w.shape[0] or tuple(b.shape) != (w.shape[1],):
        raise ValueError("conv_train: x %s, w %s, b %s do not match" % (tuple(x.shape), tuple(w.shape), tuple(b.shape)))
    if bn and (gamma is None or beta is None):
        raise ValueError("conv_train: bn=True needs gamma and beta")
    z = torch.zeros((0,), dtype=torch.float32, device=x.device)
    return _ConvTrain.apply(x, w, b, gamma if bn else z, beta if bn else z,
                            (bool(bn), bool(relu), float(decay), (moving_mean, moving_var), debug, stats_out, operands))


class _GroupMax(torch.autograd.Function):
    @staticmethod
    def forward(ctx, y, pool, rowmask):
        ctx.save_for_backward(y, rowmask)
        ctx.pool = pool
        return rowgroup_max(y, pool, rowmask)

    @staticmethod
    def backward(ctx, g):
        y, rowmask = ctx.saved_tensors
        return rowgroup_max_grad(y, g.contiguous(), ctx.pool, rowmask), None, None


def group_max_train(y, pool, rowmask=None):
    """Differentiable rowgroup_max (tf.reduce_max(axis=2) * mask): ties share the gradient evenly, as in TF."""
    return _GroupMax.apply(y, int(pool), rowmask)


class _GroupConcat(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xyz, points, new_xyz, idx):
        ctx.save_for_backward(idx)
        ctx.n, ctx.c = xyz.shape[1], 0 if points is None else points.shape[2]
        return group_concat(xyz, points, new_xyz, idx)

    @staticmethod
    def backward(ctx, g):
        (idx,) = ctx.saved_tensors
        need = ctx.needs_input_grad
        gp, gxyz, gnew = group_concat_grad(g.contiguous(), idx, ctx.n, ctx.c, need[1], need[0], need[2])
        return gxyz, gp, gnew, None


def group_concat_train(xyz, points, new_xyz, idx):
    """Differentiable group_concat: gradients reach points, xyz and the query centres new_xyz."""
    return _GroupConcat.apply(xyz, points, new_xyz, idx)


class _VoteTranslate(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xyz, offsets, min_range):
        ctx.save_for_backward(offsets)
        ctx.min_range = min_range
        return vote_translate(xyz, offsets, min_range)

    @staticmethod
    def backward(ctx, g):
        (offsets,) = ctx.saved_tensors
        g = g.contiguous()
        return g, vote_translate_grad(offsets, g, ctx.min_range), None


def vote_translate_train(xyz, offsets, min_range):
    """Differentiable vote_translate: identity for xyz, the clamp's gradient (inclusive bounds) for the offsets."""
    return _VoteTranslate.apply(xyz, offsets, tuple(float(v) for v in min_range))


# ---- training targets and detection losses (DESIGN.md section 3.8) --------------------------------------------------

DET_TARGETS = ("assigned_idx", "assigned_box", "pmask", "nmask", "cls_label", "angle_bin", "angle_res", "offset_target",
               "vote_mask", "vote_target")
_LOSS_TARGETS = ("assigned_box", "pmask", "nmask", "cls_label", "angle_bin", "angle_res", "vote_mask", "vote_target")


def det_assign(base_xyz, vote_base, gt_boxes, gt_labels, angle_bins=12):
    """'Mask' assignment + vote targets (ssd3d_det_assign): base_xyz (b, n, 3), vote_base (b, nv, 3), gt_boxes (b, g, 7)
    zero-padded, gt_labels (b, g) int32 -> dict of the DET_TARGETS tensors."""
    base_xyz = _req(base_xyz, "base_xyz", torch.float32, 3, 3)
    vote_base = _req(vote_base, "vote_base", torch.float32, 3, 3)
    gt_boxes = _req(gt_boxes, "gt_boxes", torch.float32, 3, 7)
    gt_labels = _req(gt_labels, "gt_labels", torch.int32, 2)
    b, n, _ = base_xyz.shape
    nv, g = vote_base.shape[1], gt_boxes.shape[1]
    if vote_base.shape[0] != b or gt_boxes.shape[0] != b or tuple(gt_labels.shape) != (b, g):
        raise ValueError("det_assign: base_xyz %s, vote_base %s, gt_boxes %s, gt_labels %s do not share the batch"
                         % (tuple(base_xyz.shape), tuple(vote_base.shape), tuple(gt_boxes.shape), tuple(gt_labels.shape)))
    dev = base_xyz.device
    f = lambda *s: torch.empty(s, dtype=torch.float32, device=dev)
    i = lambda *s: torch.empty(s, dtype=torch.int32, device=dev)
    t = dict(assigned_idx=i(b, n), assigned_box=f(b, n, 7), pmask=f(b, n), nmask=f(b, n), cls_label=f(b, n),
             angle_bin=i(b, n), angle_res=f(b, n), offset_target=f(b, n, 6), vote_mask=f(b, nv), vote_target=f(b, nv, 3))
    check(lib().ssd3d_det_assign(b, n, nv, g, int(angle_bins), _p(base_xyz), _p(vote_base), _p(gt_boxes), _p(gt_labels),
                                 *[_p(t[k]) for k in DET_TARGETS], _stream()), "det_assign")
    return t


def _rows(t, name, b, n, width):
    """(b, n, [1,] width) float32 CUDA tensor, read in place when its last axis is dense and its rows evenly strided (a
    column block of a wider tensor, e.g. the head's [b, n, 1, 30] regression output) -> (tensor, row stride in floats)."""
    t = _req(t, name, torch.float32, copy=None)
    if t.dim() < 3 or tuple(t.shape[:2]) != (b, n) or t.shape[-1] != width or any(s != 1 for s in t.shape[2:-1]):
        raise ValueError("%s must be (%d, %d, [1,] %d), got %s" % (name, b, n, width, tuple(t.shape)))
    ld = t.stride(1)
    if t.stride(-1) != 1 or ld < width or (b > 1 and t.stride(0) != n * ld):
        t, ld = t.contiguous(), width
    return t, ld


def _det_inputs(base_xyz, pred_cls, pred_offset, pred_angle_cls, pred_angle_res, vote_offset, tg, angle_bins):
    base_xyz = _req(base_xyz, "base_xyz", torch.float32, 3, 3)
    b, n, _ = base_xyz.shape
    nv = tg["vote_mask"].shape[1]
    ins = [(base_xyz,)]
    for t, name, w in ((pred_cls, "pred_cls", 1), (pred_offset, "pred_offset", 6), (pred_angle_cls, "pred_angle_cls", angle_bins),
                       (pred_angle_res, "pred_angle_res", angle_bins)):
        ins.append(_rows(t, name, b, n, w))
    ins.append(_rows(vote_offset, "vote_offset", b, nv, 3))
    for k in _LOSS_TARGETS:
        if tg[k].shape[:2] != (b, nv if k.startswith("vote") else n):
            raise ValueError("target %s %s does not match the inputs" % (k, tuple(tg[k].shape)))
    return b, n, nv, ins


def _det_args(ins, tg):
    args = [_p(ins[0][0])]
    for t, ld in ins[1:]:
        args += [_p(t), ld]
    return args + [_p(tg[k]) for k in _LOSS_TARGETS]


def det_loss(base_xyz, pred_cls, pred_offset, pred_angle_cls, pred_angle_res, vote_offset, tg, angle_bins=12):
    """The six detection losses (ssd3d_det_loss) -> (loss (6,) = cls, offset, angle bin, angle residual, corner, vote;
    norm (3,) = the classification, positive and vote normalisers).  The head outputs are read in place."""
    b, n, nv, ins = _det_inputs(base_xyz, pred_cls, pred_offset, pred_angle_cls, pred_angle_res, vote_offset, tg, angle_bins)
    dev = ins[0][0].device
    ws = torch.empty((int(lib().ssd3d_det_loss_workspace(b)),), dtype=torch.uint8, device=dev)
    loss = torch.empty((6,), dtype=torch.float32, device=dev)
    norm = torch.empty((3,), dtype=torch.float32, device=dev)
    check(lib().ssd3d_det_loss(b, n, nv, int(angle_bins), *_det_args(ins, tg), _p(ws), _p(loss), _p(norm), _stream()), "det_loss")
    return loss, norm


def det_loss_grad(base_xyz, pred_cls, pred_offset, pred_angle_cls, pred_angle_res, vote_offset, tg, grad_loss, norm, angle_bins=12):
    """Backward of det_loss from grad_loss (6,) -> (grad_base_xyz (b, n, 3), grad_cls (b, n, 1), grad_reg (b, n, 6 + 2 *
    angle_bins) laid out as the head's [offset | angle logits | angle residuals], grad_vote_offset (b, nv, 3))."""
    b, n, nv, ins = _det_inputs(base_xyz, pred_cls, pred_offset, pred_angle_cls, pred_angle_res, vote_offset, tg, angle_bins)
    grad_loss, norm = _req(grad_loss, "grad_loss", torch.float32, 1, 6), _req(norm, "norm", torch.float32, 1, 3)
    dev = ins[0][0].device
    ldr = 6 + 2 * angle_bins
    gbase = torch.empty((b, n, 3), dtype=torch.float32, device=dev)
    gcls = torch.empty((b, n, 1), dtype=torch.float32, device=dev)
    greg = torch.empty((b, n, ldr), dtype=torch.float32, device=dev)
    gvote = torch.empty((b, nv, 3), dtype=torch.float32, device=dev)
    check(lib().ssd3d_det_loss_grad(b, n, nv, int(angle_bins), *_det_args(ins, tg), _p(grad_loss), _p(norm), _p(gbase), _p(gcls), 1,
                                    _p(greg), ldr, ctypes.c_void_p(greg.data_ptr() + 4 * 6), ldr,
                                    ctypes.c_void_p(greg.data_ptr() + 4 * (6 + angle_bins)), ldr, _p(gvote), _stream()),
          "det_loss_grad")
    return gbase, gcls, greg, gvote


class _DetLoss(torch.autograd.Function):
    """det_loss forward; det_loss_grad backward (one kernel for every input's gradient)."""

    @staticmethod
    def forward(ctx, base_xyz, pred_cls, pred_offset, pred_angle_cls, pred_angle_res, vote_offset, tg, angle_bins):
        loss, norm = det_loss(base_xyz, pred_cls, pred_offset, pred_angle_cls, pred_angle_res, vote_offset, tg, angle_bins)
        ctx.save_for_backward(base_xyz, pred_cls, pred_offset, pred_angle_cls, pred_angle_res, vote_offset, norm)
        ctx.tg, ctx.angle_bins = tg, angle_bins
        return loss

    @staticmethod
    def backward(ctx, g):
        base_xyz, pred_cls, pred_offset, pred_angle_cls, pred_angle_res, vote_offset, norm = ctx.saved_tensors
        nb = ctx.angle_bins
        gbase, gcls, greg, gvote = det_loss_grad(base_xyz, pred_cls, pred_offset, pred_angle_cls, pred_angle_res, vote_offset,
                                                 ctx.tg, g.contiguous(), norm, nb)
        return (gbase, gcls.reshape(pred_cls.shape), greg[..., :6].reshape(pred_offset.shape),
                greg[..., 6:6 + nb].reshape(pred_angle_cls.shape), greg[..., 6 + nb:].reshape(pred_angle_res.shape), gvote, None, None)


def det_loss_train(base_xyz, pred_cls, pred_offset, pred_angle_cls, pred_angle_res, vote_offset, tg, angle_bins=12):
    """Differentiable det_loss -> loss (6,); gradients reach base_xyz, the four head outputs and vote_offset."""
    return _DetLoss.apply(base_xyz, pred_cls, pred_offset, pred_angle_cls, pred_angle_res, vote_offset, tg, int(angle_bins))


# ---- training-scene augmentation (csrc/augment.cu, DESIGN.md section 3.12) -------------------------------------------
AUG_TRIES = 100               # noise tries per box
AUG_MAX_BOXES = 256           # GT rows per scene
AUG_MAX_POINTS = 131072       # points per scene
AUG_MAX_CHOOSE = 16384        # points chosen per scene (sorted in shared memory)


def _aug_ragged(points, offsets, max_n):
    """points [T, 4] float32 and device offsets [b + 1] int32 of ragged scenes whose largest holds max_n points."""
    points = _req(points, "points", torch.float32, 2, 4)
    offsets = _req(offsets, "offsets", torch.int32, 1)
    if offsets.shape[0] < 2:
        raise ValueError("offsets must hold b + 1 >= 2 entries, got %d" % offsets.shape[0])
    if not 1 <= int(max_n) <= AUG_MAX_POINTS:
        raise ValueError("a scene must hold 1 .. %d points, got max_n=%d" % (AUG_MAX_POINTS, max_n))
    return points, offsets, offsets.shape[0] - 1


def _aug_boxes_in(gt_boxes, b=None):
    gt_boxes = _req(gt_boxes, "gt_boxes", torch.float32, 3, 7)
    if b is not None and gt_boxes.shape[0] != b:
        raise ValueError("gt_boxes %s does not hold %d scenes" % (tuple(gt_boxes.shape), b))
    if gt_boxes.shape[1] > AUG_MAX_BOXES:
        raise ValueError("at most %d GT rows per scene, got %d" % (AUG_MAX_BOXES, gt_boxes.shape[1]))
    return gt_boxes


def augment_sem_labels(points, offsets, gt_boxes, gt_labels, max_n):
    """Semantic labels of ragged scenes (ssd3d_augment_sem_labels) -> [T] int32: the class of the first valid box grown by
    0.1 that holds the point, else 0."""
    points, offsets, b = _aug_ragged(points, offsets, max_n)
    gt_boxes = _aug_boxes_in(gt_boxes, b)
    gt_labels = _req(gt_labels, "gt_labels", torch.int32, 2)
    if tuple(gt_labels.shape) != tuple(gt_boxes.shape[:2]):
        raise ValueError("gt_labels %s does not match gt_boxes %s" % (tuple(gt_labels.shape), tuple(gt_boxes.shape)))
    sem = torch.empty((points.shape[0],), dtype=torch.int32, device=points.device)
    check(lib().ssd3d_augment_sem_labels(b, gt_boxes.shape[1], int(max_n), _p(points), _p(offsets), _p(gt_boxes), _p(gt_labels),
                                         _p(sem), _stream()), "augment_sem_labels")
    return sem


def augment_boxes(gt_boxes, scene_u, loc_noise, rot_u):
    """Flip, per-object noise, global rotation and scale of the boxes (ssd3d_augment_boxes) -> (boxes [b, g, 7], chosen
    try [b, g] int32, -1 for none, workspace uint8 for augment_points)."""
    gt_boxes = _aug_boxes_in(gt_boxes)
    b, g = gt_boxes.shape[:2]
    scene_u = _req(scene_u, "scene_u", torch.float64, 2, 6)
    loc_noise = _req(loc_noise, "loc_noise", torch.float64, 4, 2)
    rot_u = _req(rot_u, "rot_u", torch.float64, 3)
    if scene_u.shape[0] != b or tuple(loc_noise.shape[:3]) != (b, g, AUG_TRIES) or tuple(rot_u.shape) != (b, g, AUG_TRIES):
        raise ValueError("draws scene_u %s, loc_noise %s, rot_u %s do not match gt_boxes %s" % (
            tuple(scene_u.shape), tuple(loc_noise.shape), tuple(rot_u.shape), tuple(gt_boxes.shape)))
    dev = gt_boxes.device
    out = torch.empty((b, g, 7), dtype=torch.float32, device=dev)
    chosen = torch.empty((b, g), dtype=torch.int32, device=dev)
    ws = torch.empty((int(lib().ssd3d_augment_workspace(b, g)),), dtype=torch.uint8, device=dev)
    check(lib().ssd3d_augment_boxes(b, g, _p(gt_boxes), _p(scene_u), _p(loc_noise), _p(rot_u), _p(out), _p(chosen), _p(ws),
                                    _stream()), "augment_boxes")
    return out, chosen, ws


def augment_points(points, offsets, max_n, sem_labels, keys, workspace, g, want_moved=False):
    """Flip, noise move, global transform and context filter of the points (ssd3d_augment_points) with the workspace of
    augment_boxes for g GT rows -> (points [T, 4], sort keys [T] int64 (-1: dropped), survivors [b] int32, the box
    that moved each point [T] int32 (-1: none) when want_moved else None)."""
    points, offsets, b = _aug_ragged(points, offsets, max_n)
    t = points.shape[0]
    sem_labels = _req(sem_labels, "sem_labels", torch.int32, 1)
    keys = _req(keys, "keys", torch.int32, 1)
    workspace = _req(workspace, "workspace", torch.uint8, 1, copy=False)
    if sem_labels.shape[0] != t or keys.shape[0] != t:
        raise ValueError("sem_labels %s and keys %s must hold one entry per point (%d)" % (
            tuple(sem_labels.shape), tuple(keys.shape), t))
    if not 0 <= int(g) <= AUG_MAX_BOXES or workspace.numel() < int(lib().ssd3d_augment_workspace(b, int(g))):
        raise ValueError("workspace does not come from augment_boxes of %d scenes x %d rows" % (b, g))
    dev = points.device
    out = torch.empty((t, 4), dtype=torch.float32, device=dev)
    sort_keys = torch.empty((t,), dtype=torch.int64, device=dev)
    survivors = torch.empty((b,), dtype=torch.int32, device=dev)
    moved = torch.empty((t,), dtype=torch.int32, device=dev) if want_moved else None
    check(lib().ssd3d_augment_points(b, int(g), int(max_n), _p(points), _p(offsets), _p(sem_labels), _p(keys), _p(workspace),
                                     _p(out), _p(sort_keys), _p(survivors), _p(moved), _stream()), "augment_points")
    return out, sort_keys, survivors, moved


def augment_choose(points, offsets, sort_keys, survivors, refill):
    """The point choice (ssd3d_augment_choose) -> [b, num_points, 4], num_points = refill.shape[1]."""
    points = _req(points, "points", torch.float32, 2, 4)
    offsets = _req(offsets, "offsets", torch.int32, 1)
    sort_keys = _req(sort_keys, "sort_keys", torch.int64, 1)
    survivors = _req(survivors, "survivors", torch.int32, 1)
    refill = _req(refill, "refill", torch.int32, 2)
    b, m = refill.shape
    if offsets.shape[0] != b + 1 or survivors.shape[0] != b or sort_keys.shape[0] != points.shape[0]:
        raise ValueError("augment_choose: offsets %s, survivors %s, sort_keys %s, points %s, refill %s disagree" % (
            tuple(offsets.shape), tuple(survivors.shape), tuple(sort_keys.shape), tuple(points.shape), tuple(refill.shape)))
    if not 1 <= m <= AUG_MAX_CHOOSE:
        raise ValueError("num_points must be 1 .. %d, got %d" % (AUG_MAX_CHOOSE, m))
    out = torch.empty((b, m, 4), dtype=torch.float32, device=points.device)
    check(lib().ssd3d_augment_choose(b, m, _p(points), _p(offsets), _p(sort_keys), _p(survivors), _p(refill), _p(out), _stream()),
          "augment_choose")
    return out


# ---- mixup paste and its object database (csrc/mixup.cu, DESIGN.md section 3.13) -------------------------------------
MIXUP_MAX_ROWS = 256          # GT rows plus drawn objects per scene
MIXUP_MAX_SLOTS = AUG_MAX_POINTS


def mixup_db_count(points, offsets, max_n, gt_boxes):
    """Points of each frame inside each valid GT row grown by 0.1 (ssd3d_mixup_db_count) -> counts [b, g] int32."""
    points, offsets, b = _aug_ragged(points, offsets, max_n)
    gt_boxes = _aug_boxes_in(gt_boxes, b)
    if gt_boxes.shape[1] < 1:
        raise ValueError("mixup_db_count needs at least one GT row")
    counts = torch.empty((b, gt_boxes.shape[1]), dtype=torch.int32, device=points.device)
    check(lib().ssd3d_mixup_db_count(b, gt_boxes.shape[1], int(max_n), _p(points), _p(offsets), _p(gt_boxes), _p(counts),
                                     _stream()), "mixup_db_count")
    return counts


def mixup_db_write(points, offsets, gt_boxes, objects, object_offsets, total):
    """The points of each database object (ssd3d_mixup_db_write): objects [O, 2] int32 (frame, row), object_offsets [O + 1]
    int64 (device), total = object_offsets[-1] -> points [total, 4], each object's points in frame order."""
    points = _req(points, "points", torch.float32, 2, 4)
    offsets = _req(offsets, "offsets", torch.int32, 1)
    gt_boxes = _aug_boxes_in(gt_boxes, offsets.shape[0] - 1)
    objects = _req(objects, "objects", torch.int32, 2, 2)
    object_offsets = _req(object_offsets, "object_offsets", torch.int64, 1)
    o = objects.shape[0]
    if object_offsets.shape[0] != o + 1 or o < 1 or gt_boxes.shape[1] < 1:
        raise ValueError("objects %s and object_offsets %s disagree (or hold no object)" % (
            tuple(objects.shape), tuple(object_offsets.shape)))
    out = torch.empty((int(total), 4), dtype=torch.float32, device=points.device)
    check(lib().ssd3d_mixup_db_write(gt_boxes.shape[1], o, _p(points), _p(offsets), _p(gt_boxes), _p(objects), _p(object_offsets),
                                     _p(out), _stream()), "mixup_db_write")
    return out


def _mixup_db_in(db_boxes, db_classes):
    db_boxes = _req(db_boxes, "db_boxes", torch.float32, 2, 7)
    db_classes = _req(db_classes, "db_classes", torch.int32, 1)
    if db_classes.shape[0] != db_boxes.shape[0]:
        raise ValueError("db_classes %s does not match db_boxes %s" % (tuple(db_classes.shape), tuple(db_boxes.shape)))
    return db_boxes, db_classes


def mixup_paste_boxes(gt_boxes, gt_labels, ids, db_boxes, db_classes, planes):
    """box_3d_collision_test of the drawn objects ids [b, s] int32 (-1: none) against each scene (ssd3d_mixup_paste_boxes)
    -> (boxes [b, g + s, 7], labels [b, g + s] int32, accepted [b, s] int32).  The ids must be in range (checked on the
    host by mixup.layout)."""
    gt_boxes = _aug_boxes_in(gt_boxes)
    b, g = gt_boxes.shape[:2]
    gt_labels = _req(gt_labels, "gt_labels", torch.int32, 2)
    ids = _req(ids, "ids", torch.int32, 2)
    db_boxes, db_classes = _mixup_db_in(db_boxes, db_classes)
    planes = _req(planes, "planes", torch.float64, 2, 4)
    s = ids.shape[1]
    if tuple(gt_labels.shape) != (b, g) or ids.shape[0] != b or planes.shape[0] != b:
        raise ValueError("gt_boxes %s, gt_labels %s, ids %s and planes %s disagree" % (
            tuple(gt_boxes.shape), tuple(gt_labels.shape), tuple(ids.shape), tuple(planes.shape)))
    if s < 1 or g + s > MIXUP_MAX_ROWS:
        raise ValueError("GT rows plus drawn objects must be at most %d (and s >= 1), got %d + %d" % (MIXUP_MAX_ROWS, g, s))
    dev = gt_boxes.device
    out = torch.empty((b, g + s, 7), dtype=torch.float32, device=dev)
    labels = torch.empty((b, g + s), dtype=torch.int32, device=dev)
    accepted = torch.empty((b, s), dtype=torch.int32, device=dev)
    check(lib().ssd3d_mixup_paste_boxes(b, g, s, _p(gt_boxes), _p(gt_labels), _p(ids), _p(db_boxes), _p(db_classes), _p(planes),
                                        _p(out), _p(labels), _p(accepted), _stream()), "mixup_paste_boxes")
    return out, labels, accepted


def mixup_paste_points(points, offsets, sem_labels, ids, db_points, db_offsets, db_boxes, db_classes, planes, accepted,
                       out_offsets, slot_start, max_slots, total):
    """The pasted clouds (ssd3d_mixup_paste_points) of the layout out_offsets [b + 1], slot_start [b, s + 1] (device int32,
    from mixup.layout), total = out_offsets[-1] -> (points [total, 4], semantic labels [total] int32, -1 where a dropped
    object's slot holds no point)."""
    points = _req(points, "points", torch.float32, 2, 4)
    offsets = _req(offsets, "offsets", torch.int32, 1)
    b = offsets.shape[0] - 1
    sem_labels = _req(sem_labels, "sem_labels", torch.int32, 1)
    ids = _req(ids, "ids", torch.int32, 2)
    db_points = _req(db_points, "db_points", torch.float32, 2, 4)
    db_offsets = _req(db_offsets, "db_offsets", torch.int64, 1)
    db_boxes, db_classes = _mixup_db_in(db_boxes, db_classes)
    planes = _req(planes, "planes", torch.float64, 2, 4)
    accepted = _req(accepted, "accepted", torch.int32, 2)
    out_offsets = _req(out_offsets, "out_offsets", torch.int32, 1)
    slot_start = _req(slot_start, "slot_start", torch.int32, 2)
    s = ids.shape[1]
    if (b < 1 or sem_labels.shape[0] != points.shape[0] or ids.shape[0] != b or planes.shape[0] != b or
            tuple(accepted.shape) != (b, s) or out_offsets.shape[0] != b + 1 or tuple(slot_start.shape) != (b, s + 1) or
            db_offsets.shape[0] != db_boxes.shape[0] + 1):
        raise ValueError("mixup_paste_points: points %s, offsets %s, sem_labels %s, ids %s, planes %s, accepted %s, out_offsets %s,"
                         " slot_start %s, db_offsets %s, db_boxes %s disagree" % tuple(tuple(t.shape) for t in (
                             points, offsets, sem_labels, ids, planes, accepted, out_offsets, slot_start, db_offsets, db_boxes)))
    if not 1 <= s <= MIXUP_MAX_ROWS or not 1 <= int(max_slots) <= MIXUP_MAX_SLOTS:
        raise ValueError("1 <= s <= %d and 1 <= max_slots <= %d, got s=%d max_slots=%d" % (MIXUP_MAX_ROWS, MIXUP_MAX_SLOTS, s,
                                                                                            max_slots))
    dev = points.device
    out = torch.empty((int(total), 4), dtype=torch.float32, device=dev)
    sem = torch.empty((int(total),), dtype=torch.int32, device=dev)
    check(lib().ssd3d_mixup_paste_points(b, s, int(max_slots), _p(points), _p(offsets), _p(sem_labels), _p(ids), _p(db_points),
                                         _p(db_offsets), _p(db_boxes), _p(db_classes), _p(planes), _p(accepted), _p(out_offsets),
                                         _p(slot_start), _p(out), _p(sem), _stream()), "mixup_paste_points")
    return out, sem


# ---- KITTI preprocessing (csrc/prepare.cu, DESIGN.md section 3.14) --------------------------------------------------
PREP_MAX_FRAMES = 4096              # frames per call
PREP_MAX_FRAME_POINTS = 262144      # raw points per frame
PREP_MAX_BATCH_POINTS = 16777216    # raw points per call
PREP_EXTENTS = (-40.0, 40.0, -5.0, 3.0, 0.0, 70.0)   # POINT_CLOUD_RANGE of 3dssd.yaml: x, y, z of the rect frame


def _prep_host(a, name, dtype):
    if isinstance(a, torch.Tensor):
        if a.device.type != "cpu":
            raise ValueError("%s must be a host array (it is checked before the launch)" % name)
        a = a.numpy()
    return np.ascontiguousarray(np.asarray(a), dtype)


def prepare_points(points, offsets, calib, image_hw, extents=PREP_EXTENTS):
    """The image-FOV and extents filters of raw velodyne frames in the rect frame (ssd3d_prepare_points): points [T, 4]
    float32 (device) packed frame after frame, offsets [b + 1] (host), calib [b, 33] float64 (device: V2C 12, R0 9, P2 12,
    row-major), image_hw [b, 2] (host, H and W > 0), extents 6 floats (host) -> (kept [T, 4] float64, kept_offsets [b + 1]
    int32) on the device: frame s's kept points (rect x, y, z, intensity) in input order at rows kept_offsets[s] ..
    kept_offsets[s+1]-1; rows from kept_offsets[b] on are not written.  Nothing synchronises the host, so the kept total
    is known on the host only after the caller reads kept_offsets."""
    points = _req(points, "points", torch.float32, 2, 4)
    calib = _req(calib, "calib", torch.float64, 2, 33)
    off = _prep_host(offsets, "offsets", np.int64).reshape(-1)
    hw = _prep_host(image_hw, "image_hw", np.int64)
    ext = _prep_host(extents, "extents", np.float64).reshape(-1)
    b = off.size - 1
    if b < 1 or b > PREP_MAX_FRAMES:
        raise ValueError("offsets must hold b + 1 entries with 1 <= b <= %d, got %d" % (PREP_MAX_FRAMES, off.size))
    n = np.diff(off)
    if off[0] != 0 or off[-1] != points.shape[0] or (n < 0).any():
        raise ValueError("offsets must rise from 0 to the point count %d, got %s .. %s" % (points.shape[0], off[0], off[-1]))
    if n.max() > PREP_MAX_FRAME_POINTS or off[-1] > PREP_MAX_BATCH_POINTS:
        raise ValueError("at most %d points per frame and %d per call, got %d and %d" % (
            PREP_MAX_FRAME_POINTS, PREP_MAX_BATCH_POINTS, n.max(), off[-1]))
    if calib.shape[0] != b or hw.shape != (b, 2):
        raise ValueError("calib %s and image_hw %s must hold %d frames" % (tuple(calib.shape), hw.shape, b))
    if (hw <= 0).any() or (hw > 2 ** 31 - 1).any():
        raise ValueError("every image size H, W must be positive, got %s" % hw[(hw <= 0).any(1)][:1].tolist())
    if ext.shape != (6,) or np.isnan(ext).any():
        raise ValueError("extents must be 6 numbers (x0, x1, y0, y1, z0, z1), got %s" % (ext.tolist(),))
    max_n = int(n.max())
    dev = points.device
    up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev, non_blocking=True)
    d_off, d_hw, d_ext = up(off.astype(np.int32)), up(hw.astype(np.int32)), up(ext)
    ws = torch.empty((int(lib().ssd3d_prepare_workspace(b, max_n)),), dtype=torch.uint8, device=dev)
    kept = torch.empty((points.shape[0], 4), dtype=torch.float64, device=dev)
    kept_off = torch.empty((b + 1,), dtype=torch.int32, device=dev)
    check(lib().ssd3d_prepare_points(b, max_n, int(off[-1]), _p(points), _p(d_off), _p(calib), _p(d_hw), _p(d_ext), _p(ws), _p(kept),
                                     _p(kept_off), _stream()), "prepare_points")
    return kept, kept_off
