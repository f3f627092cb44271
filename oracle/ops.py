"""numpy front-end of the CPU oracle (oracle/ssd3d_oracle.c).

TEST INFRASTRUCTURE ONLY -- see the header of ssd3d_oracle.c.  Function names and argument
orders follow the reference's Python operator surface
(/root/reference/lib/utils/tf_ops/{sampling/tf_sampling.py:24-62, grouping/tf_grouping.py:53-122,
interpolation/tf_interpolate.py:8-31}) with numpy arrays in place of TF tensors.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "liboracle.so")
_lib = None

_f32p = ctypes.POINTER(ctypes.c_float)
_i32p = ctypes.POINTER(ctypes.c_int)


def build(force=False):
    """Compile liboracle.so with gcc (seconds)."""
    srcs = ("ssd3d_oracle.c", "fps_pruned_model.c", "ffps_prune_model.c", "bq_grid_model.c", "Makefile")
    newest = max(os.path.getmtime(os.path.join(_HERE, f)) for f in srcs)
    if force or not os.path.exists(_LIB_PATH) or os.path.getmtime(_LIB_PATH) < newest:
        subprocess.check_call(["make", "-C", _HERE, "liboracle.so"], stdout=subprocess.DEVNULL)
    return _LIB_PATH


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = ctypes.CDLL(_LIB_PATH)
        _lib.oracle_get_threads.restype = ctypes.c_int
    return _lib


def set_threads(n):
    lib().oracle_set_threads(ctypes.c_int(int(n)))


def get_threads():
    return int(lib().oracle_get_threads())


def _f(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a, a.ctypes.data_as(_f32p)


def _i(a):
    a = np.ascontiguousarray(a, dtype=np.int32)
    return a, a.ctypes.data_as(_i32p)


def farthest_point_sample(npoint, inp):
    inp, p = _f(inp)
    b, n, c = inp.shape
    out = np.zeros((b, npoint), np.int32)
    temp = np.empty((b, n), np.float32)
    lib().oracle_farthest_point_sample(b, n, c, int(npoint), p, temp.ctypes.data_as(_f32p), out.ctypes.data_as(_i32p))
    return out


def fps_pruned_model(npoint, inp, rounds=None, temp=None, out=None, idx_offset=0, contract=True):
    """CPU model of the PRODUCT's pruned D-FPS (3dssd_b200/csrc/fps_bucket.cu, see oracle/fps_pruned_model.c): used by
    the CPU tests to check that kernel's exactness claim against farthest_point_sample above.  rounds=(j0, j1) runs a
    range of rounds with the resume state in temp [b, 2n] (distances in original order + bucket permutation), out is
    the [b, npoint] index array a resumed launch continues.  Returns (indices, stats) with stats =
    (bucket updates, rounds run per scene summed, most bucket updates in one round)."""
    inp, p = _f(inp)
    b, n, c = inp.shape
    assert c == 3
    j0, j1 = (0, int(npoint)) if rounds is None else (int(rounds[0]), int(rounds[1]))
    if out is None:
        out = np.zeros((b, npoint), np.int32)
    assert out.dtype == np.int32 and out.flags.c_contiguous and out.shape == (b, npoint)
    tp = None
    if temp is not None:
        assert temp.dtype == np.float32 and temp.flags.c_contiguous and temp.shape == (b, 2 * n)
        tp = temp.ctypes.data_as(_f32p)
    stats = np.zeros(3, np.int64)
    rc = lib().oracle_fps_pruned_model(b, n, int(npoint), p, out.ctypes.data_as(_i32p), int(npoint), int(idx_offset), j0, j1, tp,
                                       int(bool(contract)), stats.ctypes.data_as(ctypes.POINTER(ctypes.c_longlong)))
    if rc != 0:
        raise ValueError("fps_pruned_model: unsupported arguments (n <= 16384, temp needed for partial rounds)")
    return out, tuple(int(v) for v in stats)


def ffps_prune_model(npoint, x, with_margin=True):
    """CPU model of the skip rule of the PRODUCT's pruned F-FPS (ffps_bucket_kernel in 3dssd_b200/csrc/fps_bucket.cu, see
    oracle/ffps_prune_model.c) on one scene x [n, c] (n <= 4096, 3 <= c <= 68): used by the CPU tests to check that
    kernel's exactness claim.  with_margin=False drops the rounding margin of the skip test.  Returns (indices, stats)
    with stats = (points of skipped buckets whose value was below their running distance, bucket updates summed over
    rounds)."""
    x, p = _f(x)
    n, c = x.shape
    out = np.zeros(int(npoint), np.int32)
    touched = ctypes.c_longlong(0)
    fn = lib().oracle_ffps_prune_model
    fn.restype = ctypes.c_longlong
    bad = fn(n, c, int(npoint), p, int(bool(with_margin)), out.ctypes.data_as(_i32p), ctypes.byref(touched))
    if bad < 0:
        raise ValueError("ffps_prune_model: unsupported arguments (n <= 4096, 3 <= c <= 68)")
    return out, (int(bad), int(touched.value))


def farthest_point_sample_with_distance(npoint, dist):
    dist, p = _f(dist)
    b, n, n2 = dist.shape
    assert n == n2
    out = np.zeros((b, npoint), np.int32)
    temp = np.empty((b, n), np.float32)
    lib().oracle_farthest_point_sample_with_distance(b, n, int(npoint), p, temp.ctypes.data_as(_f32p),
                                                     out.ctypes.data_as(_i32p))
    return out


def gather_point(inp, idx):
    inp, p = _f(inp)
    idx, q = _i(idx)
    b, n, c = inp.shape
    m = idx.shape[1]
    out = np.empty((b, m, c), np.float32)
    lib().oracle_gather_point(b, n, m, c, p, q, out.ctypes.data_as(_f32p))
    return out


def query_ball_point(radius, nsample, xyz1, xyz2):
    xyz1, p1 = _f(xyz1)
    xyz2, p2 = _f(xyz2)
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    idx = np.zeros((b, m, nsample), np.int32)
    cnt = np.zeros((b, m), np.int32)
    lib().oracle_query_ball_point(b, n, m, ctypes.c_float(radius), int(nsample), p1, p2,
                                  idx.ctypes.data_as(_i32p), cnt.ctypes.data_as(_i32p))
    return idx, cnt


def query_ball_point_dilated(min_radius, max_radius, nsample, xyz1, xyz2):
    xyz1, p1 = _f(xyz1)
    xyz2, p2 = _f(xyz2)
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    idx = np.zeros((b, m, nsample), np.int32)
    cnt = np.zeros((b, m), np.int32)
    lib().oracle_query_ball_point_dilated(b, n, m, ctypes.c_float(min_radius), ctypes.c_float(max_radius),
                                          int(nsample), p1, p2, idx.ctypes.data_as(_i32p), cnt.ctypes.data_as(_i32p))
    return idx, cnt


def query_ball_point_grid_model(min_radius_list, max_radius_list, nsample_list, xyz1, xyz2, dilated):
    """CPU model of the PRODUCT's culled ball query (3dssd_b200/csrc/ball_query_grid.cu, see oracle/bq_grid_model.c): all
    shells of a layer in one call.  Returns (idx_list, cnt_list, units_list, stats) with units as the kernel lists them
    (int32 [1 + b*m*ceil(k/8)], [0] = count, then group << 4 | j) and stats = (queries on the dense path, candidates
    streamed by the sparse path)."""
    xyz1, p1 = _f(xyz1)
    xyz2, p2 = _f(xyz2)
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    nq = len(max_radius_list)
    lo = (ctypes.c_float * nq)(*[float(v) for v in min_radius_list])
    hi = (ctypes.c_float * nq)(*[float(v) for v in max_radius_list])
    ks = (ctypes.c_int * nq)(*[int(v) for v in nsample_list])
    idx = [np.full((b, m, int(k)), -9, np.int32) for k in nsample_list]
    cnt = [np.full((b, m), -9, np.int32) for _ in nsample_list]
    units = [np.full((1 + b * m * ((int(k) + 7) // 8),), -1, np.int32) for k in nsample_list]
    arr = lambda ts: (ctypes.c_void_p * nq)(*[t.ctypes.data for t in ts])
    stats = np.zeros(2, np.int64)
    rc = lib().oracle_bq_grid_model(b, n, m, nq, 1 if dilated else 0, lo, hi, ks, p1, p2, arr(idx), arr(cnt), arr(units),
                                    stats.ctypes.data_as(ctypes.POINTER(ctypes.c_longlong)))
    if rc != 0:
        raise ValueError("bq_grid_model: unsupported arguments (n <= 16384, 1..4 shells)")
    return idx, cnt, units, tuple(int(v) for v in stats)


def group_point(points, idx):
    points, p = _f(points)
    idx, q = _i(idx)
    b, n, c = points.shape
    _, m, ns = idx.shape
    out = np.empty((b, m, ns, c), np.float32)
    lib().oracle_group_point(b, n, c, m, ns, p, q, out.ctypes.data_as(_f32p))
    return out


def three_nn(xyz1, xyz2):
    xyz1, p1 = _f(xyz1)
    xyz2, p2 = _f(xyz2)
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    dist = np.empty((b, n, 3), np.float32)
    idx = np.empty((b, n, 3), np.int32)
    with np.errstate(over="ignore"):
        lib().oracle_three_nn(b, n, m, p1, p2, dist.ctypes.data_as(_f32p), idx.ctypes.data_as(_i32p))
    return dist, idx


def three_interpolate(points, idx, weight):
    points, p = _f(points)
    idx, q = _i(idx)
    weight, w = _f(weight)
    b, m, c = points.shape
    n = idx.shape[1]
    out = np.empty((b, n, c), np.float32)
    lib().oracle_three_interpolate(b, m, c, n, p, q, w, out.ctypes.data_as(_f32p))
    return out


def calc_square_dist(a):
    """model_util.calc_square_dist(a, a, norm=False) with the pinned fp32 summation order."""
    a, p = _f(a)
    b, n, c = a.shape
    out = np.empty((b, n, n), np.float32)
    lib().oracle_calc_square_dist(b, n, c, p, out.ctypes.data_as(_f32p))
    return out


def farthest_point_sample_features(npoint, xyz, points=None):
    """Row-by-row restatement of the product's matrix-free F-FPS (include/ssd3d.h,
    ssd3d_farthest_point_sample_features): the value used for point k in the round after `old` was picked is the
    matrix entry (sq[old] + sq[k]) - 2*dot(old, k) of calc_square_dist, evaluated on the fly -- so the result must equal
    farthest_point_sample_with_distance(npoint, calc_square_dist(concat[xyz, points])) index for index
    (lib/utils/layers_util.py:94-96 of the reference).  Pure numpy/python, small inputs only."""
    f = np.ascontiguousarray(xyz if points is None else np.concatenate([xyz, points], -1), dtype=np.float32)
    b, n, c = f.shape
    out = np.zeros((b, npoint), np.int32)
    key = (np.arange(n) % 1024).astype(np.int64) * (1 << 21) + np.arange(n) // 1024     # tie-break of the reference scan
    for s in range(b):
        fs = f[s]
        sq = np.zeros(n, np.float32)
        for l in range(c):                                   # sequential fp32 fma chain; products of fp32 are exact in f64
            sq = (sq.astype(np.float64) + fs[:, l].astype(np.float64) * fs[:, l].astype(np.float64)).astype(np.float32)
        td = np.full(n, 1e38, np.float32)
        old = 0
        for j in range(1, npoint):
            dot = np.zeros(n, np.float32)
            for l in range(c):
                dot = (dot.astype(np.float64) + np.float64(fs[old, l]) * fs[:, l].astype(np.float64)).astype(np.float32)
            d = (np.float32(sq[old]) + sq) - np.float32(2.0) * dot
            td = np.minimum(d, td)
            best = td.max()
            cand = np.flatnonzero(td == best)
            old = int(cand[np.argmin(key[cand])])
            out[s, j] = old
    return out


def linear_bn_relu(x, w, bias=None, bn=None, relu=True):
    """conv(1x1)+BN+ReLU over the last axis; bn = (gamma, beta, moving_mean, moving_var) or None."""
    x, px = _f(x)
    w, pw = _f(w)
    cin, cout = w.shape
    assert x.shape[-1] == cin
    rows = int(np.prod(x.shape[:-1]))
    y = np.empty(x.shape[:-1] + (cout,), np.float32)
    null = ctypes.cast(None, _f32p)
    keep = []

    def opt(v):
        if v is None:
            return null
        v, pv = _f(v)
        keep.append(v)
        return pv

    pb = opt(bias)
    if bn is None:
        g = be = mu = va = null
    else:
        g, be, mu, va = (opt(t) for t in bn)
    lib().oracle_linear_bn_relu(ctypes.c_long(rows), cin, cout, px, pw, pb, g, be, mu, va, int(bool(relu)),
                                y.ctypes.data_as(_f32p))
    return y


def gather_point_grad(inp_shape, idx, out_g):
    idx, q = _i(idx)
    out_g, p = _f(out_g)
    b, n, c = inp_shape
    m = idx.shape[1]
    g = np.empty((b, n, c), np.float32)
    lib().oracle_scatter_add_rows(ctypes.c_long(b * m), ctypes.c_long(m), n, c, p, q, g.ctypes.data_as(_f32p),
                                  ctypes.c_long(g.size), 0)
    return g


def group_point_grad(points_shape, idx, grad_out):
    idx, q = _i(idx)
    grad_out, p = _f(grad_out)
    b, n, c = points_shape
    _, m, ns = idx.shape
    g = np.empty((b, n, c), np.float32)
    lib().oracle_scatter_add_rows(ctypes.c_long(b * m * ns), ctypes.c_long(m * ns), n, c, p, q, g.ctypes.data_as(_f32p),
                                  ctypes.c_long(g.size), 1)
    return g


def three_interpolate_grad(points_shape, idx, weight, grad_out):
    idx, q = _i(idx)
    weight, w = _f(weight)
    grad_out, p = _f(grad_out)
    b, m, c = points_shape
    n = idx.shape[1]
    g = np.empty((b, m, c), np.float32)
    lib().oracle_three_interpolate_grad(b, n, c, m, p, q, w, g.ctypes.data_as(_f32p))
    return g


def bev_nms(boxes, scores, iou_threshold=0.1, max_output=100, cls_id=0):
    """C twin of oracle/head.py:bev_nms (the reference runs this stage on the CPU: postprocessor.py:76-88)."""
    boxes, pb = _f(boxes)
    scores, ps = _f(scores)
    b, n, _ = boxes.shape
    block = np.zeros((b, int(max_output), 9), np.float32)
    cnt = np.zeros((b,), np.int32)
    lib().oracle_bev_nms(b, n, pb, ps, ctypes.c_float(iou_threshold), int(max_output), int(cls_id),
                         block.ctypes.data_as(_f32p), cnt.ctypes.data_as(_i32p))
    return block, cnt
