"""The C-boundary calls of every public tf_ops wrapper, pinned on the CPU.  `tf_ops.lib` is replaced by a recording
stand-in and `is_cuda` is forced on, so each wrapper runs its checks, output placement and argument packing without a
GPU or a built library.  Every call into the library is recorded as its entry point, its scalars, its pointers (the
argument or returned tensor they point into and the byte offset there, 0 for NULL, 'scratch' for anything the wrapper
allocated and did not return) and the decoded host arrays; every returned tensor as its shape, dtype, strides and the
argument it aliases.  The trace must equal tests/golden/tf_ops_abi_trace.json; SSD3D_RECORD_ABI=<file> re-records it.
Malformed operands must raise ValueError before anything reaches the library."""
import ctypes
import importlib
import json
import os

import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tf_ops_abi_trace.json")
_STREAM = object()

# host-only queries: fixed answers that depend only on their arguments
_QUERIES = {
    "ssd3d_fps_temp_elems": lambda n, c, npoint, flags: n + c + flags,
    "ssd3d_fps_needs_temp": lambda n, c: int(n > 600),
    "ssd3d_fps_supports_rounds": lambda n, c: int(c == 3),
    "ssd3d_ffps_supported": lambda n, c: int(c <= 64),
    "ssd3d_query_ball_point_workspace": lambda b, n: 0 if n > 4096 else 256 * b,
    "ssd3d_bn_train_workspace": lambda c: 8 * c,
    "ssd3d_bn_train_grad_workspace": lambda c: 16 * c,
    "ssd3d_linear_wgrad_workspace": lambda rows, cin, cout: 4 * cin * cout,
    "ssd3d_det_loss_workspace": lambda b: 64 * b,
}


def _host_arrays(name, a):
    """Host arrays of an entry point, decoded by position: {position: list of values}."""
    def arr(ctype, pos, count):
        return [] if not a[pos].value else list((ctype * count).from_address(a[pos].value))
    if name == "ssd3d_query_ball_point_multi_ws":
        nq = a[3]
        return {5: arr(ctypes.c_float, 5, nq), 6: arr(ctypes.c_float, 6, nq), 7: arr(ctypes.c_int, 7, nq),
                10: arr(ctypes.c_void_p, 10, nq), 11: arr(ctypes.c_void_p, 11, nq), 12: arr(ctypes.c_void_p, 12, nq)}
    if name == "ssd3d_sa_mlp_fused":
        return {12: arr(ctypes.c_int, 12, a[11])}
    if name == "ssd3d_sa_mlp_fused_hoisted":
        return {14: arr(ctypes.c_int, 14, a[13])}
    if name == "ssd3d_concat_rows":
        return {2: arr(ctypes.c_void_p, 2, a[1]), 3: arr(ctypes.c_int, 3, a[1])}
    return {}


_POINTER_ARRAYS = {("ssd3d_query_ball_point_multi_ws", 10), ("ssd3d_query_ball_point_multi_ws", 11),
                   ("ssd3d_query_ball_point_multi_ws", 12), ("ssd3d_concat_rows", 2)}


class _FakeLib:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*a):
            self.calls.append((name, a, _host_arrays(name, a)))
            return _QUERIES[name](*a) if name in _QUERIES else 0
        return fn


def _walk(obj, path, out):
    """(path, tensor) of every tensor reachable from obj, in a fixed order."""
    if isinstance(obj, torch.Tensor):
        out.append((path, obj))
    elif isinstance(obj, (tuple, list)):
        for i, v in enumerate(obj):
            _walk(v, "%s.%d" % (path, i), out)
    elif isinstance(obj, dict):
        for k in sorted(obj):
            _walk(obj[k], "%s.%s" % (path, k), out)
    elif hasattr(obj, "__slots__") or hasattr(obj, "__dict__"):
        names = getattr(obj, "__slots__", None) or sorted(vars(obj))
        for k in names:
            if not k.startswith("_"):
                _walk(getattr(obj, k, None), "%s.%s" % (path, k), out)
    return out


def _extent(t):
    if t.numel() == 0:
        return t.data_ptr(), t.data_ptr()
    span = sum((s - 1) * st for s, st in zip(t.shape, t.stride())) + 1
    return t.data_ptr(), t.data_ptr() + span * t.element_size()


def _where(p, known):
    if not p:
        return 0
    for path, t in known:
        lo, hi = _extent(t)
        if p == lo or lo <= p < hi:
            return [path, p - lo]
    return "scratch"


def _value(v, known):
    if v is _STREAM:
        return "stream"
    if isinstance(v, ctypes.c_void_p):
        return _where(v.value, known)
    if isinstance(v, bool) or not isinstance(v, (int, float)):
        raise AssertionError("unexpected argument %r" % (v,))
    return v


class _Recorder:
    def __init__(self, fake):
        self.fake, self.trace = fake, {}

    def __call__(self, case, fn, *args, **kw):
        start = len(self.fake.calls)
        ret = fn(*args, **kw)
        inputs = _walk(list(args), "a", []) + _walk(kw, "k", [])
        known = inputs + _walk(ret, "r", [])
        calls = []
        for name, a, arrays in self.fake.calls[start:]:
            vals = []
            for i, v in enumerate(a):
                if i in arrays:
                    ptrs = (name, i) in _POINTER_ARRAYS
                    vals.append({"host": [_where(x, known) if ptrs else x for x in arrays[i]]})
                else:
                    vals.append(_value(v, known))
            calls.append([name] + vals)
        rets = []
        for path, t in _walk(ret, "r", []):
            alias = None
            for ipath, it in inputs:
                if it.untyped_storage().data_ptr() == t.untyped_storage().data_ptr():
                    alias = [ipath, t.data_ptr() - it.data_ptr()]
                    break
            rets.append([path, list(t.shape), str(t.dtype), list(t.stride()), alias])
        self.trace.setdefault(case, []).append({"calls": calls, "returns": rets})
        return ret


@pytest.fixture()
def abi(monkeypatch):
    T = importlib.import_module("3dssd_b200.tf_ops")
    fake = _FakeLib()
    monkeypatch.setattr(T, "lib", lambda: fake)
    monkeypatch.setattr(T, "_stream", lambda: _STREAM)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    return T, fake


def _f(*s):
    return torch.zeros(s, dtype=torch.float32)


def _i(*s):
    return torch.zeros(s, dtype=torch.int32)


def _bf(*s):
    return torch.zeros(s, dtype=torch.bfloat16)


def _fold(cin, cout):
    P = importlib.import_module("3dssd_b200.params")
    g = torch.Generator().manual_seed(cin * 1000 + cout)
    return P.FoldedConv(torch.randn((cin, cout), generator=g), torch.rand((cout,), generator=g) + 0.5, torch.randn((cout,), generator=g))


def _stack(cin, nout):
    P = importlib.import_module("3dssd_b200.params")
    convs, c = [], cin
    for n in nout:
        convs.append(_fold(c, n))
        c = n
    return P.FusedStack(convs, cin)


def _grouping(b=2, n=40, c=5, m=6, ns=16):
    return _f(b, n, 3), _f(b, n, c), _f(b, m, 3), _i(b, m, ns), _i(b, m)


def _sampling(T, rec):
    big = _f(2, 50, 3)
    wide = _f(2, 30, 7)
    buf = _i(2, 24)
    rec("fps_temp_elems", T.fps_temp_elems, 1000, 3, 64, packet_kernel=True, bucket_kernel=False)
    rec("fps", T.farthest_point_sample, 8, _f(2, 30, 3))
    rec("fps_scene_strided", T.farthest_point_sample, 8, big[:, 10:40], idx_offset=5, cluster=-4, packet_kernel=True)
    rec("fps_copied", T.farthest_point_sample, 8, wide[..., :3], bucket_kernel=True)
    rec("fps_out", T.farthest_point_sample, 8, _f(2, 30, 3), out=(buf, 4), bucket_kernel=False)
    rec("fps_auto_temp", T.farthest_point_sample, 8, _f(2, 700, 3))
    temp = _f(2, 700 + 3 + 2)
    for r in ((0, 3), (3, 8)):
        rec("fps_rounds", T.farthest_point_sample, 8, _f(2, 700, 3), out=(buf, 12), rounds=r, temp=temp, bucket_kernel=False)
    rec("fps_supports_rounds", T.fps_supports_rounds, 100, 3)
    rec("fpsd", T.farthest_point_sample_with_distance, 4, _f(2, 9, 9))
    rec("fpsd_out", T.farthest_point_sample_with_distance, 4, _f(2, 9, 9), out=(buf, 2), idx_offset=3, cluster=2)
    rec("ffps_supported", T.ffps_supported, 100, 67)
    rec("ffps_xyz", T.farthest_point_sample_features, 6, _f(2, 20, 3))
    rec("ffps_points", T.farthest_point_sample_features, 6, big[:, 5:25], wide[:, 10:30, :4], out=(buf, 0), idx_offset=7)
    rec("ffps_empty_points", T.farthest_point_sample_features, 6, _f(2, 20, 3), _f(2, 20, 0))
    tf = _f(2 * 20)
    for r in ((0, 2), (2, 6)):
        rec("ffps_rounds", T.farthest_point_sample_features, 6, _f(2, 20, 3), _f(2, 20, 4), out=(buf, 18), rounds=r, temp=tf)
    rec("gather_point", T.gather_point, _f(2, 20, 4), _i(2, 5))
    rec("gather_point_column_block", T.gather_point, wide[..., 2:6], buf[:, 3:8])
    rec("gather_point_grad", T.gather_point_grad, _f(2, 20, 4), _i(2, 5), _f(2, 5, 4))
    rec("iota_idx", T.iota_idx, 2, 5, "cpu")
    rec("iota_idx_out", T.iota_idx, 2, 5, "cpu", out=(buf, 9), start=3)


def _queries(T, rec):
    x1, x2 = _f(2, 40, 3), _f(2, 6, 3)
    g1 = _f(2, 2500, 3)
    h1 = _f(1, 5000, 3)
    rec("qbp_direct", T.query_ball_point, 0.5, 8, x1, x2)
    rec("qbp_grid", T.query_ball_point, 0.5, 8, g1, x2)
    rec("qbp_dilated_direct", T.query_ball_point_dilated, 0.2, 0.5, 8, x1, x2)
    rec("qbp_dilated_grid", T.query_ball_point_dilated, 0.2, 0.5, 8, g1, x2)
    rec("qbp_dilated_no_workspace", T.query_ball_point_dilated, 0.2, 0.5, 8, h1, x2[:1])
    rec("qbp_multi", T.query_ball_point_multi, [0.0, 0.0], [0.2, 0.4], [8, 16], x1, x2, False)
    rec("qbp_multi_grid", T.query_ball_point_multi, [0.1, 0.2, 0.3], [0.2, 0.4, 0.8], [8, 16, 32], x1, x2, True, grid=True)
    rec("qbp_multi_nogrid", T.query_ball_point_multi, [0.0], [0.2], [8], g1, x2, False, grid=False)
    rec("qbp_multi_units", T.query_ball_point_multi, [0.0, 0.0], [0.2, 0.4], [16, 128], g1, x2, False, return_units=True)
    rec("qbp_multi_units_wide", T.query_ball_point_multi, [0.0, 0.0], [0.2, 0.4], [16, 256], x1, x2, False, return_units=True)
    rec("group_point", T.group_point, _f(2, 20, 4), _i(2, 5, 8))
    rec("group_point_grad", T.group_point_grad, _f(2, 20, 4), _i(2, 5, 8), _f(2, 5, 8, 4))
    rec("three_nn", T.three_nn, _f(2, 20, 3), _f(2, 7, 3))
    rec("three_interpolate", T.three_interpolate, _f(2, 7, 5), _i(2, 20, 3), _f(2, 20, 3))
    rec("three_interpolate_grad", T.three_interpolate_grad, _f(2, 7, 5), _i(2, 20, 3), _f(2, 20, 3), _f(2, 20, 5))
    rec("calc_square_dist", T.calc_square_dist, _f(2, 9, 4))


def _grouping_ops(T, rec):
    xyz, pts, nxyz, idx, cnt = _grouping()
    rec("group_concat", T.group_concat, xyz, pts, nxyz, idx)
    rec("group_concat_ldx", T.group_concat, xyz, None, nxyz, idx, ldx=8)
    rec("group_concat_split", T.group_concat_split, xyz, pts, nxyz, idx)
    rec("group_concat_split_kp", T.group_concat_split, xyz, None, nxyz, idx, kp=32)
    rec("group_concat_grad", T.group_concat_grad, _f(2, 6, 16, 8), idx, 40, 5)
    rec("group_concat_grad_some", T.group_concat_grad, _f(2, 6, 16, 8), idx, 40, 5, want_points=False, want_new_xyz=False)
    z = _f(2, 40, 48)
    wx = _f(3, 20)
    rec("hoist_expand_split", T.hoist_expand_split, xyz, z, 8, wx, nxyz, idx)
    rec("hoist_expand_split_units", T.hoist_expand_split, xyz, z, 4, wx, nxyz, idx, units=_i(1 + 2 * 6 * 2))


def _dense_mlp(T, rec):
    w, sc, sh = _f(7, 24), _f(24), _f(24)
    cnt = _i(2, 6)
    rec("linear_bn_relu", T.linear_bn_relu, _f(2, 6, 7), w, sc, sh)
    rec("linear_bn_relu_cin", T.linear_bn_relu, _f(2, 6, 16, 8), w, sc, sh, relu=False, cin=7)
    rec("linear_bn_relu_pool", T.linear_bn_relu, _f(2, 6, 16, 7), w, sc, sh, pool=16, rowmask=cnt)
    rec("linear_bn_relu_pool_odd", T.linear_bn_relu, _f(2, 6, 3, 7), w, sc, sh, pool=3, rowmask=cnt)
    rec("linear_bn_relu_pool_odd_nomask", T.linear_bn_relu, _f(2, 6, 3, 7), w, sc, sh, pool=3)
    rec("rowgroup_max", T.rowgroup_max, _f(2, 6, 16, 24), 16)
    rec("rowgroup_max_mask", T.rowgroup_max, _f(2, 6, 16, 24), 16, cnt)
    rec("rowgroup_max_grad", T.rowgroup_max_grad, _f(2, 6, 16, 24), _f(2, 6, 24), 16)
    rec("rowgroup_max_grad_mask", T.rowgroup_max_grad, _f(2, 6, 16, 24), _f(2, 6, 24), 16, cnt)
    rec("split_rows", T.split_rows, _f(2, 6, 7))
    rec("split_rows_kp", T.split_rows, _f(2, 6, 7)[:, :, :5], kp=32)


def _tc(T, rec):
    f = _fold(20, 24)
    hi, lo = _bf(2, 6, 16, 32), _bf(2, 6, 16, 32)
    cnt = _i(2, 6)
    rec("linear_tc", T.linear_tc, hi, lo, f)
    rec("linear_tc_split", T.linear_tc, hi, lo, f, relu=False, want_f32=False, want_split=True)
    rec("linear_tc_both", T.linear_tc, hi, lo, f, want_f32=True, want_split=True)
    for k in T.TC_POOL_WIDTHS:
        h, l = _bf(2, 3, k, 32), _bf(2, 3, k, 32)
        rec("linear_tc_pool_%d" % k, T.linear_tc, h, l, f, pool=k, rowmask=_i(2, 3), want_f32=True, want_split=True)
    cat, ch, cl = _f(2, 6, 64), _bf(2, 6, 64), _bf(2, 6, 64)
    rec("linear_tc_out", T.linear_tc, hi, lo, f, pool=16, rowmask=cnt, out_f32=(cat, 8), out_split=(ch, cl, 16))
    rec("linear_tc_out_f32_want_split", T.linear_tc, hi, lo, f, pool=16, out_f32=(cat, 40), want_split=True)
    units = _i(1 + 2 * 6 * 2)
    rec("linear_tc_units", T.linear_tc, hi, lo, f, want_f32=False, want_split=True, units=units)
    rec("linear_tc_unit_pool", T.linear_tc, hi, lo, f, want_split=False, out_f32=(cat, 16), units=units, unit_pool=True)
    xyz, pts, nxyz, idx, _ = _grouping(c=17)
    fg = _fold(20, 32)
    rec("linear_tc_gather", T.linear_tc_gather, xyz, pts, nxyz, idx, fg)
    rec("linear_tc_gather_pool", T.linear_tc_gather, xyz, pts, nxyz, idx, fg, pool=16, rowmask=cnt, want_f32=True,
        want_split=False)
    rec("linear_tc_gather_out", T.linear_tc_gather, xyz, pts, nxyz, idx, fg, pool=16, rowmask=cnt, out_f32=(cat, 32),
        out_split=(ch, cl, 0))
    rec("linear_tc_gather_xyz_only", T.linear_tc_gather, xyz, None, nxyz, idx, _fold(3, 16), relu=False)
    z, wx = _f(2, 40, 48), _f(3, 20)
    f2 = _fold(20, 24)
    rec("linear_tc_hoisted", T.linear_tc_hoisted, xyz, z, 8, wx, nxyz, idx, f2)
    rec("linear_tc_hoisted_pool", T.linear_tc_hoisted, xyz, z, 28, wx, nxyz, idx, f2, pool=16, rowmask=cnt, want_f32=True,
        want_split=True)
    rec("linear_tc_hoisted_out", T.linear_tc_hoisted, xyz, z, 0, wx, nxyz, idx, f2, pool=16, rowmask=cnt, out_f32=(cat, 8),
        out_split=(ch, cl, 24))
    rec("linear_tc_hoisted_units", T.linear_tc_hoisted, xyz, z, 8, wx, nxyz, idx, f2, units=units)
    rec("linear_tc_hoisted_unit_pool", T.linear_tc_hoisted, xyz, z, 8, wx, nxyz, idx, f2, want_split=False,
        out_f32=(cat, 40), units=units, unit_pool=True)


def _fused(T, rec):
    xyz, pts, nxyz, idx, cnt = _grouping(c=13)
    st = _stack(16, [16, 24, 40])
    cat, ch, cl = _f(2, 6, 64), _bf(2, 6, 64), _bf(2, 6, 64)
    units = _i(1 + 2 * 6 * 2)
    rec("sa_mlp_fused", T.sa_mlp_fused, xyz, pts, nxyz, idx, cnt, st)
    rec("sa_mlp_fused_no_cnt", T.sa_mlp_fused, xyz, pts, nxyz, idx, None, st)
    rec("sa_mlp_fused_out", T.sa_mlp_fused, xyz, pts, nxyz, idx, cnt, st, out_f32=(cat, 8), out_split=(ch, cl, 16))
    rec("sa_mlp_fused_split_only", T.sa_mlp_fused, xyz, pts, nxyz, idx, cnt, st, out_split=(ch, cl, 24))
    rec("sa_mlp_fused_units", T.sa_mlp_fused, xyz, pts, nxyz, idx, cnt, st, out_f32=(cat, 16), units=units)
    rec("sa_mlp_fused_xyz_only", T.sa_mlp_fused, xyz, None, nxyz, idx, cnt, _stack(3, [16, 32]))
    z, wx = _f(2, 40, 48), _f(3, 24)
    hs = _stack(24, [32, 40])
    rec("sa_mlp_fused_hoisted", T.sa_mlp_fused_hoisted, xyz, z, 16, wx, nxyz, idx, cnt, hs)
    rec("sa_mlp_fused_hoisted_out", T.sa_mlp_fused_hoisted, xyz, z, 0, wx, nxyz, idx, cnt, hs, out_f32=(cat, 24),
        out_split=(ch, cl, 8))
    rec("sa_mlp_fused_hoisted_units", T.sa_mlp_fused_hoisted, xyz, z, 8, wx, nxyz, idx, cnt, hs, out_f32=(cat, 0), units=units)


def _misc(T, rec):
    blk, bc = _f(2, 5, 9), _i(2)
    rec("bev_nms", T.bev_nms, _f(2, 30, 7), _f(2, 30), 0.1, 5)
    rec("bev_nms_out", T.bev_nms, _f(2, 30, 7), _f(2, 30), 0.1, 5, cls_id=2, out=(blk, bc))
    rec("fill_zero", T.fill_zero, _f(2, 6, 64))
    rec("peer_allgather", T.peer_allgather, torch.zeros(64, dtype=torch.uint8), torch.zeros(2, dtype=torch.int64), 2, 1,
        64, (4096, 8192), (128, 256), _i(3), torch.zeros(128, dtype=torch.uint8))
    rec("split_points", T.split_points, _f(2, 20, 4))
    rec("split_points_xyz", T.split_points, _f(2, 20, 3))
    big, wide = _f(2, 50, 3), _f(2, 30, 7)
    rec("concat_cols", T.concat_cols, big[:, 10:40], wide[:, :, 3:])
    rec("vote_translate", T.vote_translate, _f(2, 20, 3), _f(2, 20, 6), (-3.0, -2.0, -1.5))
    rec("vote_translate_grad", T.vote_translate_grad, _f(2, 20, 6), _f(2, 20, 3), (-3.0, -2.0, -1.5))
    rec("decode", T.decode_dist_anchor_free, _f(2, 20, 3), _f(2, 20, 30), _f(2, 20, 1))
    rec("concat_rows_one", T.concat_rows, [_f(2, 5, 4)])
    rec("concat_rows", T.concat_rows, [_f(2, 5, 4), _f(2, 3, 4), _f(2, 7, 4)])


def _training(T, rec):
    x, g, bt = _f(2, 6, 24), _f(24), _f(24)
    mm, mv = _f(24), _f(24)
    rec("bn_train", T.bn_train, x, g, bt)
    rec("bn_train_moving", T.bn_train, x, g, bt, mm, mv, decay=0.8, relu=False)
    rec("bn_train_grad", T.bn_train_grad, x, _f(2, 6, 24), _f(24), _f(24), _f(24), _f(24), g, relu=False)
    rec("linear_wgrad", T.linear_wgrad, _f(2, 6, 7), _f(2, 6, 24))
    rec("linear_wgrad_nobias", T.linear_wgrad, _f(2, 6, 7), _f(2, 6, 24), want_bias=False)
    f = _fold(7, 24)
    rec("linear_bn_train", T.linear_bn_train, _f(2, 6, 7), f, g, bt, mm, mv)
    rec("linear_bn_train_nobn", T.linear_bn_train, _f(2, 6, 7), f, bn=False, relu=True)

    def conv_fb(x, w, b, gamma, beta, go, bn):
        y = T.conv_train(x, w, b, gamma, beta, mm, mv, bn=bn)
        return (y,) + torch.autograd.grad(y, [x, w, b] + ([gamma, beta] if bn else []), go)

    leaf = lambda *s: _f(*s).requires_grad_()
    rec("conv_train", conv_fb, leaf(2, 6, 7), leaf(7, 24), leaf(24), leaf(24), leaf(24), _f(2, 6, 24), True)
    rec("conv_train_nobn", conv_fb, leaf(2, 6, 7), leaf(7, 24), leaf(24), leaf(24), leaf(24), _f(2, 6, 24), False)

    def group_max_fb(y, rowmask, go):
        out = T.group_max_train(y, 16, rowmask)
        return out, torch.autograd.grad(out, [y], go)[0]

    rec("group_max_train", group_max_fb, leaf(2, 6, 16, 24), _i(2, 6), _f(2, 6, 24))

    def group_concat_fb(xyz, points, new_xyz, idx, go):
        out = T.group_concat_train(xyz, points, new_xyz, idx)
        return (out,) + torch.autograd.grad(out, [xyz, points, new_xyz], go)

    rec("group_concat_train", group_concat_fb, leaf(2, 40, 3), leaf(2, 40, 5), leaf(2, 6, 3), _i(2, 6, 16), _f(2, 6, 16, 8))

    def vote_fb(xyz, offsets, go):
        out = T.vote_translate_train(xyz, offsets, (-3.0, -2.0, -1.5))
        return (out,) + torch.autograd.grad(out, [xyz, offsets], go)

    rec("vote_translate_train", vote_fb, leaf(2, 20, 3), leaf(2, 20, 3), _f(2, 20, 3))

    def gather_fb(inp, idx, go):
        out = T.gather_point(inp, idx)
        return out, torch.autograd.grad(out, [inp], go)[0]

    rec("gather_point_train", gather_fb, leaf(2, 20, 4), _i(2, 5), _f(2, 5, 4))

    def group_point_fb(points, idx, go):
        out = T.group_point(points, idx)
        return out, torch.autograd.grad(out, [points], go)[0]

    rec("group_point_train", group_point_fb, leaf(2, 20, 4), _i(2, 5, 8), _f(2, 5, 8, 4))

    def interp_fb(points, idx, weight, go):
        out = T.three_interpolate(points, idx, weight)
        return out, torch.autograd.grad(out, [points], go)[0]

    rec("three_interpolate_train", interp_fb, leaf(2, 7, 5), _i(2, 20, 3), _f(2, 20, 3), _f(2, 20, 5))


def _det(T, rec):
    b, n, nv, g = 2, 12, 10, 4
    base, vb = _f(b, n, 3), _f(b, nv, 3)
    tg = rec("det_assign", T.det_assign, base, vb, _f(b, g, 7), _i(b, g))
    cls = _f(b, n, 1, 1)
    reg = _f(b, n, 1, 30)
    off, acls, ares = reg[..., :6], reg[..., 6:18], reg[..., 18:]
    vo = _f(b, nv, 8)[..., 2:5]
    rec("det_loss", T.det_loss, base, cls, off, acls, ares, vo, tg)
    rec("det_loss_contiguous", T.det_loss, base, _f(b, n, 1), _f(b, n, 6), _f(b, n, 12), _f(b, n, 12), _f(b, nv, 3), tg)
    rec("det_loss_grad", T.det_loss_grad, base, cls, off, acls, ares, vo, tg, _f(6), _f(3))

    def det_fb(base, reg, cls, vo, go):
        loss = T.det_loss_train(base, cls, reg[..., :6], reg[..., 6:18], reg[..., 18:], vo, tg)
        return (loss,) + torch.autograd.grad(loss, [base, reg, cls, vo], go)

    leaf = lambda *s: _f(*s).requires_grad_()
    rec("det_loss_train", det_fb, leaf(b, n, 3), leaf(b, n, 1, 30), leaf(b, n, 1, 1), leaf(b, nv, 3), _f(6))


def test_abi_trace_matches_recording(abi):
    T, fake = abi
    rec = _Recorder(fake)
    for part in (_sampling, _queries, _grouping_ops, _dense_mlp, _tc, _fused, _misc, _training, _det):
        part(T, rec)
    got = json.loads(json.dumps(rec.trace))
    path = os.environ.get("SSD3D_RECORD_ABI")
    if path:
        with open(path, "w") as fh:
            json.dump(got, fh, indent=0, sort_keys=True)
        return
    with open(GOLDEN) as fh:
        exp = json.load(fh)
    assert sorted(got) == sorted(exp)
    for case in sorted(exp):
        assert got[case] == exp[case], case


# ---- malformed operands: rejected before anything reaches the library ------------------------------------------------

def _bad_grouping_cases(T):
    xyz, pts, nxyz, idx, cnt = _grouping(c=13)
    st = _stack(16, [16, 32])
    f = _fold(16, 32)
    z, wx = _f(2, 40, 48), _f(3, 16)
    hst = _stack(16, [32])
    f2 = _fold(16, 32)
    wrappers = {
        "group_concat": lambda x, p, q, i, c: T.group_concat(x, p, q, i),
        "group_concat_split": lambda x, p, q, i, c: T.group_concat_split(x, p, q, i),
        "linear_tc_gather": lambda x, p, q, i, c: T.linear_tc_gather(x, p, q, i, f),
        "linear_tc_hoisted": lambda x, p, q, i, c: T.linear_tc_hoisted(x, z, 0, wx, q, i, f2),
        "hoist_expand_split": lambda x, p, q, i, c: T.hoist_expand_split(x, z, 0, wx, q, i),
        "sa_mlp_fused": lambda x, p, q, i, c: T.sa_mlp_fused(x, p, q, i, c, st),
        "sa_mlp_fused_hoisted": lambda x, p, q, i, c: T.sa_mlp_fused_hoisted(x, z, 0, wx, q, i, c, hst),
    }
    bad = {
        "new_xyz_rows": (xyz, pts, _f(2, 8, 3), _i(2, 16, 16), _i(2, 16)),
        "new_xyz_batch": (xyz, pts, _f(3, 6, 3), idx, cnt),
        "idx_batch": (xyz, pts, nxyz, _i(3, 6, 16), cnt),
        "idx_rows": (xyz, pts, nxyz, _i(2, 5, 16), cnt),
        "points_rows": (xyz, _f(2, 39, 13), nxyz, idx, cnt),
        "points_batch": (xyz, _f(1, 40, 13), nxyz, idx, cnt),
    }
    for wname, w in wrappers.items():
        for bname, args in bad.items():
            if "hoist" in wname and bname.startswith("points"):
                continue                               # the hoisted wrappers take the table z, not points
            yield "%s-%s" % (wname, bname), w, args
    for wname in ("sa_mlp_fused", "sa_mlp_fused_hoisted"):
        for bname, c in (("cnt_int64", cnt.long()), ("cnt_shape", _i(2, 5)), ("cnt_float", cnt.float())):
            yield "%s-%s" % (wname, bname), wrappers[wname], (xyz, pts, nxyz, idx, c)


def _bad_output_cases(T):
    f = _fold(20, 24)
    hi, lo = _bf(2, 6, 16, 32), _bf(2, 6, 16, 32)
    xyz, pts, nxyz, idx, cnt = _grouping(c=17)
    fg = _fold(20, 24)
    z, wx = _f(2, 40, 48), _f(3, 20)
    st = _stack(20, [16, 24])
    hst = _stack(20, [24])
    ops = {
        "linear_tc": lambda **kw: T.linear_tc(hi, lo, f, pool=16, **kw),
        "linear_tc_gather": lambda **kw: T.linear_tc_gather(xyz, pts, nxyz, idx, fg, pool=16, **kw),
        "linear_tc_hoisted": lambda **kw: T.linear_tc_hoisted(xyz, z, 0, wx, nxyz, idx, f, pool=16, **kw),
        "sa_mlp_fused": lambda **kw: T.sa_mlp_fused(xyz, pts, nxyz, idx, cnt, st, **kw),
        "sa_mlp_fused_hoisted": lambda **kw: T.sa_mlp_fused_hoisted(xyz, z, 0, wx, nxyz, idx, cnt, hst, **kw),
    }
    ch, cl = _bf(2, 6, 64), _bf(2, 6, 64)
    bad = {
        "f32_past_row": dict(out_f32=(_f(2, 6, 64), 60)),
        "f32_negative_col": dict(out_f32=(_f(2, 6, 64), -8)),
        "f32_dtype": dict(out_f32=(torch.zeros((2, 6, 64), dtype=torch.float64), 0)),
        "f32_rows": dict(out_f32=(_f(2, 5, 64), 0)),
        "f32_flat": dict(out_f32=(_f(12, 64), 0)),
        "f32_strided_rows": dict(out_f32=(_f(2, 6, 128)[..., :64], 0)),
        "split_past_row": dict(out_split=(ch, cl, 48)),
        "split_dtype": dict(out_split=(_f(2, 6, 64), _f(2, 6, 64), 0)),
        "split_lo_shape": dict(out_split=(ch, _bf(2, 6, 48), 0)),
        "split_rows": dict(out_split=(_bf(2, 7, 64), _bf(2, 7, 64), 0)),
        "split_strided_rows": dict(out_split=(_bf(2, 6, 128)[..., 64:], _bf(2, 6, 128)[..., 64:], 0)),
    }
    for oname, op in ops.items():
        for bname, kw in bad.items():
            yield "%s-%s" % (oname, bname), op, kw


def _bad_rowmask_cases(T):
    f = _fold(20, 24)
    hi, lo = _bf(2, 6, 16, 32), _bf(2, 6, 16, 32)
    xyz, pts, nxyz, idx, cnt = _grouping(c=17)
    z, wx = _f(2, 40, 48), _f(3, 20)
    w = _f(7, 24)
    ops = {
        "linear_tc": lambda m: T.linear_tc(hi, lo, f, pool=16, rowmask=m),
        "linear_tc_gather": lambda m: T.linear_tc_gather(xyz, pts, nxyz, idx, _fold(20, 24), pool=16, rowmask=m),
        "linear_tc_hoisted": lambda m: T.linear_tc_hoisted(xyz, z, 0, wx, nxyz, idx, f, pool=16, rowmask=m),
        "linear_bn_relu": lambda m: T.linear_bn_relu(_f(2, 6, 16, 7), w, _f(24), _f(24), pool=16, rowmask=m),
        "linear_bn_relu_odd_pool": lambda m: T.linear_bn_relu(_f(2, 6, 3, 7), w, _f(24), _f(24), pool=3, rowmask=m),
        "rowgroup_max": lambda m: T.rowgroup_max(_f(2, 6, 16, 24), 16, m),
    }
    for oname, op in ops.items():
        for bname, m in (("int64", cnt.long()), ("float", cnt.float()), ("size", _i(2, 5))):
            yield "%s-%s" % (oname, bname), op, m


def _cases(kind):
    T = importlib.import_module("3dssd_b200.tf_ops")
    return list({"grouping": _bad_grouping_cases, "output": _bad_output_cases, "rowmask": _bad_rowmask_cases}[kind](T))


@pytest.mark.parametrize("kind", ["grouping", "output", "rowmask"])
def test_malformed_operands_raise_before_any_launch(abi, kind):
    T, fake = abi
    failures = []
    for case in _cases(kind):
        name, op, arg = case
        fake.calls.clear()
        try:
            if kind == "grouping":
                op(*arg)
            elif kind == "output":
                op(**arg)
            else:
                op(arg)
        except ValueError:
            if fake.calls:
                failures.append("%s: raised after calling %s" % (name, [c[0] for c in fake.calls]))
            continue
        failures.append("%s: accepted" % name)
    assert not failures, "\n".join(failures)
