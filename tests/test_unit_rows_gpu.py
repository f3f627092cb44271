"""Unit lists of 4-row units (include/ssd3d.h, ssd3d_query_ball_point_multi_ws_ex) on the GPU: the lists the ball query
builds, and every unit-list route of the grouped MLP, at 4 rows per unit against the same route at 8 rows and the dense
route -- bit for bit, since the rows a 4-row unit adds beyond cnt repeat the group's first hit."""
import importlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def N(t):
    return t.detach().cpu().numpy()


def _want(cnt, k, w):
    """(group, j) of every unit a list of w-row units holds: ceil(min(cnt, k) / w) per group"""
    cnt = cnt.reshape(-1)
    return sorted((g, j) for g in range(cnt.size) for j in range((min(int(cnt[g]), k) + w - 1) // w))


def _scene(seed, b, n, m):
    """Clustered + uniform points; the last centres have no neighbour (cnt = 0), the clusters fill whole balls"""
    rng = np.random.default_rng(seed)
    centres = rng.uniform(0, 40, (b, 10, 3))
    cl = centres[np.arange(b)[:, None], rng.integers(0, 10, (b, n // 3))] + rng.normal(0, 0.15, (b, n // 3, 3))
    xyz = np.concatenate([cl, rng.uniform(0, 40, (b, n - n // 3, 3))], 1).astype(np.float32)
    return np.ascontiguousarray(xyz[:, rng.permutation(n)]), rng


@pytest.mark.parametrize("grid", [True, False])
def test_ball_query_unit_lists_of_4_rows(pkg, cuda, grid):
    """Both list builders (the culled kernel's emission, group_units_kernel after the exhaustive kernel): every group gets
    ceil(cnt / 4) units covering rows 0 .. 4 ceil(cnt / 4) - 1, idx / cnt unchanged; 8-row shells next to 4-row ones."""
    b, n, m = 2, 4096 if grid else 1024, 500
    xyz, _ = _scene(3, b, n, m)
    tx = T(xyz, cuda)
    tn = tx[:, :m].contiguous()
    tn[:, -10:] += 500.0
    lows, highs, ks = [0.0, 0.2, 0.4], [0.2, 0.4, 0.8], [16, 32, 64]
    i8, c8, u8 = pkg.query_ball_point_multi(lows, highs, ks, tx, tn, True, grid=grid, return_units=True)
    i4, c4, u4 = pkg.query_ball_point_multi(lows, highs, ks, tx, tn, True, grid=grid, return_units=True, unit_rows=[4, 8, 4])
    for s, w in enumerate([4, 8, 4]):
        assert torch.equal(i8[s], i4[s]) and torch.equal(c8[s], c4[s])
        assert u4[s].unit_rows == w and u8[s].unit_rows == 8
        assert u4[s].numel() == 1 + b * m * (ks[s] // w)
        cnt = N(c4[s])
        for lst, ww in ((u4[s], w), (u8[s], 8)):
            u = N(lst); nu = int(u[0])
            assert sorted(zip((u[1:1 + nu] >> 4).tolist(), (u[1:1 + nu] & 15).tolist())) == _want(cnt, ks[s], ww)
        assert (cnt == 0).any() and (cnt == 1).any() and (cnt >= 9).any()
    with pytest.raises(ValueError):
        pkg.query_ball_point_multi([0.0], [0.4], [128], tx, tn, False, return_units=True, unit_rows=[4])


def _stack(P, rng, mlp, c):
    prm, scopes, cin = {}, [], c + 3
    for j, cout in enumerate(mlp):
        P._conv_init(rng, prm, "s/conv0_%d" % j, cin, cout, True)
        prm["s/conv0_%d/bn/gamma" % j][1::3] *= -1.0                     # negative-gamma columns
        scopes.append("s/conv0_%d" % j); cin = cout
    return prm, scopes


@pytest.mark.parametrize("c,k,mlp,route", [
    (1, 32, [16, 16, 32], "fused"),                  # layer 1 shapes (compile-time twins)
    (32, 64, [32, 32, 64], "fused_hoisted"),
    (64, 32, [64, 64, 128], "fused_hoisted"),        # layer 2 shapes
    (64, 64, [64, 96, 128], "fused_hoisted"),
    (7, 16, [48, 32], "fused"),                      # run-time-shape kernel
    (64, 32, [64, 96, 128], "hoisted"),              # layer 3: hoisted second conv built in the GEMM
    (64, 64, [64, 128], "hoisted"),
    (256, 32, [256, 256, 320], "expand"),            # layer 4: expand + TMA GEMMs + TMA unit pool
    (32, 16, [32, 40], "expand"),
])
def test_routes_at_4_rows_equal_8_rows_and_dense(pkg, cuda, c, k, mlp, route):
    """Every unit-list route at 4 rows per unit gives the bits of the same route at 8 and of the dense route, on groups of
    cnt = 0, 1, 4, 5, 8, 9 and full balls (the centres are planted at exact multiples of the hit counts)."""
    b, n, m = 2, 2048, 300
    xyz, rng = _scene(c + k, b, n, m)
    # centres with exactly 1, 4, 5, 8, 9 points within 0.05: lines of points far from everything else
    for i, cnt in enumerate([1, 4, 5, 8, 9]):
        base = np.array([100.0 + 10 * i, 100.0, 100.0])
        xyz[:, 20 * i: 20 * i + cnt] = base + np.arange(cnt)[:, None] * np.array([0.004, 0.0, 0.0])
    tx, tf = T(xyz, cuda), T(np.maximum(rng.standard_normal((b, n, c)), 0).astype(np.float32), cuda)
    tn = tx[:, :m].contiguous()
    tn[:, -10:] += 500.0
    (idx,), (cnt,), (u8,) = pkg.query_ball_point_multi([0.0], [0.8], [k], tx, tn, False, return_units=True)
    (_,), (_,), (u4,) = pkg.query_ball_point_multi([0.0], [0.8], [k], tx, tn, False, return_units=True, unit_rows=[4])
    cn = set(N(cnt).reshape(-1).tolist())
    assert {0, 1, 4, 5, 8, 9, k} <= cn
    P = importlib.import_module("3dssd_b200.params")
    prm, scopes = _stack(P, rng, mlp, c)
    pp = P.prepare(prm, cuda)
    zconv, wxs, n1s = pp.hoisted([scopes[0]], True, c)
    p_hi, p_lo = pkg.split_rows(tf)
    z, _ = pkg.linear_tc(p_hi, p_lo, zconv, relu=False, want_f32=True, want_split=False)
    ld = mlp[-1] + 32

    def run(units):
        out = torch.full((b, m, ld), -1.0, device=cuda)
        if units is not None:
            out[..., 16:16 + mlp[-1]] = 0.0
        last = dict(pool=k, rowmask=cnt) if units is None else dict(units=units, unit_pool=True)
        mid = {} if units is None else dict(units=units)
        if route == "fused":
            stack = pp.fused_stack(scopes, True, c + 3, limit=0)
            pkg.sa_mlp_fused(tx, tf, tn, idx, cnt, stack, out_f32=(out, 16), **mid)
        elif route == "fused_hoisted":
            stack = pp.fused_stack(scopes[1:], True, n1s[0], limit=0)
            pkg.sa_mlp_fused_hoisted(tx, z, 0, wxs[0], tn, idx, cnt, stack, out_f32=(out, 16), **mid)
        else:
            convs = [pp.conv(s, True) for s in scopes[1:]]
            if route == "expand":
                hi, lo = pkg.tf_ops.hoist_expand_split(tx, z, 0, wxs[0], tn, idx, **mid)
                op = lambda f, **kw: pkg.linear_tc(hi, lo, f, **kw)
            else:
                op = lambda f, **kw: pkg.linear_tc_hoisted(tx, z, 0, wxs[0], tn, idx, f, **kw)
            for f in convs[:-1]:
                _, (hi, lo) = op(f, want_f32=False, want_split=True, **mid)
                op = lambda f, hi=hi, lo=lo, **kw: pkg.linear_tc(hi, lo, f, **kw)
            op(convs[-1], want_split=False, out_f32=(out, 16), **last)
        return out

    dense, r8, r4 = run(None), run(u8), run(u4)
    assert torch.equal(dense, r8) and torch.equal(dense, r4)
    assert float(dense[..., 16:16 + mlp[-1]].max()) > 0


def test_whole_step_at_4_rows_equals_8_rows(pkg, cuda):
    """The benchmarked backbone (8 scenes x 16384 points) with 4-row units where nsample <= 64 gives the bits of the
    8-row plan, eager and replayed from a captured graph."""
    lu = importlib.import_module("3dssd_b200.layers_util")
    synth = importlib.import_module("3dssd_b200.synth")
    arch = pkg.config.ARCH_3DSSD
    params = pkg.params.init_params(arch, 1, seed=0)
    pts = torch.from_numpy(synth.kitti_like(8, 16384, seed=1000)).to(cuda)
    assert lu.UNIT_ROWS == 4
    outs = {}
    try:
        for w in (8, 4):
            lu.UNIT_ROWS = w
            net = pkg.SABackbone(arch, params, in_channels=1, device=cuda)
            eager = net.forward(pts)
            torch.cuda.synchronize()
            replay = net.capture(pts)
            graphed, _ = replay(pts)
            torch.cuda.synchronize()
            outs[w] = (eager, graphed)
    finally:
        lu.UNIT_ROWS = 4

    def flat(o):
        if isinstance(o, torch.Tensor):
            return [o]
        return [t for x in (o if isinstance(o, (list, tuple)) else []) for t in flat(x)]
    ref = flat(outs[8][0])
    assert len(ref) >= 8
    for other in (outs[4][0], outs[4][1], outs[8][1]):
        got = flat(other)
        assert len(got) == len(ref)
        for x, y in zip(ref, got):
            assert torch.equal(x, y)
