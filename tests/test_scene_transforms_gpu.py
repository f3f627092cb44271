"""The pruned D-FPS, pruned F-FPS, culled ball query and the whole benchmarked step on scaled, translated and stretched
scenes, on the GPU.

The maps and their exact ranges are tests/test_scene_transforms_cpu.py's.  Under 2^k scaling (radii scaled too) and
translation on the 2^-4 grid the reference's arithmetic is unchanged, so indices, neighbour lists, counts and unit
lists must not change by a bit -- only the kernels' skip and cull decisions may.  The untransformed runs are checked
once against the CPU oracle, the recorded reference outputs (tests/golden) scaled by 2^k must come out unchanged, and
the scenes with no exact relation (float translations by 1e2..1e5 m, one stray return 1e3..1e6 m away, flat, collinear,
tied widest extents) must equal the oracle -- and the reference's own kernels where oracle/_ref is built."""
import importlib
import os

import numpy as np
import pytest
import torch

from oracle import ref_ops
from test_bench_step_gpu import SCENES, bench, flatten, make_net, run_step, scene_vs_oracle_layerwise  # noqa: F401
from test_ffps_bucket_gpu import _scene as ffps_scene
from test_fps_instantiations_gpu import CASES, _device_input, _fps_kw, _keeps
from test_scene_transforms_cpu import (EXACT_IDS, FLOAT_IDS, LAYER1_SHELLS, PLAIN_SHELLS, apply_map, base_scene, dyadic,
                                       exact_map, float_map, scale2, scale2_in_range, shift, stretch)

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
layers_util = importlib.import_module("3dssd_b200.layers_util")


def _dev(x, cuda):
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(cuda)


def _same(got, exp, what):
    got, exp = np.asarray(got), np.asarray(exp)
    assert got.shape == exp.shape and np.array_equal(got, exp), \
        "%s: first difference at %s" % (what, np.argwhere(got != exp)[:1].tolist() if got.shape == exp.shape else "shape")


# ---------------------------------------------------------------------------------------------------------------------
# D-FPS: every route of the layer-1 shape, and the c = 3 instantiations of the launch plan
# ---------------------------------------------------------------------------------------------------------------------
L1_N, L1_M = 16384, 4096
LATENCY_PARTS = (0.34, 0.28, 0.22, 0.16)       # SABackbone's default fps_parts: the latency schedule's resumed cuts
L1_ROUTES = {"bucket": (dict(cluster=-4), False),                        # automatic plan at 16384 -> 4096: pruned kernel
             "cluster0": (dict(cluster=0, bucket_kernel=False), False),
             "cluster8": (dict(cluster=8, bucket_kernel=False), False),
             "latency": (dict(cluster=0, bucket_kernel=False), True),     # the latency-mode net's resumable launches
             "bucket-resumed": (dict(bucket_kernel=True), True)}


def _dfps(pkg, x, m, kw, resumed, cuda):
    inp = _dev(x, cuda)
    if not resumed:
        return pkg.farthest_point_sample(m, inp, **kw).cpu().numpy()
    b, n, _ = x.shape
    out = torch.full((b, m), -7, dtype=torch.int32, device=cuda)
    temp = torch.empty((b, pkg.tf_ops.fps_temp_elems(n, 3, m, bucket_kernel=kw.get("bucket_kernel"))), device=cuda)
    for j0, j1 in layers_util._part_bounds(m, LATENCY_PARTS):
        pkg.farthest_point_sample(m, inp, out=(out, 0), rounds=(j0, j1), temp=temp, **kw)
    return out.cpu().numpy()


class _Lazy(dict):
    """key -> value computed on first use"""
    def __init__(self, fn):
        super().__init__()
        self.fn = fn

    def __missing__(self, key):
        v = self[key] = self.fn(key)
        return v


@pytest.fixture(scope="module")
def l1_oracle(oracle_ops):
    """scene key -> (scene, oracle indices): 'kitti' / 'dyadic' bases and every float map of the kitti base"""
    def make(key):
        x = base_scene(key, 2, L1_N, 1000) if key in ("kitti", "dyadic") else float_map(key)[1](base_scene("kitti", 2, L1_N, 1000))
        return x, oracle_ops.farthest_point_sample(L1_M, x)
    return _Lazy(make)


def _check_ref_fps(x, m, got, cuda, what):
    if ref_ops.available():
        _same(got, ref_ops.farthest_point_sample(m, _dev(x, cuda)).cpu().numpy(), what + " vs the reference kernel")


@pytest.mark.parametrize("route", list(L1_ROUTES))
def test_dfps_layer1_routes(pkg, cuda, l1_oracle, route):
    kw, resumed = L1_ROUTES[route]
    base = {}
    for kind in ("kitti", "dyadic"):
        x, exp = l1_oracle[kind]
        base[kind] = _dfps(pkg, x, L1_M, kw, resumed, cuda)
        _same(base[kind], exp, "%s, untransformed %s scene vs oracle" % (route, kind))
    for name in EXACT_IDS:
        _, kind, fn, _ = exact_map(name)
        _same(_dfps(pkg, fn(l1_oracle[kind][0]), L1_M, kw, resumed, cuda), base[kind], "%s, %s" % (route, name))
    for name in FLOAT_IDS:
        x, exp = l1_oracle[name]
        got = _dfps(pkg, x, L1_M, kw, resumed, cuda)
        _same(got, exp, "%s, %s vs oracle" % (route, name))
        if route == "bucket":
            _check_ref_fps(x, L1_M, got, cuda, name)


INST = [c for c in CASES if c.family == "fps" and c.c == 3]
INST_EXACT = ["scale-16", "scale+16", "scale-56", "translate-diag"]
INST_FLOAT = ["shift-1e5", "stretch-1e6", "tied"]


@pytest.mark.parametrize("case", INST, ids=[c.id for c in INST])
def test_dfps_instantiations_under_maps(pkg, oracle_ops, cuda, case):
    """The smallest- and largest-n key of every D-FPS outcome of the plan table, at the key's cluster request, flags and
    alignment: 2^+-16 and 2^-56 scaling and a far dyadic translation leave the indices alone; a 1e5 m float translation,
    a stray 1e6 m out and tied widest extents give the oracle's."""
    n = case.n
    m = min(n, 256) if _keeps(case, min(n, 256)) else case.key_m
    kw = _fps_kw(case)
    run = lambda x: pkg.farthest_point_sample(m, _device_input(torch, case, x, False, cuda), **kw).cpu().numpy()
    base = {}
    for kind in ("kitti", "dyadic"):
        x = base_scene(kind, 2, n, 77 + n)
        base[kind] = run(x)
        _same(base[kind], oracle_ops.farthest_point_sample(m, x), "untransformed %s scene" % kind)
    for name in INST_EXACT:
        _, kind, fn, _ = exact_map(name)
        _same(run(fn(base_scene(kind, 2, n, 77 + n))), base[kind], name)
    for name in INST_FLOAT if n >= 2 else INST_FLOAT[:2]:           # tied extents need two points
        x = float_map(name)[1](base_scene("kitti", 2, n, 77 + n))
        _same(run(x), oracle_ops.farthest_point_sample(m, x), name)


@pytest.mark.parametrize("k", [-16, -5, 9, 16])
def test_dfps_golden_scaled(pkg, cuda, k):
    """The reference's recorded D-FPS of two KITTI-like scenes (4096 -> 512), scaled by 2^k: the pruned kernel (forced)
    and the automatic route still give the recorded indices."""
    z = np.load(os.path.join(HERE, "golden", "fps_kitti_2x4096_m512.npz"))
    x = scale2(z["inp"], k)
    for kw in (dict(bucket_kernel=True), dict()):
        _same(pkg.farthest_point_sample(int(z["npoint"]), _dev(x, cuda), **kw).cpu().numpy(), z["out"], "2^%d %s" % (k, kw))


# ---------------------------------------------------------------------------------------------------------------------
# F-FPS: the pruned 4-CTA kernel, the cluster kernel and the matrix route
# ---------------------------------------------------------------------------------------------------------------------
def _ffps_all(pkg, xyz, feat, m, cuda):
    """indices of every F-FPS route at this shape, after checking that they agree"""
    tx, tf = _dev(xyz, cuda), _dev(feat, cuda)
    got = {"cluster": pkg.tf_ops.farthest_point_sample_features(m, tx, tf).cpu().numpy()}
    if 2048 < xyz.shape[1] <= 4096:
        got["bucket"] = pkg.tf_ops.farthest_point_sample_features(m, tx, tf, cluster=-4).cpu().numpy()
    d = pkg.calc_square_dist(torch.cat([tx, tf], -1))
    got["matrix"] = pkg.farthest_point_sample_with_distance(m, d).cpu().numpy()
    for r, v in got.items():
        _same(v, got["cluster"], "route %s vs cluster" % r)
    return got["cluster"]


def _ffps_operands(layer, kind):
    """layer 2: 4096 points with 64 features -> 512; layer 3: 512 points with 128 features -> 256"""
    if layer == 2:
        xyz, feat = ffps_scene("plain" if kind == "xyz-shift" else kind, 2, 4096, 31)
        m = 512
    else:
        xyz, feat = ffps_scene("plain" if kind == "xyz-shift" else kind, 2, 512, 32)
        feat = np.concatenate([feat, np.float32(0.5) * feat[..., ::-1]], -1)
        m = 256
    if kind == "xyz-shift":                      # the scene 1e4 m out: squared norms 3e8, the skip margin is what holds
        xyz = shift(xyz, [7071.07, 0.0, 7071.07])
    return xyz, feat, m


@pytest.mark.parametrize("layer", [2, 3])
@pytest.mark.parametrize("kind", ["plain", "offset", "xyz-shift"])
def test_ffps_routes_agree_and_scale(pkg, oracle_ops, cuda, layer, kind):
    xyz, feat, m = _ffps_operands(layer, kind)
    base = _ffps_all(pkg, xyz, feat, m, cuda)
    both = np.concatenate([xyz, feat], -1)
    _same(base, oracle_ops.farthest_point_sample_with_distance(m, oracle_ops.calc_square_dist(both)), "untransformed vs oracle")
    for k in (-12, -4, 3, 12):
        y = scale2(both, k, values=True)            # xyz and features together: both enter the norms and dot products
        _same(_ffps_all(pkg, y[..., :3], y[..., 3:], m, cuda), base, "2^%d" % k)


# ---------------------------------------------------------------------------------------------------------------------
# ball query: culled grid, exhaustive scan, unit lists
# ---------------------------------------------------------------------------------------------------------------------
BQ_SHAPES = {"layer1": (16384, 4096, LAYER1_SHELLS, True),
             "layer2": (4096, 1024, ([0.0, 0.4, 0.8], [0.4, 0.8, 1.6], [32, 32, 64]), True),
             "layer3": (1024, 512, ([0.0, 1.6, 3.2], [1.6, 3.2, 4.8], [32, 32, 32]), True),
             "plain16384": (16384, 1024, PLAIN_SHELLS, False),
             "vote": (512, 256, ([0.0, 0.0], [4.8, 6.4], [16, 32]), False)}


def _bq_scene(kind, n, m, seed):
    """candidates and queries: a subset of the candidates, the last quarter moved off the points (vote-like centres)"""
    pts = base_scene(kind, 2, n, seed)
    rng = np.random.default_rng(seed)
    q = np.stack([pts[s, rng.choice(n, m, replace=False)] for s in range(2)])
    q[:, -(m // 4):] += rng.normal(0, 0.3, (2, m // 4, 3)).astype(np.float32)
    return pts, (dyadic(q) if kind == "dyadic" else q.astype(np.float32))


def _units(u):
    u = u.cpu().numpy()
    return sorted(u[1:1 + int(u[0])].tolist())


def _bq_gpu(pkg, shells, dilated, x, q, f, cuda):
    """(lists, counts, unit multisets) of the grid kernel, after checking that the exhaustive scan gives the same"""
    lows, highs, ks = [r * f for r in shells[0]], [r * f for r in shells[1]], shells[2]
    tx, tq = _dev(x, cuda), _dev(q, cuda)
    res = {}
    for grid in (True, False):
        idx, cnt, units = pkg.tf_ops.query_ball_point_multi(lows, highs, ks, tx, tq, dilated, grid=grid, return_units=True)
        res[grid] = ([i.cpu().numpy() for i in idx], [c.cpu().numpy() for c in cnt], [_units(u) for u in units])
    for s in range(len(ks)):
        _same(res[False][1][s], res[True][1][s], "shell %d counts, exhaustive vs grid" % s)
        _same(res[False][0][s], res[True][0][s], "shell %d lists, exhaustive vs grid" % s)
        assert res[False][2][s] == res[True][2][s], "shell %d unit lists, exhaustive vs grid" % s
    return res[True]


def _bq_expect(oracle_ops, shells, dilated, x, q, what, cuda, got):
    lows, highs, ks = shells
    for s, (lo, hi, k) in enumerate(zip(lows, highs, ks)):
        ei, ec = (oracle_ops.query_ball_point_dilated(lo, hi, k, x, q) if dilated else oracle_ops.query_ball_point(hi, k, x, q))
        mask = (ec > 0)[..., None]
        _same(got[1][s], ec, "%s shell %d counts vs oracle" % (what, s))
        _same(got[0][s] * mask, ei * mask, "%s shell %d lists vs oracle" % (what, s))
        want = sorted((g << 4) | j for g, c in enumerate(ec.reshape(-1)) for j in range((int(c) + 7) // 8))
        assert got[2][s] == want, "%s shell %d unit list" % (what, s)
        if ref_ops.available():
            tx, tq = _dev(x, cuda), _dev(q, cuda)
            ri, rc = (ref_ops.query_ball_point_dilated(lo, hi, k, tx, tq) if dilated else ref_ops.query_ball_point(hi, k, tx, tq))
            _same(got[1][s], rc.cpu().numpy(), "%s shell %d counts vs the reference kernel" % (what, s))
            _same(got[0][s] * mask, ri.cpu().numpy() * mask, "%s shell %d lists vs the reference kernel" % (what, s))


@pytest.mark.parametrize("shape", list(BQ_SHAPES))
def test_ball_query_under_maps(pkg, oracle_ops, cuda, shape):
    n, m, shells, dilated = BQ_SHAPES[shape]
    base = {}
    for kind in ("kitti", "dyadic"):
        x, q = _bq_scene(kind, n, m, 5 + n)
        base[kind] = _bq_gpu(pkg, shells, dilated, x, q, 1.0, cuda)
        _bq_expect(oracle_ops, shells, dilated, x, q, "untransformed " + kind, cuda, base[kind])
    for name in EXACT_IDS:
        _, kind, fn, f = exact_map(name)
        x, q = _bq_scene(kind, n, m, 5 + n)
        if name.startswith("scale"):
            assert scale2_in_range(x, int(np.log2(f)), also=(q,), radii=shells[1])[0]
        x, q = apply_map(fn, x, q)
        got = _bq_gpu(pkg, shells, dilated, x, q, f, cuda)
        for s in range(len(shells[2])):
            _same(got[1][s], base[kind][1][s], "%s shell %d counts" % (name, s))
            _same(got[0][s], base[kind][0][s], "%s shell %d lists" % (name, s))
            assert got[2][s] == base[kind][2][s], "%s shell %d unit list" % (name, s)
    for name in FLOAT_IDS:
        x, q = apply_map(float_map(name)[1], *_bq_scene("kitti", n, m, 5 + n))
        _bq_expect(oracle_ops, shells, dilated, x, q, name, cuda, _bq_gpu(pkg, shells, dilated, x, q, 1.0, cuda))


BQ_GOLDEN = ["bq_kitti_r0.4_k16", "bq_kitti_r1.6_k32", "bqd_kitti_0_0.4_k32", "bqd_kitti_0.4_0.8_k32", "bqd_kitti_0.8_1.6_k64"]


@pytest.mark.parametrize("name", BQ_GOLDEN)
def test_ball_query_golden_scaled(pkg, cuda, name):
    """The reference's recorded neighbour lists, with points, queries and radii scaled by 2^k: grid and exhaustive scan
    still give the recorded lists and counts."""
    z = np.load(os.path.join(HERE, "golden", name + ".npz"))
    dilated = "min_radius" in z.files
    lo = float(z["min_radius"]) if dilated else 0.0
    hi = float(z["max_radius"]) if dilated else float(z["radius"])
    mask = (z["cnt"] > 0)[..., None]
    for k in (-16, -5, 7, 16):
        x, q = scale2(z["xyz1"], k, also=(z["xyz2"],), radii=(lo, hi)), scale2(z["xyz2"], k, also=(z["xyz1"],))
        lo_k, hi_k = float(np.ldexp(np.float32(lo), k)), float(np.ldexp(np.float32(hi), k))
        for grid in (True, False):
            idx, cnt = pkg.tf_ops.query_ball_point_multi([lo_k], [hi_k], [int(z["nsample"])], _dev(x, cuda), _dev(q, cuda),
                                                          dilated, grid=grid)
            _same(cnt[0].cpu().numpy(), z["cnt"], "2^%d grid=%s counts" % (k, grid))
            _same(idx[0].cpu().numpy() * mask, z["idx"] * mask, "2^%d grid=%s lists" % (k, grid))


# ---------------------------------------------------------------------------------------------------------------------
# the whole step: scene 0 transformed, scenes 1-7 clean
# ---------------------------------------------------------------------------------------------------------------------
STEP_MAPS = {"scale-3": lambda x: scale2(x, -3), "shift-1e5": float_map("shift-1e5")[1],
             "stretch-1e4": lambda x: stretch(x, 1e4), "stretch-1e6": lambda x: stretch(x, 1e6), "flat": float_map("flat")[1]}
NETS = {"throughput": {}, "latency": dict(fps_cluster=0, latency_mode=True)}


@pytest.fixture(scope="module")
def step_nets(pkg, bench):
    """the bench net and the latency-mode net, with their clean batch-8 outputs"""
    out = {}
    for name, over in NETS.items():
        net = make_net(pkg, bench, **over) if over else bench.net
        out[name] = (net, flatten(bench.arch, *run_step(net, bench.pts)))
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("name", list(STEP_MAPS))
def test_step_with_one_transformed_scene(oracle_ops, bench, step_nets, name):
    """Scenes 1-7 keep every bit of every layer and of the head whatever scene 0 holds (a stray point 1e6 m out
    included), in the throughput and the latency-mode net; scene 0 equals the oracle layer by layer."""
    pts = bench.pts_np.copy()
    pts[0:1, :, :3] = STEP_MAPS[name](pts[0:1, :, :3])
    dev_pts = torch.from_numpy(pts).to(bench.dev)
    steps = {}
    for net_name, (net, clean) in step_nets.items():
        steps[net_name] = run_step(net, dev_pts)
        got = flatten(bench.arch, *steps[net_name])
        assert got.keys() == clean.keys()
        for key in clean:
            assert torch.equal(got[key][1:], clean[key][1:]), "%s net, %s: %s of scenes 1-%d changed" % (
                net_name, name, key, SCENES - 1)
    a, b = (flatten(bench.arch, *steps[k]) for k in NETS)
    for key in a:
        assert torch.equal(a[key][:1], b[key][:1]), "%s: %s of scene 0 differs between the nets" % (name, key)
    scene_vs_oracle_layerwise(oracle_ops, bench.arch, bench.params, steps["throughput"], 0)
