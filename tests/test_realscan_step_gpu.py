"""The benchmarked step and its routes on the eight real-scan scenes of tests/test_realscan_cpu.py, on the GPU.

The scenes are regions of the reference's sample KITTI scan filled to 16 384 points with the loader's choice rule, so
they carry what synthetic scenes do not: concentric ground rings, a roughly 1/r^2 density, near-planar walls and car
sides, long empty stretches, and exact duplicates.  In S3 layer 1's D-FPS runs out of distinct points, in S7 layer 2's
F-FPS and D-FPS do too: from there every round runs at min-distance 0 and only the tie rule and the skip rules of the
pruned kernels decide the pick.

One batch of 8 like bench.py:
  * the throughput and latency-mode nets are bit-identical, and every scene equals its single-scene run;
  * every layer and the head against float64, the FPS and ball-query properties, decode and NMS
    (tests/test_bench_step_gpu.py's checks), and the CPU oracle layer by layer on S0, S3 and S7;
  * route agreement, bit for bit: every layer-1 D-FPS route, the layer-2/3 F-FPS routes on the step's own features,
    the culled ball query and its unit lists against the exhaustive scan at five layer shapes, COMPACT_GROUPS on and
    off, and the reference's kernels where oracle/_ref is built;
  * training: the Augmentor on a ragged batch of the whole scan and two short regions against its twin, and the
    teacher-forced full-size gradients on S0 and S3."""
import importlib

import numpy as np
import pytest
import torch

from oracle import augment as OA
from test_augment_gpu import check_against_twin
from test_bench_step_gpu import (Bench, assert_equal_outputs, ball_query_vs_float64, bench, decode_and_nms,  # noqa: F401
                                 every_layer_vs_float64, flatten, fps_farthest_point_property, make_net, run_step,
                                 scene_vs_oracle_layerwise)
from test_realscan_cpu import (L1_SAMPLES, NAMES, NPOINTS, camera_frame, distinct_rows, full_scan, realscan_scenes,
                               scene_sources)
from test_scene_transforms_gpu import BQ_SHAPES, L1_ROUTES, _bq_expect, _bq_gpu, _check_ref_fps, _dfps, _ffps_all, _same
from test_train_backward_gpu import full_size_gradients_teacher_forced

pytestmark = pytest.mark.gpu
A = importlib.import_module("3dssd_b200.augment")


@pytest.fixture(scope="module")
def real(bench):
    """bench.py's net and head on the eight real scenes"""
    r = Bench()
    r.__dict__.update(bench.__dict__)
    r.pts_np = realscan_scenes()[0]
    r.pts = torch.from_numpy(r.pts_np).to(bench.dev)
    return r


@pytest.fixture(scope="module")
def step(real):
    s = run_step(real.net, real.pts)
    torch.cuda.synchronize()
    return s


def _np(t):
    return t.detach().cpu().numpy()


# ---------------------------------------------------------------------------------------------------------------------
# the step: nets, scenes alone, float64, oracle
# ---------------------------------------------------------------------------------------------------------------------
def test_exhausted_scenes_reach_min_distance_zero(step):
    """The premise: S3's layer-1 samples and S7's layer-2 samples hold fewer distinct points than were drawn."""
    xyz_l, feat_l, fps_l, _ = step[0]
    s3, s7 = NAMES.index("S3"), NAMES.index("S7")
    assert distinct_rows(_np(xyz_l[1][s3])) == 1505 < L1_SAMPLES
    rows7 = np.concatenate([_np(xyz_l[1][s7]), _np(feat_l[1][s7])], 1)
    assert distinct_rows(rows7) <= 343 < 512                       # layer 2's F-FPS operand rows
    assert distinct_rows(_np(xyz_l[2][s7][:512])) <= 343 and distinct_rows(_np(xyz_l[2][s7][512:])) <= 343


def test_latency_net_and_single_scenes_are_bit_identical(pkg, real, step):
    exp = flatten(real.arch, *step)
    lat = flatten(real.arch, *run_step(make_net(pkg, real, fps_cluster=0, latency_mode=True), real.pts))
    assert_equal_outputs(lat, exp, what="latency-mode net: ")
    for s in range(len(NAMES)):
        got = flatten(real.arch, *run_step(real.net, real.pts[s:s + 1]))
        assert_equal_outputs(got, exp, rows=slice(s, s + 1), what="%s alone: " % NAMES[s])


def test_every_layer_vs_float64(pkg, real, step):
    every_layer_vs_float64(pkg, real, step)


def test_fps_farthest_point_property(step):
    fps_farthest_point_property(step)


def test_ball_query_vs_float64(real, step):
    ball_query_vs_float64(real, step)


def test_decode_and_nms(pkg, step):
    decode_and_nms(pkg, step)


@pytest.mark.parametrize("name", ["S0", "S3", "S7"])
def test_scene_vs_oracle_layerwise(oracle_ops, real, step, name):
    scene_vs_oracle_layerwise(oracle_ops, real.arch, real.params, step, NAMES.index(name))


# ---------------------------------------------------------------------------------------------------------------------
# routes, bit for bit
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def l1_oracle(oracle_ops, real):
    return oracle_ops.farthest_point_sample(L1_SAMPLES, real.pts_np[..., :3])


@pytest.mark.parametrize("route", list(L1_ROUTES))
def test_dfps_layer1_routes(pkg, cuda, real, step, l1_oracle, route):
    """bucket (the step's own), cluster 0 and 8, the latency schedule's resumed cuts, the bucket kernel resumed."""
    kw, resumed = L1_ROUTES[route]
    x = np.ascontiguousarray(real.pts_np[..., :3])
    got = _dfps(pkg, x, L1_SAMPLES, kw, resumed, cuda)
    for s, name in enumerate(NAMES):
        _same(got[s], l1_oracle[s], "%s, %s vs oracle" % (route, name))
    _same(got, _np(step[0][2][1]), route + " vs the step")
    if route == "bucket":
        _check_ref_fps(x, L1_SAMPLES, got, cuda, "real scenes")


@pytest.mark.parametrize("layer", [2, 3])
def test_ffps_routes_on_the_steps_features(oracle_ops, cuda, pkg, step, layer):
    """The pruned 4-CTA kernel (layer 2), the cluster kernel and the matrix route on the step's own operands pick the
    step's samples; the oracle agrees."""
    xyz_l, feat_l, fps_l, _ = step[0]
    if layer == 2:
        xyz, feat, m, exp = _np(xyz_l[1]), _np(feat_l[1]), 512, _np(fps_l[2][:, :512])
    else:
        xyz, feat, m, exp = _np(xyz_l[2][:, :512]), _np(feat_l[2][:, :512]), 256, _np(fps_l[3][:, :256])
    got = _ffps_all(pkg, xyz, feat, m, cuda)
    _same(got, exp, "layer %d F-FPS routes vs the step" % layer)
    _same(got, oracle_ops.farthest_point_sample_with_distance(m, oracle_ops.calc_square_dist(np.concatenate([xyz, feat], -1))),
          "layer %d F-FPS vs oracle" % layer)


def _bq_operands(real, step, shape):
    """(candidates, queries, shells, dilated, the step's own lists or None) of one layer shape on the real scenes"""
    xyz_l, _, _, dbg = step[0]
    layer = {"layer1": 1, "layer2": 2, "layer3": 3, "vote": 6}.get(shape)
    if layer is None:                       # plain query on the raw scenes, centred on D-FPS samples and beside them
        n, m, shells, dilated = BQ_SHAPES[shape]
        x = real.pts_np[..., :3].copy()
        q = _np(xyz_l[1][:, :m]).copy()
        q[:, -(m // 4):] += np.random.default_rng(7).normal(0, 0.3, (len(NAMES), m // 4, 3)).astype(np.float32)
        return x, q, shells, dilated, None
    spec = real.arch[layer - 1]
    radii, ks, dilated = list(spec[2]), list(spec[3]), spec[13]
    lows = ([0.0] + radii[:-1]) if dilated else [0.0] * len(radii)
    x, q = _np(xyz_l[spec[0][0]]), _np(xyz_l[layer])
    assert (x.shape[1], q.shape[1]) == BQ_SHAPES[shape][:2], shape
    return x, q, (lows, radii, ks), dilated, (dbg[layer - 1]["idx"], dbg[layer - 1]["cnt"])


@pytest.mark.parametrize("shape", list(BQ_SHAPES))
def test_ball_query_routes(oracle_ops, pkg, cuda, real, step, shape):
    """The culled grid and the exhaustive scan give the same lists, counts and unit lists; those equal the oracle's,
    the reference kernels' where built, and the step's own."""
    x, q, shells, dilated, own = _bq_operands(real, step, shape)
    got = _bq_gpu(pkg, shells, dilated, x, q, 1.0, cuda)
    _bq_expect(oracle_ops, shells, dilated, x, q, shape, cuda, got)
    if own is not None:
        for s in range(len(shells[2])):
            _same(_np(own[1][s]), got[1][s], "%s shell %d counts vs the step" % (shape, s))
            _same(_np(own[0][s]), got[0][s], "%s shell %d lists vs the step" % (shape, s))


def test_compact_groups_do_not_change_a_bit(pkg, real, step):
    lu = pkg.layers_util
    assert lu.COMPACT_GROUPS
    try:
        lu.COMPACT_GROUPS = False
        off = run_step(real.net, real.pts)
    finally:
        lu.COMPACT_GROUPS = True
    assert_equal_outputs(flatten(real.arch, *off), flatten(real.arch, *step), what="COMPACT_GROUPS off: ")


# ---------------------------------------------------------------------------------------------------------------------
# training on real data
# ---------------------------------------------------------------------------------------------------------------------
def _ground_boxes(pts, count, seed):
    """car boxes (x, y, z, l, h, w, ry) standing on the scan's ground: centred on in-range scan points at least 5 m
    apart, y the 95th percentile of y (down) of the points within 2 m"""
    rng = np.random.default_rng(seed)
    boxes = np.zeros((count, 7), np.float32)
    cand = pts[(np.abs(pts[:, 0]) < 30) & (pts[:, 2] > 4) & (pts[:, 2] < 60)]
    placed = 0
    for i in rng.permutation(cand.shape[0]):
        c = cand[i]
        if placed and (np.hypot(boxes[:placed, 0] - c[0], boxes[:placed, 2] - c[2]) < 5).any():
            continue
        near = pts[np.hypot(pts[:, 0] - c[0], pts[:, 2] - c[2]) < 2.0]
        boxes[placed] = (c[0], np.percentile(near[:, 1], 95), c[2], rng.uniform(3.4, 4.4), rng.uniform(1.4, 1.7),
                         rng.uniform(1.5, 1.8), rng.uniform(-np.pi, np.pi))
        placed += 1
        if placed == count:
            break
    assert placed == count
    return boxes


def test_augmentor_on_the_whole_scan_and_short_regions(cuda):
    """The whole scan (123 398 points, under the 131 072-point limit), S2 and S3 before padding, boxes on the ground:
    the kernels equal the twin bit for bit; the whole scan is thinned, the short regions padded."""
    clouds = [camera_frame(full_scan()), scene_sources()["S2"], scene_sources()["S3"]]
    sizes = [c.shape[0] for c in clouds]
    pts = np.ascontiguousarray(np.concatenate(clouds), dtype=np.float32)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    g = 16
    counts = (g, g, 8)                                               # the far region has room for fewer cars
    boxes = np.zeros((len(clouds), g, 7), np.float32)
    labels = np.zeros((len(clouds), g), np.int32)
    for s, (c, k) in enumerate(zip(clouds, counts)):
        boxes[s, :k], labels[s, :k] = _ground_boxes(c, k, 40 + s), 1
    gen = torch.Generator(device=cuda).manual_seed(21)
    d = A.draw(len(clouds), g, off[-1], NPOINTS, gen, cuda)
    d = d._replace(scene_u=torch.tensor([[0.7, 0.2, 0.3, 0.4, 0.8, 0.2], [0.1, 0.6, 0.2, 0.9, 0.3, 0.7],
                                         [0.5, 0.5, 0.5, 0.5, 0.1, 0.9]], dtype=torch.float64, device=cuda))
    got, rec = check_against_twin(cuda, pts, off, None, boxes, labels, d, NPOINTS)
    n = rec["survivors"]
    assert n[0] > NPOINTS and n[1] < NPOINTS and n[2] < NPOINTS, n
    sem = OA.sem_labels(pts[:sizes[0]], boxes[0], labels[0])
    assert (sem > 0).sum() > 100                                    # the boxes hold scan points


def test_full_size_gradients_on_real_scenes(pkg, cuda):
    pts, _ = realscan_scenes()
    full_size_gradients_teacher_forced(pkg, cuda, pts[[NAMES.index("S0"), NAMES.index("S3")]])
