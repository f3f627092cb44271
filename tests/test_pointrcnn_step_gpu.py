"""PointRCNN's first stage (the RPN) at the shape tools/time_pointrcnn.py times: batches of eight 16 384-point scenes
through the net of tests/test_pointrcnn_gpu.py, eager with the debug lists.  Two batches:
  * "real":  the eight real-scan scenes S0..S7 of tests/test_realscan_cpu.py, with the exhausted S3 and S7 whose
             duplicate points put zero-distance ties into every FP layer;
  * "timed": synth.kitti_like(8, 16384) with time_pointrcnn.py's default seed.
Every FP layer meets d = 0 on both: its known points are a subset of its unknown ones.

Checked on each batch:
  * scene independence: every scene alone is the same bits as its row of the batch;
  * execution variants: the D-FPS cluster cap, the cluster kernel instead of the pruned one, and latency mode (every
    SA layer's D-FPS cut into resumable parts) give the same bits as the default net;
  * the four SA layers against float64 teacher-forced, their D-FPS and all eight ball-query scales against float64
    distances;
  * the four FP layers against float64 teacher-forced: three_nn's neighbours against float64 distances, the
    interpolation and both convs, and the fused operand against the C oracle bit for bit;
  * the head's convs against float64, the Bin-Anchor decode bit for bit, the BEV NMS against the C twin;
  * the hand-off: SABackbone.detections, which passes the head the split features that rpn_fp_layer1's last conv
    wrote, equals the head on the fp32 features, also when it is given the outputs of an older forward.
And once: three CUDA graphs of the one net replayed concurrently, a scene of 60 distinct points whose NMS block stops
short of 100, and the CPU oracle layer by layer on S0, S3, S7."""
import importlib

import numpy as np
import pytest
import torch

from test_bench_step_gpu import (assert_close, assert_equal_outputs, assert_fps, assert_scores_2ulp,
                                 ball_query_check, conv64, flatten, sa_layer64, scene_vs_oracle_layerwise)
from test_pointrcnn_cpu import decode_bin_anchor, without_aggregation
from test_pointrcnn_gpu import check_fp_operand, make_rpn
from test_pointrcnn_step_cpu import AMBIGUOUS_REL, fp_layer64, nn_ambiguous, sqdist64, three_nn64
from test_realscan_cpu import NAMES, distinct_rows, loader_choice, realscan_scenes, scene_sources

pytestmark = pytest.mark.gpu

synth = importlib.import_module("3dssd_b200.synth")
C = importlib.import_module("3dssd_b200.config")

SCENES, NPOINTS = 8, 16384
TIMED_SEED = 21                                   # tools/time_pointrcnn.py --seed
ARCH = without_aggregation(C.ARCH_POINTRCNN_RPN)  # the table as the RPN runs it: no SA layer has an aggregation conv
STAGE = C.STAGE_POINTRCNN_RPN
BATCHES = ["real", "timed"]


def batch_points(name, seed=TIMED_SEED):
    pts = realscan_scenes()[0] if name == "real" else synth.kitti_like(SCENES, NPOINTS, seed=seed)
    return np.ascontiguousarray(pts, np.float32)


def run_rpn(net, pts):
    """Eager forward with the debug lists, the detections of the hand-off (net.detections) and the head on the fp32
    features with its raw outputs."""
    out = net.forward(pts, return_debug=True)
    det = net.detections(out[0], out[1])
    head = net.head.forward(out[0], out[1], return_raw=True)
    return out, det, head


def outputs(out, det, head):
    """Every output of one RPN run by name: fps_idx, xyz, features and ball-query idx / cnt of all eight layers, raw
    cls / reg, boxes, scores, and the NMS block and count of both the hand-off and the head."""
    t = flatten(ARCH, out, head)
    t["hand-off block"], t["hand-off count"] = det
    return t


class Run:
    pass


@pytest.fixture(scope="module")
def rpn(pkg, cuda):
    return make_rpn(pkg, cuda)


@pytest.fixture(scope="module")
def runs(cuda, rpn):
    """name -> the batch's run on the RPN net (computed once)"""
    cache = {}

    def get(name):
        if name not in cache:
            r = Run()
            r.name = name
            r.net, r.params, r.hp = rpn
            r.pts_np = batch_points(name)
            r.pts = torch.from_numpy(r.pts_np).to(cuda)
            r.out, r.det, r.head = run_rpn(r.net, r.pts)
            torch.cuda.synchronize()
            cache[name] = r
        return cache[name]
    return get


# ---------------------------------------------------------------------------------------------------------------------
# bit-exact: scenes alone, execution variants
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", BATCHES)
def test_every_scene_equals_its_single_scene_run(runs, name):
    r = runs(name)
    exp = outputs(r.out, r.det, r.head)
    for s in range(SCENES):
        got = outputs(*run_rpn(r.net, r.pts[s:s + 1]))
        assert_equal_outputs(got, exp, rows=slice(s, s + 1), what="%s scene %d alone: " % (name, s))


# The default net runs fps_cluster=0 (the heuristic CTA count) with the pruned single-CTA D-FPS where it applies.
VARIANTS = {"fps_cluster=-4": dict(fps_cluster=-4), "cluster_kernel": dict(fps_bucket=False),
            "latency_mode": dict(latency_mode=True)}


@pytest.mark.parametrize("variant", list(VARIANTS))
@pytest.mark.parametrize("name", BATCHES)
def test_execution_variants_are_bit_identical(pkg, cuda, runs, name, variant):
    """The D-FPS cluster cap, the kernel choice and the latency schedule are execution details.  Latency mode cuts the
    D-FPS of SA layers 1, 2 and 3 into 4, 4 and 2 resumable launches (tests/test_pointrcnn_step_cpu.py), so a resumed
    launch that lost its running distances would pick other samples."""
    r = runs(name)
    net = pkg.SABackbone(C.ARCH_POINTRCNN_RPN, r.params, in_channels=1, device=cuda, head=r.net.head, aggregation=False,
                         **VARIANTS[variant])
    got = outputs(*run_rpn(net, r.pts))
    assert_equal_outputs(got, outputs(r.out, r.det, r.head), what="%s, %s: " % (name, variant))


# ---------------------------------------------------------------------------------------------------------------------
# float64, teacher-forced on the run's own inputs and indices
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", BATCHES)
def test_sa_layers_vs_float64(runs, name):
    """SA layers 1-4 (pointnet_sa_module_msg without aggregation) on the run's own samples and neighbour lists, every
    D-FPS as a farthest-point walk, and every ball-query scale against float64 squared distances."""
    r = runs(name)
    xyz_l, feat_l, fps_l, dbg = r.out
    d = lambda t: t.double()
    sa = [(li, spec) for li, spec in enumerate(ARCH, start=1) if spec[11] == "SA_Layer"]
    assert [li for li, _ in sa] == [1, 2, 3, 4]
    for li, spec in sa:
        xi, fi = spec[0][0], spec[1][0]
        idx, cnt = dbg[li - 1]["idx"], dbg[li - 1]["cnt"]
        nx, nf = sa_layer64(r.params, spec, d(xyz_l[xi]), d(feat_l[fi]), fps_l[li], d(xyz_l[xi]), idx, cnt)
        assert torch.equal(nx.float(), xyz_l[li]), "centres of layer %d" % li
        assert_close(feat_l[li], nf, "%s: features of layer %d" % (name, li))
        assert_fps(d(xyz_l[xi]), fps_l[li], "%s: layer-%d D-FPS" % (name, li))
        ball_query_check(xyz_l[xi], xyz_l[li], spec[2], spec[3], spec[13], idx, cnt, "%s: layer %d ball query" % (name, li))


@pytest.mark.parametrize("name", BATCHES)
def test_fp_layers_vs_float64(pkg, oracle_ops, cuda, runs, name):
    """FP layers 4..1 (pointnet_fp_module) on the run's own inputs:
      * three_nn: wherever float64 orders the four nearest known points unambiguously (nn_ambiguous), the kernel's three
        neighbours are float64's, and its squared distances are the float64 ones to float32 rounding;
      * fp_layer64 on the kernel's neighbours -- weights, interpolation, [interpolated | points1], both convs -- against
        the layer's features at FEATURE_TOL;
      * the fused operand (fp_interp_split) bit for bit against the C oracle's three_nn and the pinned weight order."""
    r = runs(name)
    xyz_l, feat_l, _, _ = r.out
    T = pkg.tf_ops
    fp = [(li, spec) for li, spec in enumerate(ARCH, start=1) if spec[11] == "FP_Layer"]
    assert [li for li, _ in fp] == [5, 6, 7, 8]
    for li, spec in fp:
        xyz1, xyz2 = xyz_l[spec[0][0]], xyz_l[spec[0][1]]
        p1, p2 = feat_l[spec[1][0]], feat_l[spec[1][1]]
        dist, idx = T.three_nn(xyz1, xyz2)
        d4, i4 = three_nn64(xyz1, xyz2)
        amb = nn_ambiguous(xyz2, d4, i4)
        assert amb.double().mean() <= 1e-3, "%s layer %d: %d of %d points ambiguous" % (name, li, int(amb.sum()), amb.numel())
        bad = ~amb & (idx.long() != i4[..., :3]).any(-1)
        if bad.any():
            s, q = [int(v) for v in bad.nonzero()[0]]
            raise AssertionError("%s layer %d three_nn: %d points off float64's neighbours, e.g. scene %d point %d: %s vs %s"
                                 % (name, li, int(bad.sum()), s, q, idx[s, q].tolist(), i4[s, q, :3].tolist()))
        d64 = sqdist64(xyz1, xyz2, idx)
        assert ((dist.double() - d64).abs() <= AMBIGUOUS_REL * d64).all(), "%s layer %d three_nn distances" % (name, li)
        assert (dist[..., 0] == 0).any(-1).all(), "%s layer %d: the known points are among the unknown ones" % (name, li)
        y64, _ = fp_layer64(r.params, spec[12], len(spec[4]), spec[5], xyz1, xyz2, p1, p2, idx=idx)
        assert_close(feat_l[li], y64, "%s: features of layer %d" % (name, li))
        check_fp_operand(pkg, oracle_ops, cuda, *(t.cpu().numpy() for t in (xyz1, xyz2, p2, p1)))
        if name == "real" and li == 8:            # the copies of S3 and S7 tie at d = 0
            assert (d4[..., 1] == 0).any()


@pytest.mark.parametrize("name", BATCHES)
def test_head_decode_and_nms(oracle_ops, runs, name):
    """pred_cls_base -> pred_cls and pred_reg_base -> pred_reg against float64 on the run's fp1 features; the numpy
    Bin-Anchor decode of the run's own raw outputs, bit for bit (scores within 2 ulp); the C twin's BEV NMS at 0.85 / 100
    on the run's boxes, bit for bit.  Every scene fills its block; in the real batch S7's 343 distinct points give
    copies of boxes at equal scores, which the NMS must suppress within its chunks of candidates."""
    r = runs(name)
    xyz_l, feat_l, _, _ = r.out
    blk, cnt, raw = r.head
    f, hp = feat_l[8].double(), r.hp
    cls = conv64(hp, "rpn_head/pred_cls", conv64(hp, "rpn_head/pred_cls_base", f, True, True), False, False)
    reg = conv64(hp, "rpn_head/pred_reg", conv64(hp, "rpn_head/pred_reg_base", f, True, True), False, False)
    assert_close(raw["cls"], cls, "%s: head cls" % name)
    assert_close(raw["reg"], reg, "%s: head reg" % name)
    eb, _ = decode_bin_anchor(xyz_l[8].cpu().numpy(), raw["reg"].cpu().numpy(), raw["cls"].cpu().numpy(),
                              STAGE["ANCHOR_SIZE"], STAGE["HALF_BIN_SEARCH_RANGE"], STAGE["BIN_CLASS_NUM"])
    boxes = raw["boxes"][:, :, 0].cpu().numpy()
    np.testing.assert_array_equal(boxes.view(np.uint32), eb.view(np.uint32))
    assert_scores_2ulp(raw["score"][..., 0], raw["cls"][..., 0])
    eblk, ecnt = oracle_ops.bev_nms(boxes, raw["score"][..., 0].cpu().numpy(), STAGE["NMS_THRESH"], STAGE["MAX_OUTPUT_NUM"])
    np.testing.assert_array_equal(cnt.cpu().numpy(), ecnt)
    np.testing.assert_array_equal(blk.cpu().numpy().view(np.uint32), eblk.view(np.uint32))
    assert (ecnt == STAGE["MAX_OUTPUT_NUM"]).all(), "%s: counts %s" % (name, ecnt.tolist())
    if name == "real":
        assert distinct_rows(boxes[NAMES.index("S7")]) <= 343


def test_nms_stops_short_on_a_scene_of_few_points(oracle_ops, cuda, rpn):
    """The other NMS outcome: 60 distinct points of S7's region, filled to 16 384 with the loader's copies, give at
    most 60 distinct boxes, so the block stops short of 100.  The NMS is the C twin's bit for bit, and the hand-off
    equals the head on the fp32 features."""
    net = rpn[0]
    src = scene_sources()["S7"][:60]
    pts = src[loader_choice(len(src), np.random.default_rng(7))][None]
    assert distinct_rows(pts[0]) == 60
    out, det, (blk, cnt, raw) = run_rpn(net, torch.from_numpy(np.ascontiguousarray(pts, np.float32)).to(cuda))
    boxes, score = raw["boxes"][:, :, 0].cpu().numpy(), raw["score"][..., 0].cpu().numpy()
    eblk, ecnt = oracle_ops.bev_nms(boxes, score, STAGE["NMS_THRESH"], STAGE["MAX_OUTPUT_NUM"])
    np.testing.assert_array_equal(cnt.cpu().numpy(), ecnt)
    np.testing.assert_array_equal(blk.cpu().numpy().view(np.uint32), eblk.view(np.uint32))
    assert 0 < ecnt[0] <= 60
    assert torch.equal(det[0], blk) and torch.equal(det[1], cnt)


# ---------------------------------------------------------------------------------------------------------------------
# the hand-off of rpn_fp_layer1's split features
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", BATCHES)
def test_handoff_equals_the_head_on_fp32_features(runs, name):
    """net.detections (the head reads the split operand rpn_fp_layer1's last conv wrote) and net.head.forward without
    split= (the head splits the fp32 features itself) give the same block and count, bit for bit."""
    r = runs(name)
    blk, cnt, _ = r.head
    assert torch.equal(r.det[0], blk) and torch.equal(r.det[1], cnt), name


@pytest.mark.parametrize("name", BATCHES)
def test_detections_of_an_older_forward(runs, name):
    """The net keeps the split features of its latest forward only for those very features: detections on the
    outputs of forward(A), asked after forward(B), are A's detections, not a mix with B's split."""
    r = runs(name)
    a, b = r.pts, r.pts.flip(0).contiguous()
    oa = r.net.forward(a)
    ob = r.net.forward(b)
    late = r.net.detections(oa[0], oa[1])
    assert torch.equal(late[0], r.det[0]) and torch.equal(late[1], r.det[1]), name
    db = r.net.detections(ob[0], ob[1])
    assert not torch.equal(db[0], late[0])                  # B's detections are another answer
    assert torch.equal(db[0], r.det[0].flip(0)) and torch.equal(db[1], r.det[1].flip(0))


# ---------------------------------------------------------------------------------------------------------------------
# concurrent CUDA graphs of one RPN net
# ---------------------------------------------------------------------------------------------------------------------
def test_concurrent_graphs_of_one_rpn_net(cuda, rpn):
    """Three graphs captured from the one RPN net, each with its own scenes (real, timed, another seed), replayed
    interleaved on three streams without synchronisation between replays: each equals an eager forward plus
    detections of its own scenes."""
    net = rpn[0]
    inputs = [torch.from_numpy(p).to(cuda) for p in (batch_points("real"), batch_points("timed"),
                                                      batch_points("timed", seed=TIMED_SEED + 1))]
    runners = [net.capture(p) for p in inputs]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(device=cuda) for _ in inputs]
    main = torch.cuda.current_stream()
    for st in streams:
        st.wait_stream(main)
    results = [None] * len(inputs)
    for rnd in range(4):
        for j in range(len(inputs)):
            k = (j + rnd) % len(inputs)                  # rotate which graph is enqueued first
            with torch.cuda.stream(streams[k]):
                results[k] = runners[k]()
    for st in streams:
        main.wait_stream(st)
    torch.cuda.synchronize()
    for k, p in enumerate(inputs):
        (xyz_l, feat_l, fps_l), (blk, cnt) = results[k]
        eager = net.forward(p)
        eblk, ecnt = net.detections(eager[0], eager[1])
        torch.cuda.synchronize()
        for li in range(1, len(ARCH) + 1):
            if eager[2][li] is not None:
                assert torch.equal(fps_l[li], eager[2][li]), "graph %d: fps_idx of layer %d" % (k, li)
            assert torch.equal(xyz_l[li], eager[0][li]), "graph %d: xyz of layer %d" % (k, li)
            assert torch.equal(feat_l[li], eager[1][li]), "graph %d: features of layer %d" % (k, li)
        assert torch.equal(blk, eblk) and torch.equal(cnt, ecnt), "graph %d: detection block" % k
    assert not torch.equal(results[1][1][0], results[2][1][0])     # the graphs saw different scenes


# ---------------------------------------------------------------------------------------------------------------------
# the CPU oracle, layer by layer
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scene", ["S0", "S3", "S7"])
def test_scene_vs_oracle_layerwise(oracle_ops, runs, scene):
    """SA and FP layers of one real scene through oracle/layers.py on the run's own inputs to each layer: D-FPS and
    ball query bit for bit, features at FEATURE_TOL."""
    r = runs("real")
    scene_vs_oracle_layerwise(oracle_ops, ARCH, r.params, (r.out, r.head), NAMES.index(scene))
