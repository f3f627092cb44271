"""PointRCNN's second stage on the GPU (DESIGN.md section 3.16): query_boxes_3d_points against the reference's own
kernel (queryBoxes3dPointsLauncher of tf_grouping_g.cu, recorded in tests/golden/roi_pool_ref.npz), the fused region pool
against the scan and the numpy / float64 restatements of tests/test_pointrcnn_rcnn_cpu.py, the stage-2 decode, the
counted NMS, and the whole two-stage forward at B = 8 with its graph replay.

The reference outputs are replayed from the fixture; SSD3D_RECORD_ROI=<path> runs the live reference kernel
(oracle/_ref/libref_ops.so) instead and writes the fixture there."""
import ctypes
import hashlib
import importlib
import os

import numpy as np
import pytest
import torch

from test_bench_step_gpu import FEATURE_TOL, assert_close, assert_fps, conv64, rel_err, sa_layer64
from test_pointrcnn_rcnn_cpu import canonical_np, decode_rows_np, expand, info_conv64, scan_np
from test_realscan_cpu import realscan_scenes

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "roi_pool_ref.npz")
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libref_ops.so")
synth = importlib.import_module("3dssd_b200.synth")
C = importlib.import_module("3dssd_b200.config")
B = 8


class RefQuery:
    """queryBoxes3dPointsLauncher's (idx, pts_cnt), keyed by the bytes of the inputs: replayed from the fixture, or run
    live and recorded when SSD3D_RECORD_ROI is set."""

    def __init__(self):
        self.record = os.environ.get("SSD3D_RECORD_ROI")
        self.data = {} if self.record else dict(np.load(GOLDEN))

    @staticmethod
    def key(nsample, xyz, boxes):
        h = hashlib.sha1(repr(int(nsample)).encode())
        for a in (xyz, boxes):
            h.update(str(a.shape).encode())
            h.update(np.ascontiguousarray(a, np.float32).tobytes())
        return h.hexdigest()[:20]

    def __call__(self, nsample, xyz, boxes):
        k = self.key(nsample, xyz, boxes)
        if not self.record:
            if k + "_idx" not in self.data:
                raise KeyError("no recorded reference output for these inputs: record %s again" % GOLDEN)
            return self.data[k + "_idx"].astype(np.int32), self.data[k + "_cnt"].astype(np.int32)
        lib = ctypes.CDLL(REF_LIB)
        b, n, _ = xyz.shape
        m = boxes.shape[1]
        x = torch.from_numpy(np.ascontiguousarray(xyz, np.float32)).cuda()
        p = torch.from_numpy(np.ascontiguousarray(boxes, np.float32)).cuda()
        idx = torch.zeros((b, m, nsample), dtype=torch.int32, device="cuda")     # rows without a hit stay 0
        cnt = torch.zeros((b, m), dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        lib._Z26queryBoxes3dPointsLauncheriiiiPKfS0_PiS1_(b, n, m, int(nsample), ctypes.c_void_p(x.data_ptr()),
                                                          ctypes.c_void_p(p.data_ptr()), ctypes.c_void_p(idx.data_ptr()),
                                                          ctypes.c_void_p(cnt.data_ptr()))
        torch.cuda.synchronize()
        self.data[k + "_idx"] = idx.cpu().numpy().astype(np.int16)
        self.data[k + "_cnt"] = cnt.cpu().numpy().astype(np.int16)
        return idx.cpu().numpy(), cnt.cpu().numpy()

    def save(self):
        if self.record:
            np.savez_compressed(self.record, **self.data)


@pytest.fixture(scope="module")
def ref_query(cuda):
    r = RefQuery()
    yield r
    r.save()


def proposals_around(xyz, m, rng, big=0):
    """Boxes centred on scene points (clusters of hits), rotated, some overlapping, `big` of them large enough to hold
    more than 512 points, plus two far away (empty)."""
    pick = xyz[rng.choice(len(xyz), m, replace=False)]
    bx = np.zeros((m, 7), np.float32)
    bx[:, 0], bx[:, 2] = pick[:, 0], pick[:, 2]
    bx[:, 1] = pick[:, 1] + rng.uniform(0.2, 1.5, m)
    bx[:, 3] = rng.uniform(2.0, 5.0, m)
    bx[:, 4] = rng.uniform(1.0, 2.5, m)
    bx[:, 5] = rng.uniform(1.0, 2.5, m)
    bx[:, 6] = rng.uniform(-np.pi, np.pi, m)
    bx[m // 2:m // 2 + 4] = bx[m // 2]                       # identical / overlapping boxes
    bx[m // 2 + 1:m // 2 + 4, 6] += np.float32([0.5, np.pi / 2, np.pi])
    if big:
        bx[:big, 3:6] = [30.0, 10.0, 30.0]
    bx[-2:, 0] = 500.0
    bx[[0, -3], 6] = [np.pi / 2, 0.0]
    return bx


def scenes():
    """(name, xyz [b, n, 3] float32): synthetic KITTI-like scenes and real-scan scenes."""
    syn = synth.kitti_like(2, 16384, seed=31)[..., :3]
    real = realscan_scenes()[0][[0, 3]][..., :3]
    return {"synthetic": np.ascontiguousarray(syn, np.float32), "realscan": np.ascontiguousarray(real, np.float32)}


CLUSTER_BOX = np.array([0, 0, 0, 2.0, 1.5, 2.0, 0.3], np.float32)   # placed on a cluster: its points >= 0.55 m off a face


def edge_scene(n, rng, clusters):
    """A scene of n points spread over x in [-30, 30], z in [0, 60], with point clusters far outside that region:
    clusters is a list of index arrays, cluster j's points lie within 0.3 m of (50 + 10 j, -0.6, 80) horizontally and
    0.4 m vertically.  Returns the xyz [n, 3] and one bottom-centred box per cluster (CLUSTER_BOX at the cluster's
    foot) that holds exactly that cluster's points, also after the pool's expansion by 1 m."""
    xyz = np.stack([rng.uniform(-30, 30, n), rng.uniform(-2.5, 1.0, n), rng.uniform(0, 60, n)], -1).astype(np.float32)
    boxes = []
    for j, members in enumerate(clusters):
        c = np.array([50 + 10 * j, -0.6, 80], np.float32)
        k = len(members)
        xyz[members] = c + np.stack([rng.uniform(-0.3, 0.3, k), rng.uniform(-0.4, 0.4, k), rng.uniform(-0.3, 0.3, k)], -1)
        boxes.append(CLUSTER_BOX + np.array([c[0], 0, c[2], 0, 0, 0, 0], np.float32))
    return xyz, boxes


def random_boxes(xyz, m, rng):
    """m boxes on random scene points (with replacement), one holding every point, one far from all of them."""
    pick = xyz[rng.integers(0, len(xyz), m)]
    bx = np.zeros((m, 7), np.float32)
    bx[:, 0], bx[:, 2] = pick[:, 0], pick[:, 2]
    bx[:, 1] = pick[:, 1] + rng.uniform(0.2, 1.5, m)
    bx[:, 3:6] = rng.uniform(1.0, 6.0, (m, 3))
    bx[:, 6] = rng.uniform(-np.pi, np.pi, m)
    bx[0] = [10, 2, 40, 200, 10, 200, 0.1]
    bx[1] = [500, 0, 500, 2, 2, 2, 0]
    return bx


# kernel edges: name -> (n, nsample).  "n*": scenes whose last warp is partial (n = 1 and 33 are nearly nothing else),
# with a cluster in that warp; "ns*": nsample around a warp and at its limit, with clusters of nsample - 1, nsample and
# nsample + 1 points scattered through the scene's index order.
EDGES = {"n1": (1, 512), "n33": (33, 512), "n1000": (1000, 512), "n16383": (16383, 512), "ns1": (8192, 1),
         "ns31": (8192, 31), "ns32": (8192, 32), "ns33": (8192, 33), "ns1024": (8192, 1024)}


def edge_case(name, m=24):
    """(xyz [2, n, 3], boxes [2, m, 7], nsample, designed) for an EDGES shape: two scenes (another batch offset each),
    the cluster boxes first, then random_boxes.  designed: (scene, row, the cluster's indices) of every cluster box."""
    n, ns = EDGES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    xyz, boxes, designed = [], [], []
    for s in range(2):
        if name.startswith("n") and not name.startswith("ns"):
            tail = np.arange(32 * ((n - 1) // 32), n)                 # the last warp, partial for every n here
            clusters = [tail]
        else:
            perm = rng.permutation(n)
            sizes = [max(ns - 1, 0), ns, ns + 1]
            cuts = np.cumsum([0] + sizes)
            clusters = [np.sort(perm[cuts[j]:cuts[j + 1]]) for j in range(3)]
        x, cb = edge_scene(n, rng, clusters)
        xyz.append(x)
        boxes.append(np.concatenate([np.stack(cb), random_boxes(x, m - len(cb), rng)]))
        designed += [(s, r, c) for r, c in enumerate(clusters)]
    return np.stack(xyz), np.stack(boxes), ns, designed


def query_case(name):
    """(xyz, boxes, nsample, designed) of test_query_boxes_vs_reference_kernel's case"""
    if name in EDGES:
        return edge_case(name)
    xyz = scenes()[name]
    rng = np.random.default_rng(7)
    return xyz, np.stack([proposals_around(x, 100, rng, big=3) for x in xyz]), 512, []


def assert_designed_hits(idx, cnt, ns, designed, what):
    """Each cluster box lists its cluster's first ns points in index order, padded with the first one."""
    for s, r, members in designed:
        k = min(len(members), ns)
        assert cnt[s, r] == k, "%s: cluster box %d of scene %d holds %d points, expected %d" % (what, r, s, cnt[s, r], k)
        exp = np.full(ns, members[0] if k else 0, np.int32)
        exp[:k] = members[:k]
        np.testing.assert_array_equal(idx[s, r], exp, err_msg="%s: cluster box %d of scene %d" % (what, r, s))


@pytest.mark.parametrize("name", ["synthetic", "realscan"] + list(EDGES))
def test_query_boxes_vs_reference_kernel(pkg, cuda, ref_query, name):
    xyz, boxes, ns, designed = query_case(name)
    idx, cnt = pkg.tf_ops.query_boxes_3d_points(ns, torch.from_numpy(xyz).to(cuda), torch.from_numpy(boxes).to(cuda))
    idx, cnt = idx.cpu().numpy(), cnt.cpu().numpy()
    ridx, rcnt = ref_query(ns, xyz, boxes)
    assert np.array_equal(cnt, rcnt)
    assert np.array_equal(idx, ridx)
    c = rcnt.ravel()
    if name in EDGES:
        assert_designed_hits(idx, cnt, ns, designed, name)
        assert (cnt[:, len(designed) // 2] == min(xyz.shape[1], ns)).all() and not cnt[:, len(designed) // 2 + 1].any()
    else:
        assert (c == 512).sum() >= 3 and (c == 0).sum() >= 2 and ((c > 0) & (c < 512)).sum() > 50
    # the numpy restatement agrees wherever no point lies within a few ulp of a face
    rows = range(0, boxes.shape[1], 1 if name in EDGES else 7)
    compared = 0
    for s in range(len(xyz)):
        for r in rows:
            i, n, amb = scan_np(xyz[s], boxes[s, r], ns)
            if amb == 0:
                compared += 1
                assert n == rcnt[s, r] and np.array_equal(i, ridx[s, r]), "scene %d box %d" % (s, r)
    assert compared >= len(xyz) * len(rows) // 2


def pool_inputs(pkg, cuda, xyz, rng, count):
    b, n, _ = xyz.shape
    feat = rng.standard_normal((b, n, 128)).astype(np.float32)
    score = rng.uniform(0, 1, (b, n)).astype(np.float32)
    score[:, :8] = 0.5                                       # the threshold itself: mask 1
    block = np.zeros((b, 100, 9), np.float32)
    for s in range(b):
        block[s, :count[s], :7] = proposals_around(xyz[s], 100, rng, big=2)[:count[s]]
    params = pkg.params.init_rcnn_params(128, seed=3)
    return feat, score, block, params


@pytest.mark.parametrize("name", ["synthetic", "realscan"])
def test_region_pool(pkg, cuda, ref_query, name):
    T = pkg.tf_ops
    xyz = scenes()[name]
    rng = np.random.default_rng(11)
    count = np.array([100, 63], np.int32)
    feat, score, block, params = pool_inputs(pkg, cuda, xyz, rng, count)
    pp = pkg.params.prepare(params, cuda)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    oxyz, ofeat, idx, cnt = T.region_pool(t(xyz), t(feat), t(score), t(block), t(count), pp.conv("roi_pool/conv0", True))
    oxyz, ofeat, idx, cnt = (v.cpu().numpy() for v in (oxyz, ofeat, idx, cnt))
    exp_boxes = np.stack([np.stack([expand(block[s, r]) for r in range(100)]) for s in range(2)])
    ridx, rcnt = ref_query(512, xyz, exp_boxes)
    for s in range(2):
        v = count[s]
        assert np.array_equal(cnt[s, :v], rcnt[s, :v]) and np.array_equal(idx[s, :v], ridx[s, :v])
        assert not cnt[s, v:].any() and not idx[s, v:].any()                    # padding pools nothing
    oxyz, ofeat = oxyz.reshape(2, 100, 512, 3), ofeat.reshape(2, 100, 512, 256)
    for s in range(2):
        for r in list(range(0, 100, 9)) + [count[1] - 1, count[1]]:
            k = idx[s, r]
            can = canonical_np(xyz[s, k], block[s, r])
            np.testing.assert_allclose(oxyz[s, r], can, rtol=0, atol=4 * np.spacing(np.float32(np.abs(can).max() + 1)))
            p = xyz[s, k].astype(np.float64)
            info = np.concatenate([oxyz[s, r].astype(np.float64), (score[s, k] >= 0.5)[:, None],
                                   np.sqrt((p * p).sum(-1))[:, None]], -1)
            assert_close(torch.from_numpy(ofeat[s, r, :, :128]), torch.from_numpy(info_conv64(info, params)), "info conv")
            assert np.array_equal(ofeat[s, r, :, 128:], feat[s, k])
    assert np.array_equal(cnt > 0, (rcnt > 0) & (np.arange(100)[None] < count[:, None]))


def info_params(co, rng):
    """A random roi_pool/conv0 (5 -> co, with BN) under its variable names."""
    sc = "roi_pool/conv0/"
    return {sc + "weights": rng.standard_normal((5, co)).astype(np.float32), sc + "biases": rng.standard_normal(co).astype(np.float32) * 0.1,
            sc + "bn/gamma": rng.uniform(0.5, 1.5, co).astype(np.float32), sc + "bn/beta": rng.standard_normal(co).astype(np.float32) * 0.1,
            sc + "bn/moving_mean": rng.standard_normal(co).astype(np.float32) * 0.1,
            sc + "bn/moving_variance": rng.uniform(0.5, 2.0, co).astype(np.float32)}


# pool edges: name -> (query shape of EDGES, c_info, c_feat, width of a block row, count given).  c_feat = 0 passes null
# features; "nmax" is the largest scene the pool takes at nsample 512 and c_info 128 (tests/test_pointrcnn_rcnn_cpu.py
# checks that one point more is rejected).
POOL_EDGES = {"n1": ("n1", 128, 128, 9, True), "n33": ("n33", 4, 4, 7, False), "n1000": ("n1000", 256, 0, 12, True),
              "n16383": ("n16383", 128, 4, 9, True), "ns1": ("ns1", 4, 0, 9, True), "ns31": ("ns31", 128, 4, 7, True),
              "ns32": ("ns32", 256, 4, 12, False), "ns33": ("ns33", 128, 128, 9, True),
              "ns1024": ("ns1024", 256, 128, 9, True), "nmax": (None, 128, 128, 9, True)}
POOL_MAX_N = 17706


@pytest.mark.parametrize("name", list(POOL_EDGES))
def test_region_pool_kernel_edges(pkg, cuda, ref_query, name):
    """The fused pool at the kernel's edges, every row: the indices and counts against the reference kernel on the
    expanded boxes (and the designed cluster hits), padding rows empty, the canonical xyz in float32, the info conv in
    float64 with the mask of score >= 0.5 (exact 0.5 scores on cluster points), and the copied features bit for bit."""
    from test_bench_step_gpu import conv64
    shape, co, cf, ld, with_count = POOL_EDGES[name]
    if shape is None:
        rng = np.random.default_rng(5)
        xyz, cb = edge_scene(POOL_MAX_N, rng, [np.arange(POOL_MAX_N - 40, POOL_MAX_N, 3)])
        xyz = np.stack([xyz, xyz[::-1]])
        boxes = np.stack([np.concatenate([cb, random_boxes(xyz[s], 23, rng)]) for s in range(2)])
        ns, designed = 512, []
    else:
        xyz, boxes, ns, designed = edge_case(shape)
        rng = np.random.default_rng(len(name))
    b, n, _ = xyz.shape
    m = boxes.shape[1]
    count = np.array([m, m - 5], np.int32)
    valid = np.arange(m)[None] < count[:, None] if with_count else np.ones((b, m), bool)
    block = np.zeros((b, m, ld), np.float32)
    block[..., :7] = boxes
    block[..., 7:] = rng.standard_normal((b, m, ld - 7))                   # the NMS block's extra columns are not read
    block[~valid, :7] = rng.uniform(-5, 5, (int((~valid).sum()), 7))       # padding rows are not scanned either
    feat = rng.standard_normal((b, n, cf)).astype(np.float32)
    score = rng.uniform(0, 1, (b, n)).astype(np.float32)
    score[:, ::3] = 0.5                                                     # the threshold itself: mask 1
    score[:, 1::3] = np.nextafter(np.float32(0.5), np.float32(0))          # one ulp below: mask 0
    params = info_params(co, rng)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    f = t(feat) if cf else torch.empty((b, n, 0), device=cuda)
    assert cf or f.data_ptr() == 0                                          # null features
    oxyz, ofeat, idx, cnt = pkg.tf_ops.region_pool(t(xyz), f, t(score), t(block), t(count) if with_count else None,
                                                   pkg.params.prepare(params, cuda).conv("roi_pool/conv0", True), nsample=ns)
    torch.cuda.synchronize()
    assert tuple(oxyz.shape) == (b * m, ns, 3) and tuple(ofeat.shape) == (b * m, ns, co + cf)
    idx_np, cnt_np = idx.cpu().numpy(), cnt.cpu().numpy()
    exp_boxes = np.stack([np.stack([expand(block[s, r]) for r in range(m)]) for s in range(b)])
    ridx, rcnt = ref_query(ns, xyz, exp_boxes)
    assert np.array_equal(cnt_np[valid], rcnt[valid]) and np.array_equal(idx_np[valid], ridx[valid])
    assert not cnt_np[~valid].any() and not idx_np[~valid].any()           # padding pools nothing
    assert_designed_hits(idx_np, cnt_np, ns, designed, name)
    if name == "nmax":
        assert (cnt_np[:, 0] == 14).all() and (cnt_np[:, 1] == 512).all()
    for s in range(b):
        for r in np.flatnonzero(valid[s]):
            i, c, amb = scan_np(xyz[s], exp_boxes[s, r], ns)
            if amb == 0:
                assert c == cnt_np[s, r] and np.array_equal(i, idx_np[s, r]), "scene %d box %d" % (s, r)
    # every row: canonical xyz, [info conv | features]
    oxyz_np = oxyz.cpu().numpy().reshape(b, m, ns, 3)
    for s in range(b):
        for r in range(m):
            can = canonical_np(xyz[s, idx_np[s, r]], block[s, r])
            np.testing.assert_allclose(oxyz_np[s, r], can, rtol=0, atol=4 * np.spacing(np.float32(np.abs(can).max() + 1)))
    k = idx.view(b, m * ns).long()
    gx = torch.gather(t(xyz).double(), 1, k[..., None].expand(-1, -1, 3))
    gs = torch.gather(t(score), 1, k)
    info = torch.cat([oxyz.view(b, m * ns, 3).double(), (gs >= 0.5).double()[..., None], gx.norm(dim=-1, keepdim=True)], -1)
    assert (gs == 0.5).any() and ((gs < 0.5).any() or n < 2)
    assert_close(ofeat.view(b, m * ns, -1)[..., :co], conv64(params, "roi_pool/conv0", info, True, True), "%s: info conv" % name)
    if cf:
        assert torch.equal(ofeat.view(b, m * ns, -1)[..., co:], torch.gather(f, 1, k[..., None].expand(-1, -1, cf)))


def test_decode_rows_and_counted_nms(pkg, cuda):
    T = pkg.tf_ops
    rng = np.random.default_rng(5)
    b, n = 3, 100
    anchors = np.zeros((b, n, 9), np.float32)
    anchors[..., 0] = rng.uniform(-30, 30, (b, n)); anchors[..., 2] = rng.uniform(0, 60, (b, n))
    anchors[..., 1] = rng.uniform(0, 2, (b, n)); anchors[..., 3:6] = rng.uniform(1, 4, (b, n, 3))
    anchors[..., 6] = rng.uniform(-3, 3, (b, n))
    reg = rng.standard_normal((b, n, 52)).astype(np.float32)
    reg[:, ::5, 0:2] = 2.5                                     # argmax ties
    reg[:, ::7, 25] = -9.0                                     # clamped size
    cls = rng.standard_normal((b, n, 2)).astype(np.float32)
    cls[:, ::11, 1] = cls[:, ::11, 0]
    cnt = rng.integers(0, 3, (b, n)).astype(np.int32)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    boxes, scores = T.decode_bin_anchor_rows(t(anchors), t(reg), t(cls), t(cnt))
    eb, es = decode_rows_np(anchors, reg, cls, cnt)
    assert np.array_equal(boxes.cpu().numpy(), eb)
    g = scores.cpu().numpy().astype(np.float64)
    ulp = np.spacing(es.astype(np.float32)).astype(np.float64)
    assert (np.abs(g - es) <= 2 * np.maximum(ulp, 0)).all() and (g[cnt == 0] == 0).all()

    full = t(np.full(b, n, np.int32))
    blk0, c0 = T.bev_nms(boxes, scores, 0.1, 100)
    blk1, c1 = T.bev_nms_counted(boxes, scores, full, 0.1, 100)
    assert torch.equal(blk0, blk1) and torch.equal(c0, c1)
    nv = np.array([100, 37, 0], np.int32)
    blk2, c2 = T.bev_nms_counted(boxes, scores, t(nv), 0.1, 100)
    for s in range(b):
        if nv[s] == 0:
            assert c2[s].item() == 0 and not blk2[s].any()
            continue
        e, ec = T.bev_nms(boxes[s:s + 1, :nv[s]].contiguous(), scores[s:s + 1, :nv[s]].contiguous(), 0.1, 100)
        assert torch.equal(blk2[s:s + 1], e) and c2[s].item() == ec.item()


@pytest.fixture(scope="module")
def two_stage(pkg, cuda):
    net = pkg.PointRCNN(device=cuda, seed=0)
    syn = torch.from_numpy(synth.kitti_like(B, 16384, seed=21)).to(cuda)
    real = torch.from_numpy(np.ascontiguousarray(realscan_scenes()[0], np.float32)).to(cuda)
    return net, {"synthetic": syn, "realscan": real}


@pytest.mark.parametrize("name", ["synthetic", "realscan"])
def test_two_stage_forward(pkg, cuda, two_stage, name):
    net, pts = two_stage
    T = pkg.tf_ops
    block, count, d = net.forward(pts[name], return_debug=True)
    torch.cuda.synchronize()
    # the RPN at the test-time NMS equals today's RPN built on the same weights
    head = pkg.head.DetectionHead(C.HEAD_POINTRCNN_RPN, net.params, device=cuda, stage=C.STAGE_POINTRCNN_RPN_TEST)
    rpn = pkg.SABackbone(C.ARCH_POINTRCNN_RPN, net.params, in_channels=1, device=cuda, head=head, aggregation=False)
    xl, fl, _ = rpn.forward(pts[name])
    pb, pc = rpn.detections(xl, fl)
    assert torch.equal(pb, d["proposals"]) and torch.equal(pc, d["proposal_count"])
    # the pool's scan on the expanded proposals
    props, pcount = d["proposals"], d["proposal_count"].cpu().numpy()
    e = props[..., :7].clone()
    e[..., 3:6] += 1.0
    qi, qc = T.query_boxes_3d_points(512, d["rpn_xyz"][-1], e.contiguous())
    valid = torch.arange(100, device=cuda)[None] < d["proposal_count"][:, None].long()
    assert torch.equal(d["pool_cnt"], torch.where(valid, qc, 0))
    assert torch.equal(d["pool_idx"], torch.where(valid[..., None], qi, 0))
    assert tuple(d["pool_feat"].shape) == (B * 100, 512, 256) and tuple(d["rcnn_feat"][4].shape) == (B * 100, 512)
    c = count.cpu().numpy()
    assert (c <= pcount).all()
    bx = d["boxes"].cpu().numpy()
    for s in range(B):                                        # every kept box is one of the scene's real proposals
        for k in range(c[s]):
            hit = np.flatnonzero((bx[s, :pcount[s]] == block[s, k, :7].cpu().numpy()).all(-1))
            assert len(hit) >= 1


SAMPLED = 16          # pooled scenes per batch checked against the oracle and float64 (of 800; they are independent)


@pytest.mark.parametrize("name", ["synthetic", "realscan"])
def test_stage2_network_vs_oracle_and_float64(oracle_ops, cuda, two_stage, name):
    """The stage-2 network on its own inputs, teacher-forced layer by layer:
      * rcnn_layer1 / rcnn_layer2 on a seeded sample of pooled scenes (plus the last real proposal of each scene): the
        D-FPS indices, neighbour lists, counts and centres equal the CPU oracle's (oracle/layers.py) bit for bit, every
        D-FPS is a farthest-point walk in float64, and the features match float64 at the feature tolerance;
      * rcnn_layer3 (SA_Layer_SSG_Last) and the rcnn_head convs (conv1d_0, pred_cls / pred_reg chains) on all B * 100
        rows against float64;
      * the decode bit for bit against the numpy restatement, scores within 2 ulp of the float64 softmax times the
        pool mask, and the final block against the C twin's BEV NMS over each scene's real proposals."""
    from oracle import layers as olayers
    net, pts = two_stage
    block, count, d = net.forward(pts[name], return_debug=True)
    torch.cuda.synchronize()
    prm = net.params.raw
    xl, fl, fps, dbg = d["rcnn_xyz"], d["rcnn_feat"], d["rcnn_fps"], d["rcnn_dbg"]
    pcount = d["proposal_count"].cpu().numpy()
    rng = np.random.default_rng(17 if name == "synthetic" else 18)
    rows = set(rng.choice(B * 100, SAMPLED, replace=False).tolist()) | {s * 100 + max(int(pcount[s]) - 1, 0) for s in range(B)}
    rows = np.array(sorted(rows))
    sel = torch.from_numpy(rows).to(cuda)
    d64 = lambda t: t[sel].double()
    for li, spec in ((2, C.ARCH_POINTRCNN_RCNN[0]), (3, C.ARCH_POINTRCNN_RCNN[1])):
        xi, fi, scope = spec[0][0], spec[1][0], spec[12]
        idx, cnt = dbg[li - 2]["idx"], dbg[li - 2]["cnt"]
        spec64 = list(spec[:15]) + [-1]
        nx, nf = sa_layer64(prm, spec64, d64(xl[xi]), d64(fl[fi]), fps[li][sel], d64(xl[xi]), [i[sel] for i in idx],
                            [c[sel] for c in cnt])
        assert torch.equal(nx.float(), xl[li][sel]), "%s: centres of %s" % (name, scope)
        assert_close(fl[li][sel], nf, "%s: features of %s" % (name, scope))
        assert_fps(d64(xl[xi]), fps[li][sel], "%s: %s D-FPS" % (name, scope))
        for q in rows:
            npy = lambda t: t[q:q + 1].cpu().numpy()
            ex, ef, ei, ed = olayers.pointnet_sa_module_msg(
                npy(xl[xi]), npy(fl[fi]), spec[2], spec[3], spec[4], False, None, spec[5], spec[6], spec[7], spec[8], None,
                False, scope, spec[13], None, -1, params=prm, aggregation=False, return_debug=True)
            np.testing.assert_array_equal(npy(fps[li]), ei, err_msg="%s: %s D-FPS of pooled scene %d" % (name, scope, q))
            np.testing.assert_array_equal(npy(idx[0]), ed["idx"][0], err_msg="%s: %s ball query of %d" % (name, scope, q))
            np.testing.assert_array_equal(npy(cnt[0]), ed["cnt"][0], err_msg="%s: %s counts of %d" % (name, scope, q))
            np.testing.assert_array_equal(npy(xl[li]), ex, err_msg="%s: %s centres of %d" % (name, scope, q))
            e = rel_err(npy(fl[li]), ef, rtol=FEATURE_TOL)
            assert e < FEATURE_TOL, "%s: %s features of pooled scene %d vs the oracle: rel err %g" % (name, scope, q, e)
    # rcnn_layer3: concat [xyz | features] -> three convs -> max over the 32 points, all rows
    g = torch.cat([xl[3].double(), fl[3].double()], dim=-1)
    for j in range(3):
        g = conv64(prm, "rcnn_layer3/conv%d" % j, g, True, True)
    assert_close(fl[4], g.amax(dim=1), "%s: features of rcnn_layer3" % name)
    # rcnn_head on the [B, 100, 512] features
    f = fl[4].double().view(B, 100, 512)
    h = conv64(prm, "rcnn_head/conv1d_0", f, True, True)
    cls = conv64(prm, "rcnn_head/pred_cls", conv64(prm, "rcnn_head/pred_cls_base", h, True, True), False, False)
    reg = conv64(prm, "rcnn_head/pred_reg", conv64(prm, "rcnn_head/pred_reg_base", h, True, True), False, False)
    assert tuple(d["cls"].shape) == (B, 100, 2) and tuple(d["reg"].shape) == (B, 100, 52)
    # three chained split-operand convs on rcnn_layer3's output: held to FEATURE_TOL of max|exp| as a whole, elementwise
    # to rel_err's default 1e-3 of each value (the 2-channel cls output is small: its worst element on the real-scan
    # batch is 2.3e-5 of max|exp| off float64, just over FEATURE_TOL's elementwise bound of 2e-5 + 1e-4 |exp|)
    for what, got, exp in (("cls", d["cls"], cls), ("reg", d["reg"], reg)):
        e = rel_err(got.double().cpu().numpy(), exp.cpu().numpy())
        assert e < FEATURE_TOL, "%s: rcnn_head %s rel err %g" % (name, what, e)
    # decode, scores, and the NMS through the C twin over each scene's real proposals
    props = d["proposals"].cpu().numpy()
    eb, es = decode_rows_np(props, d["reg"].cpu().numpy(), d["cls"].cpu().numpy(), d["pool_cnt"].cpu().numpy())
    boxes, scores = d["boxes"].cpu().numpy(), d["scores"].cpu().numpy()
    np.testing.assert_array_equal(boxes.view(np.uint32), eb.view(np.uint32))
    ulp = np.spacing(es.astype(np.float32)).astype(np.float64)
    assert (np.abs(scores.astype(np.float64) - es) <= 2 * ulp).all(), "%s: stage-2 scores beyond 2 ulp" % name
    blk, cnt = block.cpu().numpy(), count.cpu().numpy()
    for s in range(B):
        nv = int(pcount[s])
        if nv == 0:
            assert cnt[s] == 0 and not blk[s].any()
            continue
        eblk, ecnt = oracle_ops.bev_nms(boxes[s:s + 1, :nv], scores[s:s + 1, :nv], C.STAGE_POINTRCNN_RCNN["NMS_THRESH"],
                                        C.STAGE_POINTRCNN_RCNN["MAX_OUTPUT_NUM"])
        assert cnt[s] == ecnt[0], "%s: scene %d keeps %d boxes, the C twin %d" % (name, s, cnt[s], ecnt[0])
        np.testing.assert_array_equal(blk[s].view(np.uint32), eblk[0].view(np.uint32))


def test_two_stage_graph_replay_equals_eager(pkg, cuda, two_stage):
    net, pts = two_stage
    replay = net.capture(pts["synthetic"])
    blk, cnt = replay(pts["realscan"])
    torch.cuda.synchronize()
    eb, ec = net.forward(pts["realscan"])
    assert torch.equal(blk, eb) and torch.equal(cnt, ec)
    blk, cnt = replay(pts["synthetic"])
    torch.cuda.synchronize()
    eb, ec = net.forward(pts["synthetic"])
    assert torch.equal(blk, eb) and torch.equal(cnt, ec)


def test_eval_tool_runs_the_two_stage_detector(pkg, cuda, tmp_path):
    import subprocess
    import sys
    from oracle import kitti_eval as K
    from test_kitti_eval_gpu import _label_text
    io = pkg.kitti_io
    pts = np.ascontiguousarray(realscan_scenes()[0][:4], np.float32)
    p2 = np.array([[721.5, 0, 609.6, 44.9], [0, 721.5, 172.9, 0.2], [0, 0, 1, 0.003]], np.float32)
    _, labels, _ = K.synthetic_frames(4, seed=24, max_labels=6)
    (tmp_path / "label_2").mkdir()
    (tmp_path / "samples").mkdir()
    for i, lab in enumerate(labels):
        (tmp_path / "label_2" / ("%06d.txt" % i)).write_text(_label_text(lab))
        np.save(tmp_path / "samples" / ("%06d.npy" % i),
                np.array({io.KEY_POINT_CLOUD: pts[i], io.KEY_STEREO_CALIB: p2, io.KEY_SAMPLE_NAME: i}, dtype=object),
                allow_pickle=True)
    np.savez(tmp_path / "weights.npz", **pkg.rcnn.init_pointrcnn_params(4))
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "eval_kitti.py"), "--samples", str(tmp_path / "samples"),
                          "--labels", str(tmp_path / "label_2"), "--weights", str(tmp_path / "weights.npz"), "--batch", "4",
                          "--cls-thresh", "0.0", "--model", "pointrcnn"], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "precision_3d:" in out.stdout and "evaluated 4 frames" in out.stdout
