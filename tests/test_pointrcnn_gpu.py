"""PointRCNN's first stage (the RPN of configs/kitti/pointrcnn/tiny_pointrcnn_stage1.yaml) on the GPU: the fused FP-layer
operand, the 'Bin-Anchor' decode, the BEV NMS over up to 16 384 candidates per scene, and the whole RPN from raw points
to proposals against the CPU oracle, on synthetic scenes and on regions of the real KITTI scan."""
import importlib

import numpy as np
import pytest
import torch

from oracle import head as ohead
from test_backbone_gpu import TOL, rel_err
from test_bench_step_gpu import assert_scores_2ulp
from test_pointrcnn_cpu import decode_bin_anchor, head_forward_bin_anchor, without_aggregation
from test_realscan_cpu import realscan_scenes

pytestmark = pytest.mark.gpu

synth = importlib.import_module("3dssd_b200.synth")
C = importlib.import_module("3dssd_b200.config")

# (n unknown, m known, c2 interpolated channels, c1 own channels) of rpn_fp_layer4 .. rpn_fp_layer1
FP_SHAPES = [(256, 64, 1024, 512), (1024, 256, 512, 256), (4096, 1024, 512, 96), (16384, 4096, 256, 1)]


def pinned_weights(dist):
    """The CPU oracle's weight order (oracle/layers.py:pointnet_fp_module): inv_k = 1 / max(d_k, 1e-10), norm = (inv_0 + inv_1) + inv_2, w_k = inv_k / norm."""
    f32 = np.float32
    inv = f32(1.0) / np.maximum(dist, f32(1e-10))
    norm = (inv[..., 0:1] + inv[..., 1:2]) + inv[..., 2:3]
    return (inv / norm).astype(f32)


def fp_operands(b, n, m, c2, c1, seed, dups=False):
    rng = np.random.default_rng(seed)
    xyz2 = rng.uniform(-20, 20, (b, m, 3)).astype(np.float32)
    xyz1 = rng.uniform(-20, 20, (b, n, 3)).astype(np.float32)
    if dups:                                   # repeated known points, and unknown points sitting on known ones (d = 0)
        xyz2[:, 1::3] = xyz2[:, 0:1]
        k = min(n, m)
        xyz1[:, :k:2] = xyz2[:, :k:2]
    p2 = rng.standard_normal((b, m, c2)).astype(np.float32)
    p1 = rng.standard_normal((b, n, c1)).astype(np.float32)
    return xyz1, xyz2, p2, p1


def check_fp_operand(pkg, oracle_ops, cuda, xyz1, xyz2, p2, p1):
    T = pkg.tf_ops
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    hi, lo = T.fp_interp_split(t(xyz1), t(xyz2), t(p2), t(p1))
    dist, idx = T.three_nn(t(xyz1), t(xyz2))
    edist, eidx = oracle_ops.three_nn(xyz1, xyz2)
    np.testing.assert_array_equal(idx.cpu().numpy(), eidx, err_msg="three_nn indices")
    np.testing.assert_array_equal(dist.cpu().numpy().view(np.uint32), edist.view(np.uint32), err_msg="three_nn distances")
    w = t(pinned_weights(edist))
    x = torch.cat([T.three_interpolate(t(p2), idx, w), t(p1)], dim=2).contiguous()
    ehi, elo = T.split_rows(x)
    assert torch.equal(hi.view(torch.int16), ehi.view(torch.int16)), "fp operand hi"
    assert torch.equal(lo.view(torch.int16), elo.view(torch.int16)), "fp operand lo"


@pytest.mark.parametrize("shape", FP_SHAPES, ids=["fp4", "fp3", "fp2", "fp1"])
def test_fp_operand_bit_identical(pkg, oracle_ops, cuda, shape):
    n, m, c2, c1 = shape
    check_fp_operand(pkg, oracle_ops, cuda, *fp_operands(8, n, m, c2, c1, seed=n, dups=(n == 1024)))


@pytest.mark.parametrize("m", [1, 2, 3])
def test_fp_operand_few_known_points_and_duplicates(pkg, oracle_ops, cuda, m):
    check_fp_operand(pkg, oracle_ops, cuda, *fp_operands(8, 300, m, 24, 5, seed=m, dups=True))


def test_fp_operand_rejects_no_known_points(pkg, cuda):
    z = lambda *s: torch.zeros(s, dtype=torch.float32, device=cuda)
    with pytest.raises(ValueError):
        pkg.tf_ops.fp_interp_split(z(1, 4, 3), z(1, 0, 3), z(1, 0, 8), z(1, 4, 2))


def test_fp_module_at_rpn_shape_vs_oracle(pkg, cuda):
    from oracle import layers as olayers
    n, m, c2, c1 = FP_SHAPES[1]
    xyz1, xyz2, p2, p1 = fp_operands(2, n, m, c2, c1, seed=5)
    prm = {}
    rngp = np.random.default_rng(2)
    pkg.params._conv_init(rngp, prm, "fp/conv_0", c2 + c1, 512, True)
    pkg.params._conv_init(rngp, prm, "fp/conv_1", 512, 512, True)
    t = lambda a: torch.from_numpy(a).to(cuda)
    got = pkg.pointnet_fp_module(t(xyz1), t(xyz2), t(p1), t(p2), [512, 512], False, None, "fp", True, params=prm)
    exp = olayers.pointnet_fp_module(xyz1, xyz2, p1, p2, [512, 512], False, None, "fp", True, params=prm)
    assert rel_err(got.cpu().numpy(), exp) < TOL


# ---- decode -------------------------------------------------------------------------------------------------------

def test_decode_bin_anchor_vs_oracle(pkg, cuda):
    st = C.STAGE_POINTRCNN_RPN
    rng = np.random.default_rng(3)
    b, n = 8, 4096
    xyz = rng.uniform(-40, 40, (b, n, 3)).astype(np.float32)
    reg = rng.standard_normal((b, n, 76)).astype(np.float32)
    reg[:, ::7, 0:12] = 0.5                                  # all x bins tie: the first wins
    reg[:, ::5, 24:36] = np.float32(1.0)                     # z bins tie
    reg[:, 1::5, 24 + 11] = 9.0                              # the last z bin
    reg[:, ::3, 49:52] = -10.0                               # sizes clamped to 0.1
    reg[:, 1::9, 52:64] = 0.0                                # angle bins tie
    cls = rng.standard_normal((b, n, 1)).astype(np.float32) * 6
    t = lambda a: torch.from_numpy(a).to(cuda)
    boxes, score = pkg.tf_ops.decode_bin_anchor(t(xyz), t(reg), t(cls), st["ANCHOR_SIZE"], st["HALF_BIN_SEARCH_RANGE"],
                                                st["BIN_CLASS_NUM"])
    eb, _ = decode_bin_anchor(xyz, reg, cls, st["ANCHOR_SIZE"], st["HALF_BIN_SEARCH_RANGE"], st["BIN_CLASS_NUM"])
    np.testing.assert_array_equal(boxes.cpu().numpy().view(np.uint32), eb.view(np.uint32))
    assert_scores_2ulp(score, t(cls)[..., 0])


# ---- NMS ----------------------------------------------------------------------------------------------------------

def nms_scene(rng, n, kind):
    """boxes [n, 7], scores [n]: 'mixed' random cars with bisected near-threshold pairs, 'sparse' disjoint boxes (100 are
    kept early), 'pile' boxes jittered around one spot (the walk never fills 100 at IoU 0.1)."""
    bx = np.zeros((n, 7), np.float32)
    if kind == "pile":
        bx[:, 0] = rng.uniform(-0.05, 0.05, n)
        bx[:, 2] = 20 + rng.uniform(-0.05, 0.05, n)
    else:
        bx[:, 0] = rng.uniform(-40, 40, n)
        bx[:, 2] = rng.uniform(0, 70, n)
    if kind == "sparse":
        g = int(np.ceil(np.sqrt(n)))
        bx[:, 0] = (np.arange(n) % g) * 6.0
        bx[:, 2] = (np.arange(n) // g) * 6.0
    bx[:, 1] = rng.uniform(-2, 2, n)
    bx[:, 3] = rng.uniform(3.2, 4.6, n)
    bx[:, 4] = rng.uniform(1.4, 1.8, n)
    bx[:, 5] = rng.uniform(1.4, 1.9, n)
    bx[:, 6] = rng.uniform(-np.pi, np.pi, n) if kind != "sparse" else 0.0
    sc = rng.uniform(0, 1, n).astype(np.float32)
    sc[rng.integers(0, n, n // 16)] = 0.5                   # ties
    if kind == "mixed":                                      # pairs a hair either side of IoU 0.85, the kept one first
        for p in range(min(64, n // 8)):
            i, j = 2 * p, 2 * p + 1
            bx[j] = bx[i]
            bx[i, 6] = bx[j, 6] = 0.0
            lo, hi = 0.0, float(bx[i, 3])
            for _ in range(60):                              # bisect the x shift where the float32 IoU crosses 0.85
                mid = 0.5 * (lo + hi)
                bx[j, 0] = np.float32(bx[i, 0] + mid)
                a = ohead.bev_rects(bx[[i, j]])
                iw = min(a[0, 2], a[1, 2]) - max(a[0, 0], a[1, 0])
                ih = min(a[0, 3], a[1, 3]) - max(a[0, 1], a[1, 1])
                ar = (a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1])
                iou = np.float32(iw * ih) / ((ar[0] + ar[1]) - np.float32(iw * ih))
                lo, hi = (mid, hi) if iou > np.float32(0.85) else (lo, mid)
            bx[j, 0] = np.float32(bx[i, 0] + (lo if p % 2 else hi))
            sc[i], sc[j] = np.float32(0.99 - p * 1e-3), np.float32(0.985 - p * 1e-3)
    return bx, sc


@pytest.mark.parametrize("n", [513, 4096, 16384])
@pytest.mark.parametrize("thr", [0.85, 0.1])
def test_bev_nms_large_vs_c_twin(pkg, oracle_ops, cuda, n, thr):
    rng = np.random.default_rng(n + int(thr * 100))
    kinds = ["mixed", "sparse", "pile", "mixed", "mixed", "sparse", "pile", "mixed"]
    scenes = [nms_scene(rng, n, k) for k in kinds]
    boxes = np.stack([s[0] for s in scenes])
    scores = np.stack([s[1] for s in scenes])
    blk, cnt = pkg.tf_ops.bev_nms(torch.from_numpy(boxes).to(cuda), torch.from_numpy(scores).to(cuda), thr, 100)
    eblk, ecnt = oracle_ops.bev_nms(boxes, scores, thr, 100)
    np.testing.assert_array_equal(cnt.cpu().numpy(), ecnt)
    np.testing.assert_array_equal(blk.cpu().numpy().view(np.uint32), eblk.view(np.uint32))
    assert ecnt[1] == 100                                    # the sparse scene fills the block early
    if thr == 0.1:
        assert ecnt[2] < 100                                 # the pile never fills the block


def test_bev_nms_rejects_more_than_16384(pkg, cuda):
    with pytest.raises(ValueError):
        pkg.tf_ops.bev_nms(torch.zeros((1, 16385, 7), device=cuda), torch.zeros((1, 16385), device=cuda), 0.85, 100)


# ---- the whole RPN ------------------------------------------------------------------------------------------------

def make_rpn(pkg, cuda):
    P = pkg.params
    arch, st = C.ARCH_POINTRCNN_RPN, C.STAGE_POINTRCNN_RPN
    params = P.init_params(arch, 1, seed=0, aggregation=False)
    ch = C.layer_channels(arch, 1, aggregation=False)
    hp = P.init_head_params(ch[-1], mlp=(), reg_channels=4 * st["BIN_CLASS_NUM"] + 4 + 24, seed=1, scope="rpn_head")
    head = pkg.head.DetectionHead(C.HEAD_POINTRCNN_RPN, hp, device=cuda, stage=st)
    net = pkg.SABackbone(arch, params, in_channels=1, device=cuda, head=head, aggregation=False)
    return net, params, hp


@pytest.fixture(scope="module")
def rpn(pkg, cuda):
    return make_rpn(pkg, cuda)


def rpn_scenes():
    syn = synth.kitti_like(1, 16384, seed=77)
    real = realscan_scenes()[0][[3]]
    return {"synthetic": syn.astype(np.float32), "realscan": np.ascontiguousarray(real, np.float32)}


@pytest.mark.parametrize("name", ["synthetic", "realscan"])
def test_rpn_full_size_vs_oracle(pkg, oracle_ops, cuda, rpn, name):
    from oracle import layers as olayers
    net, params, hp = rpn
    st = C.STAGE_POINTRCNN_RPN
    pts = rpn_scenes()[name]
    out = net.forward(torch.from_numpy(pts).to(cuda), return_debug=True)
    blk, cnt, raw = net.head.forward(out[0], out[1], return_raw=True)
    exp = olayers.backbone_forward(without_aggregation(C.ARCH_POINTRCNN_RPN), pts, params, return_debug=True)
    xyz_l, feat_l, fps_l, dbg = out
    for li in range(1, 9):
        if exp[2][li] is not None:
            np.testing.assert_array_equal(fps_l[li].cpu().numpy(), exp[2][li], err_msg="fps_idx layer %d" % li)
        for s, (a, b) in enumerate(zip(dbg[li - 1].get("idx", []), exp[3][li - 1].get("idx", []))):
            np.testing.assert_array_equal(a.cpu().numpy(), b, err_msg="ball-query idx layer %d scale %d" % (li, s))
        e = rel_err(feat_l[li].cpu().numpy(), exp[1][li])
        assert e < TOL, "features of layer %d: rel err %g" % (li, e)
    eb, es, eraw = head_forward_bin_anchor(exp[0][8], exp[1][8], hp, st["ANCHOR_SIZE"])
    assert rel_err(raw["cls"].cpu().numpy(), eraw["cls"]) < TOL
    assert rel_err(raw["reg"].cpu().numpy(), eraw["reg"]) < TOL
    # the decode of the kernel's own head output is the oracle's, bit for bit
    kb, _ = decode_bin_anchor(out[0][8].cpu().numpy(), raw["reg"].cpu().numpy(), raw["cls"].cpu().numpy(), st["ANCHOR_SIZE"])
    boxes = raw["boxes"][:, :, 0].cpu().numpy()
    np.testing.assert_array_equal(boxes.view(np.uint32), kb.view(np.uint32))
    # against the oracle's boxes: equal bins decide equal boxes up to the features' tolerance; a bin may flip only at a
    # near tie of two logits
    same = np.all(np.abs(boxes - eb) < 1e-2 * np.maximum(1.0, np.abs(eb)), axis=-1)
    assert same.mean() > 0.995, "boxes away from the oracle's at %d of %d points" % ((~same).sum(), same.size)
    # proposals: the oracle NMS on the kernel's own decoded boxes and scores
    oblk, ocnt = oracle_ops.bev_nms(boxes, raw["score"][..., 0].cpu().numpy(), st["NMS_THRESH"], st["MAX_OUTPUT_NUM"])
    np.testing.assert_array_equal(cnt.cpu().numpy(), ocnt)
    np.testing.assert_array_equal(blk.cpu().numpy().view(np.uint32), oblk.view(np.uint32))


def test_rpn_graph_replay_equals_eager(pkg, cuda, rpn):
    net = rpn[0]
    a = torch.from_numpy(synth.kitti_like(2, 16384, seed=5)).to(cuda)
    b = torch.from_numpy(realscan_scenes()[0][[0, 7]]).to(cuda)
    replay = net.capture(a)
    for pts in (a, b):
        out, (blk, cnt) = replay(pts)
        torch.cuda.synchronize()
        got = [f.clone() for f in out[1][1:]] + [blk.clone(), cnt.clone()]
        eo = net.forward(pts.clone())
        eblk, ecnt = net.detections(eo[0], eo[1])
        for g, e in zip(got, list(eo[1][1:]) + [eblk, ecnt]):
            assert torch.equal(g, e)
