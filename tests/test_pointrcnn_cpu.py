"""PointRCNN's first stage (configs/kitti/pointrcnn/tiny_pointrcnn_stage1.yaml) as data, checked without a GPU: the
layer table's channels, the variable names of its weights, the numpy 'Bin-Anchor' decode on hand-computed rows, the C
NMS twin at the RPN's IoU threshold, and the SA route plan of every scale."""
import importlib

import numpy as np
import pytest

from oracle import head as ohead

C = importlib.import_module("3dssd_b200.config")
P = importlib.import_module("3dssd_b200.params")

BN = ["weights", "biases", "bn/gamma", "bn/beta", "bn/moving_mean", "bn/moving_variance"]


# ---- numpy restatements of the RPN's head and decode (also used by tests/test_pointrcnn_gpu.py) ----------------------

def decode_bin_anchor(xyz, reg, cls, anchor_lhw, half_bin_search_range=3.0, bin_num=12, angle_bins=12):
    """decode_bin_anchor (lib/utils/anchor_decoder.py:115-164) on the anchors of generate_3d_anchors_by_point_tf
    (lib/utils/generate_anchors.py:33-65, one anchor size per point) + the sigmoid, in TF's float32 operation order with
    every operation rounded on its own: reg [..., 4*bin_num + 4 + 2*angle_bins] = [x_bin | x_res | z_bin | z_res | y_res |
    size_res 3 | angle_cls | angle_res] -> boxes [..., 7], score [...] (of cls[..., 0]).  argmax ties to the first index."""
    f32 = np.float32
    xyz, reg = np.asarray(xyz, f32), np.asarray(reg, f32)
    nb = bin_num
    pick = lambda v, k: np.take_along_axis(v, k[..., None], axis=-1)[..., 0]
    interval = f32(half_bin_search_range * 2 / nb)
    xb, zb = np.argmax(reg[..., 0:nb], -1), np.argmax(reg[..., 2 * nb:3 * nb], -1)
    dx = ((xb.astype(f32) + pick(reg[..., nb:2 * nb], xb)) + f32(0.5)) * interval
    dz = ((zb.astype(f32) + pick(reg[..., 3 * nb:4 * nb], zb)) + f32(0.5)) * interval
    off = reg[..., 4 * nb:4 * nb + 4]
    al, ah, aw = (f32(v) for v in anchor_lhw)
    x = (xyz[..., 0] - f32(half_bin_search_range)) + dx
    z = (xyz[..., 2] - f32(half_bin_search_range)) + dz
    y = (xyz[..., 1] + ah / f32(2.0)) + off[..., 0]
    lhw = [np.maximum(a + off[..., 1 + i], f32(0.1)) for i, a in enumerate((al, ah, aw))]
    ang = reg[..., 4 * nb + 4:]
    ab = np.argmax(ang[..., :angle_bins], -1)
    ry = f32(0.0) + ((ab.astype(f32) + pick(ang[..., angle_bins:2 * angle_bins], ab)) + f32(0.0)) * f32(2 * np.pi / angle_bins)
    boxes = np.stack([x, y, z] + lhw + [ry], -1).astype(f32)
    score = (1.0 / (1.0 + np.exp(-np.asarray(cls, np.float64)[..., 0]))).astype(f32)
    return boxes, score


def head_forward_bin_anchor(xyz, feat, params, anchor_lhw, bn=True, scope="rpn_head", half_bin_search_range=3.0, bin_num=12):
    """The 'Bin-Anchor' detection head of PointRCNN's RPN (head_builder.py:81-114, head_util.py:26-59 with an empty MLP
    list and pred_reg_channel_num = 4 * bin_num + 4): the four convs, then decode_bin_anchor + sigmoid."""
    pre = scope + "/"
    cls = ohead._conv(params, pre + "pred_cls", ohead._conv(params, pre + "pred_cls_base", feat, bn, True), False, False)
    reg = ohead._conv(params, pre + "pred_reg", ohead._conv(params, pre + "pred_reg_base", feat, bn, True), False, False)
    boxes, score = decode_bin_anchor(xyz, reg, cls, anchor_lhw, half_bin_search_range, bin_num)
    return boxes, score, {"cls": cls, "reg": reg}


def without_aggregation(arch):
    """The table as the CPU oracle's backbone_forward runs it with AGGREGATION_SA_FEATURE False: an SA layer whose
    aggregation_channel is -1 has no aggregation conv, exactly what the global switch does (layers_util.py:183-185)."""
    return [list(spec[:15]) + [-1] for spec in arch]


def test_channels():
    assert C.layer_channels(C.ARCH_POINTRCNN_RPN, 1, aggregation=False) == [1, 96, 256, 512, 1024, 512, 512, 256, 128]
    assert C.layer_channels(C.ARCH_3DSSD, 1) == C.layer_channels(C.ARCH_3DSSD, 1, aggregation=True)


def test_3dssd_params_unchanged_by_the_aggregation_argument():
    a, b = P.init_params(C.ARCH_3DSSD, 1), P.init_params(C.ARCH_3DSSD, 1, aggregation=True)
    assert a.keys() == b.keys() and all(np.array_equal(a[k], b[k]) for k in a)


def test_variable_names_and_shapes():
    """Names written out from the yaml and the reference's scopes: pointnet_sa_module_msg's conv{i}_{j} under the layer
    scope (layers_util.py:175, no 'ensemble' with AGGREGATION_SA_FEATURE False), pointnet_fp_module's conv_{j}
    (:218-222), the head's pred_{cls,reg}{_base,} under 'rpn_head' (head_util.py:36-41; MLP list empty)."""
    st = C.STAGE_POINTRCNN_RPN
    prm = P.init_params(C.ARCH_POINTRCNN_RPN, 1, aggregation=False)
    hp = P.init_head_params(128, mlp=(), reg_channels=4 * st["BIN_CLASS_NUM"] + 4 + 24, scope="rpn_head")
    want = set()
    for layer in range(1, 5):
        want |= {"rpn_layer%d/conv%d_%d/%s" % (layer, i, j, v) for i in range(2) for j in range(3) for v in BN}
    for layer in range(1, 5):
        want |= {"rpn_fp_layer%d/conv_%d/%s" % (layer, j, v) for j in range(2) for v in BN}
    want |= {"rpn_head/%s/%s" % (s, v) for s in ("pred_cls_base", "pred_reg_base") for v in BN}
    want |= {"rpn_head/%s/%s" % (s, v) for s in ("pred_cls", "pred_reg") for v in ("weights", "biases")}
    assert set(prm) | set(hp) == want
    shapes = {"rpn_layer1/conv0_0": (4, 16), "rpn_layer1/conv1_2": (32, 64), "rpn_layer2/conv0_0": (99, 64),
              "rpn_layer3/conv0_1": (128, 196), "rpn_layer3/conv1_2": (196, 256), "rpn_layer4/conv1_1": (256, 384),
              "rpn_fp_layer4/conv_0": (1536, 512), "rpn_fp_layer3/conv_0": (768, 512), "rpn_fp_layer2/conv_0": (608, 256),
              "rpn_fp_layer1/conv_0": (257, 128), "rpn_fp_layer1/conv_1": (128, 128)}
    for k, s in shapes.items():
        assert prm[k + "/weights"].shape == s, k
    assert hp["rpn_head/pred_reg/weights"].shape == (128, 76) and hp["rpn_head/pred_cls/weights"].shape == (128, 1)


def _row(xb, xr, zb, zr, yres, size, ab, ar):
    r = np.zeros(76, np.float32)
    r[0:12], r[12:24], r[24:36], r[36:48] = xb, xr, zb, zr
    r[48], r[49:52], r[52:64], r[64:76] = yres, size, ab, ar
    return r


def test_decode_bin_anchor_hand_rows():
    anchor = C.STAGE_POINTRCNN_RPN["ANCHOR_SIZE"]
    f32 = np.float32
    res = np.arange(12, dtype=np.float32) * f32(0.01)
    onehot = lambda k: np.eye(12, dtype=np.float32)[k]
    rows = np.stack([
        _row(np.zeros(12), res, np.zeros(12), res, 0.25, [0.1, 0.2, -0.3], np.zeros(12), res),     # every bin ties: bin 0
        _row(onehot(11), res, onehot(0), res, -0.5, [-9.0, -9.0, -9.0], onehot(11), res),           # last / first bins, clamp
        _row(onehot(5) * 2 + onehot(7) * 2, res, onehot(3), res, 0.0, [0, 0, 0], onehot(6), res),   # tie 5 / 7: 5
    ])
    xyz = np.array([[10.0, 1.5, 20.0], [-3.0, 0.0, 7.0], [0.0, -1.0, 0.0]], np.float32)
    cls = np.array([[0.0], [2.0], [-1.0]], np.float32)
    boxes, score = decode_bin_anchor(xyz[None], rows[None], cls[None], anchor)
    boxes, score = boxes[0], score[0]
    l, h, w = (f32(v) for v in anchor)
    # x = (ax - 3) + (bin + res + 0.5) * 0.5
    assert boxes[0, 0] == f32(7.0) + f32(0.25) and boxes[0, 2] == f32(17.0) + f32(0.25)
    assert boxes[1, 0] == f32(-6.0) + (f32(11.0) + f32(0.11) + f32(0.5)) * f32(0.5)
    assert boxes[1, 2] == f32(4.0) + f32(0.25)
    assert boxes[2, 0] == f32(-3.0) + (f32(5.0) + f32(0.05) + f32(0.5)) * f32(0.5)
    # y = (ay + h / 2) + y_res; sizes anchor + res, clamped at 0.1
    assert boxes[0, 1] == (f32(1.5) + h * f32(0.5)) + f32(0.25)
    assert boxes[0, 3] == l + f32(0.1) and boxes[0, 4] == h + f32(0.2) and boxes[0, 5] == w + f32(-0.3)
    assert np.all(boxes[1, 3:6] == f32(0.1))
    # ry = (bin + res) * 2 pi / 12
    assert boxes[0, 6] == f32(0.0)
    assert boxes[1, 6] == (f32(11.0) + f32(0.11)) * f32(2 * np.pi / 12)
    assert boxes[2, 6] == (f32(6.0) + f32(0.06)) * f32(2 * np.pi / 12)
    np.testing.assert_array_equal(score, (1.0 / (1.0 + np.exp(-cls[:, 0].astype(np.float64)))).astype(np.float32))


def test_c_nms_twin_at_the_rpn_threshold(oracle_ops):
    """oracle/ssd3d_oracle.c:oracle_bev_nms == oracle/head.py:bev_nms at n = 2048, IoU 0.85, with box pairs shifted a few
    float32 steps either side of the threshold."""
    rng = np.random.default_rng(9)
    b, n = 2, 2048
    bx = np.zeros((b, n, 7), np.float32)
    bx[..., 0] = rng.uniform(-10, 10, (b, n))
    bx[..., 2] = rng.uniform(0, 20, (b, n))
    bx[..., 3] = rng.uniform(3.2, 4.6, (b, n))
    bx[..., 4] = 1.5
    bx[..., 5] = rng.uniform(1.4, 1.9, (b, n))
    bx[..., 6] = rng.uniform(-np.pi, np.pi, (b, n))
    sc = rng.uniform(0, 1, (b, n)).astype(np.float32)
    for p in range(200):                   # IoU (l - d) / (l + d) = 0.85 at d = 0.15 l / 1.85, then +- a few ulp
        i, j = 2 * p, 2 * p + 1
        bx[:, j] = bx[:, i]
        bx[:, i, 6] = bx[:, j, 6] = 0.0
        d = np.float32(0.15 / 1.85) * bx[:, i, 3]
        for _ in range(p % 7 - 3):
            d = np.nextafter(d, np.float32(np.inf))
        for _ in range(3 - p % 7):
            d = np.nextafter(d, np.float32(0))
        bx[:, j, 0] = bx[:, i, 0] + d
        sc[:, i], sc[:, j] = 0.999, 0.998
    for thr in (0.85, 0.1):
        blk, cnt = oracle_ops.bev_nms(bx, sc, thr, 100)
        eblk, ecnt = ohead.bev_nms(bx, sc, thr, 100)
        np.testing.assert_array_equal(cnt, ecnt)
        np.testing.assert_array_equal(blk.view(np.uint32), eblk.view(np.uint32))


@pytest.mark.parametrize("layer", range(4))
def test_sa_route_plan_of_every_scale(layer):
    """Every scale of the four SA layers takes a tensor-core route (plain ball query, K = 16 / 32, a 196-wide conv in
    layer 3), computed from parameter shapes alone."""
    L = importlib.import_module("3dssd_b200.layers_util")
    arch = C.ARCH_POINTRCNN_RPN
    prm = P.init_params(arch, 1, aggregation=False)
    ch = C.layer_channels(arch, 1, aggregation=False)
    spec = arch[layer]
    plan = L._route_plan(P.prepare(prm, "cpu"), spec[12], spec[3], spec[4], True, ch[spec[1][0]], False, "tc", True, True, 2)
    assert plan.tc and plan.agg is None and not plan.split_out
    assert len(plan.scales) == 2
    for sc in plan.scales:
        assert sc.route in ("fused", "fused_hoisted", "gather", "split", "hoisted", "expand")
        if sc.route.startswith("fused"):
            assert sc.stack is not None
