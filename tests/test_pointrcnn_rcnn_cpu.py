"""PointRCNN's second stage (configs/kitti/pointrcnn/tiny_pointrcnn_stage2_test.yaml) checked without a GPU: the config
tables against the yaml, the stage-2 channels and variable names, the numpy restatements of the region pool's membership
scan and of the stage-2 decode on hand cases, and the argument checks of the new entry points.  The restatements are
also the references of tests/test_pointrcnn_rcnn_gpu.py."""
import ctypes
import importlib
import os
import subprocess

import numpy as np
import pytest
import torch

C = importlib.import_module("3dssd_b200.config")
P = importlib.import_module("3dssd_b200.params")
F32 = np.float32
BN = ["weights", "biases", "bn/gamma", "bn/beta", "bn/moving_mean", "bn/moving_variance"]


# ---- numpy restatements (also used by tests/test_pointrcnn_rcnn_gpu.py) ----------------------------------------------

def _fma32(a, b, c):
    """float32 fma: the product is exact in float64, the sum rounded there and then to float32 (a double rounding that
    can differ from the device's single rounding only within an ulp of a float32 tie: see ambiguous())."""
    return (np.float64(a) * np.float64(b) + np.float64(c)).astype(F32)


def box_constants(box):
    """point_inside_box_3d's per-box values (tf_grouping_g.cu:27-40, :65-72) by the arithmetic of the reference build."""
    cx, by, cz, l, h, w, ry = (F32(v) for v in box[:7])
    hl, hw = np.float64(l) * 0.5, np.float64(w) * 0.5
    maxd = max(F32(np.sqrt(F32(hl * hl + hw * hw))), F32(1e-20))
    c, s = F32(np.cos(ry)), F32(np.sin(ry))
    return cx, by, cz, h, c, s, maxd, hl, hw


def inside_np(xyz, box):
    """(inside [n] bool, ambiguous [n] bool) of xyz [n, 3] against one bottom-centred box.  Ambiguous: within a few ulp
    of a face, where the host's cosf / fma rounding may legitimately differ from the device's."""
    cx, by, cz, h, c, s, maxd, hl, hw = box_constants(box)
    xyz = np.asarray(xyz, F32)
    x, y, z = xyz[:, 0], xyz[:, 1], xyz[:, 2]
    dx, dz = (x - cx).astype(F32), (z - cz).astype(F32)
    pre = (np.abs(dx) <= maxd) & ~(y > by) & ~((by - y).astype(F32) > h) & (np.abs(dz) <= maxd)
    u = _fma32(dx, c, -(dz * s).astype(F32)).astype(np.float64)
    v = _fma32(dz, c, (dx * s).astype(F32)).astype(np.float64)
    inside = pre & (u >= -hl) & (u <= hl) & (v >= -hw) & (v <= hw)
    tol = 8 * np.spacing(F32(max(hl, hw, 1.0))).astype(np.float64) + 4e-7 * (np.abs(dx) + np.abs(dz))
    amb = pre & ((np.abs(np.abs(u) - hl) <= tol) | (np.abs(np.abs(v) - hw) <= tol))
    amb |= np.abs(np.abs(dx) - maxd) <= 4 * np.spacing(maxd)
    amb |= np.abs(np.abs(dz) - maxd) <= 4 * np.spacing(maxd)
    return inside, amb


def scan_np(xyz, box, nsample):
    """query_boxes_3d_points for one box: (idx [nsample], cnt, ambiguous points among those scanned)."""
    inside, amb = inside_np(xyz, box)
    hits = np.flatnonzero(inside)
    cnt = min(len(hits), nsample)
    stop = hits[nsample - 1] + 1 if len(hits) >= nsample else len(xyz)
    idx = np.full(nsample, hits[0] if cnt else 0, np.int32)
    idx[:cnt] = hits[:cnt]
    return idx, cnt, int(amb[:stop].sum())


def expand(box, context=1.0):
    """expand_proposals_context (points_pooler.py:172-183): l, h, w + context in float32, the bottom centre kept."""
    b = np.asarray(box[:7], F32).copy()
    b[3:6] = (b[3:6] + F32(context)).astype(F32)
    return b


def canonical_np(pts, box):
    """canonical_xyz (points_pooler.py:157-170): rotate_points(pts - box[:3], -ry) in float32."""
    n = (np.asarray(pts, F32) - np.asarray(box[:3], F32)).astype(F32)
    c, s = F32(np.cos(-F32(box[6]))), F32(np.sin(-F32(box[6])))
    x = (c * n[:, 0]).astype(F32) + (s * n[:, 2]).astype(F32)
    z = (-s * n[:, 0]).astype(F32) + (c * n[:, 2]).astype(F32)
    return np.stack([x, n[:, 1], z], -1).astype(F32)


def info_conv64(info, params, scope="roi_pool/conv0"):
    """align_channel_network's conv0 with BN and ReLU in float64 (tf_util.conv2d, pool_utils.py:5-16)."""
    g = np.asarray(params[scope + "/bn/gamma"], np.float64)
    inv = g / np.sqrt(np.asarray(params[scope + "/bn/moving_variance"], np.float64) + P.BN_EPS)
    y = np.asarray(info, np.float64) @ np.asarray(params[scope + "/weights"], np.float64) + params[scope + "/biases"]
    return np.maximum((y - params[scope + "/bn/moving_mean"]) * inv + params[scope + "/bn/beta"], 0.0)


def decode_rows_np(anchors, reg, cls, cnt=None, half_bin_search_range=1.5, bin_num=6, angle_bins=12):
    """The stage-2 decode (anchor_decoder.py:115-164 against the proposals, double_stage_detector.py:298-337) in TF's
    float32 operation order -> boxes [..., 7], and the softmax score in float64 times the pool mask."""
    a, reg = np.asarray(anchors, F32), np.asarray(reg, F32)
    nb = bin_num
    pick = lambda v, k: np.take_along_axis(v, k[..., None], axis=-1)[..., 0]
    interval = F32(half_bin_search_range * 2 / nb)
    xb, zb = np.argmax(reg[..., 0:nb], -1), np.argmax(reg[..., 2 * nb:3 * nb], -1)
    dx = ((xb.astype(F32) + pick(reg[..., nb:2 * nb], xb)) + F32(0.5)) * interval
    dz = ((zb.astype(F32) + pick(reg[..., 3 * nb:4 * nb], zb)) + F32(0.5)) * interval
    off = reg[..., 4 * nb:4 * nb + 4]
    x = (a[..., 0] - F32(half_bin_search_range)) + dx
    z = (a[..., 2] - F32(half_bin_search_range)) + dz
    y = a[..., 1] + off[..., 0]
    lhw = [np.maximum(a[..., 3 + i] + off[..., 1 + i], F32(0.1)) for i in range(3)]
    ang = reg[..., 4 * nb + 4:]
    ab = np.argmax(ang[..., :angle_bins], -1)
    ry = a[..., 6] + ((ab.astype(F32) + pick(ang[..., angle_bins:2 * angle_bins], ab)) + F32(0.0)) * F32(2 * np.pi / angle_bins)
    boxes = np.stack([x, y, z] + lhw + [ry], -1).astype(F32)
    c = np.asarray(cls, np.float64)
    score = 1.0 / (1.0 + np.exp(c[..., 0] - c[..., 1]))
    if cnt is not None:
        score = score * (np.asarray(cnt) > 0)
    return boxes, score


# ---- the tables ------------------------------------------------------------------------------------------------------

def test_stage2_tables_match_the_yaml():
    assert C.STAGE_POINTRCNN_RPN_TEST["NMS_THRESH"] == 0.8 and C.STAGE_POINTRCNN_RPN["NMS_THRESH"] == 0.85
    assert {k: v for k, v in C.STAGE_POINTRCNN_RPN_TEST.items() if k != "NMS_THRESH"} == \
        {k: v for k, v in C.STAGE_POINTRCNN_RPN.items() if k != "NMS_THRESH"}
    assert C.POINTS_POOLER_POINTRCNN == ['RegionPool', ['mask', 'dist'], [128], 512, 1.0, [6, 6, 6, 10], [128], True, 'roi_pool']
    assert C.POOLER_MASK_THRESHOLD == 0.5
    assert C.HEAD_POINTRCNN_RCNN == [[0], [4], 'conv1d', [256], True, 'Det', 'rcnn_head']
    assert C.STAGE_POINTRCNN_RCNN == {"REGRESSION": "Bin-Anchor", "MAX_OUTPUT_NUM": 100, "NMS_THRESH": 0.1,
                                      "HALF_BIN_SEARCH_RANGE": 1.5, "BIN_CLASS_NUM": 6, "CLS_ACTIVATION": "Softmax"}
    a = C.ARCH_POINTRCNN_RCNN
    assert [s[12] for s in a] == ["rcnn_layer1", "rcnn_layer2", "rcnn_layer3"]
    assert [s[11] for s in a] == ["SA_Layer", "SA_Layer", "SA_Layer_SSG_Last"]
    assert [s[8] for s in a[:2]] == [[128], [32]] and [s[2] for s in a[:2]] == [[0.2], [0.4]]
    assert [s[3] for s in a[:2]] == [[64], [64]] and [s[7] for s in a[:2]] == [['D-FPS'], ['D-FPS']]
    assert a[0][4] == [[128, 128, 128]] and a[1][4] == [[128, 128, 256]] and a[2][4] == [256, 256, 512]
    assert [s[0] for s in a] == [[1], [2], [3]] and [s[1] for s in a] == [[1], [2], [3]]


def test_stage2_channels_and_variable_names():
    p = P.init_rcnn_params(128)
    shapes = {k: tuple(v.shape) for k, v in p.items()}
    assert shapes["roi_pool/conv0/weights"] == (5, 128)
    want = {"rcnn_layer1/conv0_0": (259, 128), "rcnn_layer1/conv0_1": (128, 128), "rcnn_layer1/conv0_2": (128, 128),
            "rcnn_layer2/conv0_0": (131, 128), "rcnn_layer2/conv0_1": (128, 128), "rcnn_layer2/conv0_2": (128, 256),
            "rcnn_layer3/conv0": (259, 256), "rcnn_layer3/conv1": (256, 256), "rcnn_layer3/conv2": (256, 512),
            "rcnn_head/conv1d_0": (512, 256), "rcnn_head/pred_cls_base": (256, 128), "rcnn_head/pred_reg_base": (256, 128),
            "roi_pool/conv0": (5, 128)}
    names = set()
    for scope, wshape in want.items():
        assert shapes[scope + "/weights"] == wshape, scope
        for v in BN:
            names.add(scope + "/" + v)
    assert shapes["rcnn_head/pred_cls/weights"] == (128, 2)
    assert shapes["rcnn_head/pred_reg/weights"] == (128, 6 * 4 + 4 + 2 * 12)
    names |= {"rcnn_head/%s/%s" % (s, v) for s in ("pred_cls", "pred_reg") for v in ("weights", "biases")}
    assert set(p) == names
    ch = C.layer_channels([[[i - 1 for i in s[0]], [i - 1 for i in s[1]]] + list(s[2:]) for s in C.ARCH_POINTRCNN_RCNN],
                          256, aggregation=False)
    assert ch == [256, 128, 256, 512]


# ---- the membership scan on hand cases -------------------------------------------------------------------------------

def _grid(lo, hi, step):
    g = np.arange(lo, hi + step / 2, step, dtype=np.float64)
    return np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3).astype(F32)


def test_scan_faces_and_height():
    box = np.array([0, 0, 0, 2, 1, 1, 0], F32)           # x in [-1, 1], y in [-1, 0], z in [-0.5, 0.5]
    pts = np.array([[1, -0.5, 0], [-1, -0.5, 0], [0, -0.5, 0.5], [0, -0.5, -0.5],     # on the x / z faces: inside
                    [0, 0, 0], [0, -1, 0],                                            # y == by and by - y == h: inside
                    [0, np.nextafter(F32(0), F32(1)), 0], [0, np.nextafter(F32(-1), F32(-2)), 0],   # just outside
                    [np.nextafter(F32(1), F32(2)), -0.5, 0], [0, -0.5, np.nextafter(F32(0.5), F32(1))]], F32)
    ins, amb = inside_np(pts, box)
    assert ins.tolist() == [True] * 6 + [False] * 4
    # the pool's expansion by 1.0 grows the box upward only: by - y == h + 1 is the last height inside
    e = expand(box)
    ins, _ = inside_np(np.array([[0, -2, 0], [0, np.nextafter(F32(-2), F32(-3)), 0], [0, 0.25, 0]], F32), e)
    assert ins.tolist() == [True, False, False]


@pytest.mark.parametrize("ry", [0.0, np.pi / 2, -np.pi / 2, np.pi])
def test_scan_rotations(ry):
    box = np.array([1.0, 0.5, 2.0, 3.0, 1.0, 1.0, ry], F32)
    pts = _grid(-2, 4, 0.125)
    ins, amb = inside_np(pts, box)
    # the same box by exact geometry in float64: rotated by ry the long side lies along x (ry = 0, pi) or z (+-pi/2)
    d = pts.astype(np.float64) - box[:3]
    along_x = abs(np.cos(ry)) > 0.5
    lx, lz = (1.5, 0.5) if along_x else (0.5, 1.5)
    exact = (np.abs(d[:, 0]) <= lx) & (np.abs(d[:, 2]) <= lz) & (d[:, 1] <= 0) & (d[:, 1] >= -1)
    ok = ~amb
    assert ok.sum() > 0.9 * len(pts)
    assert np.array_equal(ins[ok], exact[ok])
    assert exact.sum() > 0


def test_scan_first_hits_in_order_and_empty():
    rng = np.random.default_rng(0)
    pts = rng.uniform(-1, 1, (3000, 3)).astype(F32)
    pts[:, 1] = rng.uniform(-0.9, -0.1, 3000)
    box = np.array([0, 0, 0, 1.6, 1, 1.6, 0.3], F32)
    idx, cnt, amb = scan_np(pts, box, 512)
    ins, _ = inside_np(pts, box)
    assert ins.sum() > 512 and cnt == 512
    assert np.array_equal(idx, np.flatnonzero(ins)[:512])
    idx, cnt, _ = scan_np(pts, np.array([50, 0, 50, 1, 1, 1, 0], F32), 512)
    assert cnt == 0 and not idx.any()
    idx, cnt, _ = scan_np(pts, box, 4096)                 # fewer hits than nsample: padded with the first hit
    assert cnt == ins.sum() and (idx[cnt:] == idx[0]).all()


def test_decode_rows_hand_cases():
    nb, na = 6, 12
    reg = np.zeros((3, 4 * nb + 4 + 2 * na), F32)
    reg[0, 2] = 1.0; reg[0, nb + 2] = 0.25                  # x bin 2, res 0.25
    reg[0, 2 * nb + 0] = 3.0; reg[0, 2 * nb + 5] = 3.0     # z bins tie: the first (0) wins
    reg[0, 3 * nb + 0] = -0.5
    reg[0, 4 * nb:4 * nb + 4] = [0.1, 0.2, -10.0, 0.3]     # y res, size res (h clamped to 0.1)
    reg[0, 4 * nb + 4 + 3] = 2.0; reg[0, 4 * nb + 4 + na + 3] = 0.5
    anchors = np.array([[10, 1.5, 20, 3.9, 1.6, 1.5, 0.4, 0.9, 0]] * 3, F32)
    cls = np.array([[0.0, 1.0], [2.0, 2.0], [1.0, 0.0]], F32)
    boxes, score = decode_rows_np(anchors, reg, cls, np.array([5, 1, 0]))
    assert boxes[0, 0] == F32((F32(10) - F32(1.5)) + F32((F32(2.25) + F32(0.5)) * F32(0.5)))
    assert boxes[0, 2] == F32((F32(20) - F32(1.5)) + F32((F32(-0.5) + F32(0.5)) * F32(0.5)))
    assert boxes[0, 1] == F32(F32(1.5) + F32(0.1)) and boxes[0, 4] == F32(0.1)
    assert boxes[0, 6] == F32(F32(0.4) + F32(F32(3.5) * F32(2 * np.pi / 12)))
    assert abs(score[0] - 1 / (1 + np.exp(-1.0))) < 1e-15 and score[1] == 0.5 and score[2] == 0.0


# ---- the C twin of the scan against the numpy restatement ------------------------------------------------------------

@pytest.fixture(scope="module")
def twin(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("roi_twin") / "roi_scan_twin.so")
    subprocess.check_call(["cc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC", "-Wall", "-Werror", "-o", so,
                           os.path.join(os.path.dirname(os.path.abspath(__file__)), "roi_scan_twin.c"), "-lm"])
    lib = ctypes.CDLL(so)

    def scan(xyz, boxes, nsample):
        xyz, boxes = np.ascontiguousarray(xyz, F32), np.ascontiguousarray(boxes, F32)
        m = len(boxes)
        idx, cnt = np.zeros((m, nsample), np.int32), np.zeros(m, np.int32)
        p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        lib.roi_scan(len(xyz), p(xyz), m, p(boxes), nsample, p(idx), p(cnt))
        return idx, cnt
    return scan


def _twin_cases():
    """(points, boxes): the hand cases above, and boxes on point clusters of a seeded scene with > 512 hits, empty boxes,
    overlapping boxes and ry = 0, +-pi/2, pi."""
    rng = np.random.default_rng(3)
    cases = [(np.array([[1, -0.5, 0], [-1, -0.5, 0], [0, -0.5, 0.5], [0, -0.5, -0.5], [0, 0, 0], [0, -1, 0],
                        [0, 1e-30, 0], [0, -1.0000001, 0], [1.0000001, -0.5, 0], [0, -2, 0]], F32),
              np.array([[0, 0, 0, 2, 1, 1, 0], expand([0, 0, 0, 2, 1, 1, 0])], F32))]
    pts = rng.uniform(-20, 20, (6000, 3)).astype(F32)
    pts[:, 1] = rng.uniform(-3, 1, 6000)
    pts[:2000] = (pts[:2000] * F32(0.05)).astype(F32)                # a dense cluster at the origin
    bx = np.zeros((40, 7), F32)
    bx[:, [0, 2]] = pts[rng.choice(6000, 40), :][:, [0, 2]]
    bx[:, 1] = rng.uniform(0, 1.5, 40)
    bx[:, 3:6] = rng.uniform(1, 5, (40, 3))
    bx[:, 6] = rng.uniform(-np.pi, np.pi, 40)
    bx[:4, 6] = [0, np.pi / 2, -np.pi / 2, np.pi]
    bx[4] = [0, 0.5, 0, 4, 3, 4, 0.3]                                 # holds the cluster: > 512 hits
    bx[5] = [500, 0, 500, 2, 2, 2, 0]                                 # empty
    bx[6:9] = bx[9]                                                   # identical boxes
    cases.append((pts, bx))
    return cases


def test_c_twin_scan_equals_the_numpy_scan(twin):
    seen_full = seen_empty = compared = 0
    for pts, boxes in _twin_cases():
        idx, cnt = twin(pts, boxes, 512)
        for r, box in enumerate(boxes):
            ei, ec, amb = scan_np(pts, box, 512)
            if amb:
                continue
            compared += 1
            assert cnt[r] == ec and np.array_equal(idx[r], ei), "box %d" % r
            seen_full += ec == 512
            seen_empty += ec == 0
    assert seen_full >= 1 and seen_empty >= 1 and compared >= 38


# ---- argument checks without a GPU -----------------------------------------------------------------------------------

class _Calls:
    """Stand-in for the library: records the entry points called and answers 0."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        return lambda *a: self.calls.append(name) or 0


@pytest.fixture()
def fake_cuda(monkeypatch):
    """tf_ops with its library replaced by _Calls and every tensor taken for a CUDA tensor, so each wrapper runs its own
    shape checks on the CPU."""
    T = importlib.import_module("3dssd_b200.tf_ops")
    fake = _Calls()
    monkeypatch.setattr(T, "lib", lambda: fake)
    monkeypatch.setattr(T, "_stream", lambda: None)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    return T, fake


def _f(*s):
    return torch.zeros(s, dtype=torch.float32)


def _i(*s):
    return torch.zeros(s, dtype=torch.int32)


def _conv(cin, cout):
    return P.FoldedConv(_f(cin, cout), _f(cout) + 1, _f(cout))


def test_new_entry_points_reject_cpu_and_malformed_operands():
    T = importlib.import_module("3dssd_b200.tf_ops")
    x = torch.zeros(1, 8, 3)
    with pytest.raises(ValueError, match="CUDA"):
        T.query_boxes_3d_points(16, x, torch.zeros(1, 2, 7))
    with pytest.raises(ValueError, match="CUDA"):
        T.region_pool(x, _f(1, 8, 4), _f(1, 8), _f(1, 2, 9), None, _conv(5, 8))
    with pytest.raises(ValueError, match="CUDA"):
        T.decode_bin_anchor_rows(_f(1, 2, 9), _f(1, 2, 52), _f(1, 2, 2))
    with pytest.raises(ValueError, match="CUDA"):
        T.bev_nms_counted(_f(1, 2, 7), _f(1, 2), _i(1), 0.1, 10)


def _good_and_bad(T):
    """(name, call) of well-formed operands, then of malformed ones, for the four new wrappers."""
    q = lambda *a: (lambda: T.query_boxes_3d_points(*a))
    pool = lambda xyz=None, feat=None, score=None, box=None, cnt=None, conv=None: (lambda: T.region_pool(
        _f(2, 8, 3) if xyz is None else xyz, _f(2, 8, 4) if feat is None else feat, _f(2, 8) if score is None else score,
        _f(2, 3, 9) if box is None else box, _i(2) if cnt is None else cnt, _conv(5, 8) if conv is None else conv))
    dec = lambda a=None, r=None, c=None, m=None: (lambda: T.decode_bin_anchor_rows(
        _f(2, 3, 9) if a is None else a, _f(2, 3, 52) if r is None else r, _f(2, 3, 2) if c is None else c, m))
    nms = lambda bx=None, sc=None, nv=None: (lambda: T.bev_nms_counted(
        _f(2, 5, 7) if bx is None else bx, _f(2, 5) if sc is None else sc, _i(2) if nv is None else nv, 0.1, 10))
    good = [("query", q(16, _f(2, 8, 3), _f(2, 3, 7))), ("pool", pool()), ("pool without count", lambda: T.region_pool(
        _f(2, 8, 3), _f(2, 8, 4), _f(2, 8), _f(2, 3, 7), None, _conv(5, 8))), ("decode", dec()),
        ("decode with mask", dec(m=_i(2, 3))), ("nms", nms())]
    bad = [("query: xyz rank", q(16, _f(8, 3), _f(2, 3, 7))), ("query: xyz width", q(16, _f(2, 8, 4), _f(2, 3, 7))),
           ("query: box width", q(16, _f(2, 8, 3), _f(2, 3, 9))), ("query: batch", q(16, _f(2, 8, 3), _f(1, 3, 7))),
           ("query: nsample", q(0, _f(2, 8, 3), _f(2, 3, 7))), ("query: dtype", q(16, _f(2, 8, 3).double(), _f(2, 3, 7))),
           ("pool: feature rows", pool(feat=_f(2, 7, 4))), ("pool: score shape", pool(score=_f(2, 8, 1))),
           ("pool: box width", pool(box=_f(2, 3, 6))), ("pool: box batch", pool(box=_f(1, 3, 9))),
           ("pool: count length", pool(cnt=_i(3))), ("pool: count dtype", pool(cnt=_f(2))),
           ("pool: 4-channel info conv", pool(conv=_conv(4, 8))), ("pool: scale length", pool(
               conv=P.FoldedConv(_f(5, 8), _f(7), _f(8)))), ("pool: xyz width", pool(xyz=_f(2, 8, 4))),
           ("decode: short pred_reg", dec(r=_f(2, 3, 51))), ("decode: one class", dec(c=_f(2, 3, 1))),
           ("decode: anchor width", dec(a=_f(2, 3, 6))), ("decode: rows", dec(r=_f(2, 4, 52))),
           ("decode: mask shape", dec(m=_i(2, 4))), ("decode: mask dtype", dec(m=_f(2, 3))),
           ("nms: n_valid length", nms(nv=_i(3))), ("nms: n_valid dtype", nms(nv=_f(2))), ("nms: n_valid rank", nms(nv=_i(2, 1))),
           ("nms: scores shape", nms(sc=_f(2, 4))), ("nms: box width", nms(bx=_f(2, 5, 6)))]
    return good, bad


def test_new_entry_points_check_shapes_before_any_launch(fake_cuda):
    T, fake = fake_cuda
    good, bad = _good_and_bad(T)
    for name, call in good:
        fake.calls.clear()
        call()
        assert len(fake.calls) == 1, "%s: %s" % (name, fake.calls)
    failures = []
    for name, call in bad:
        fake.calls.clear()
        try:
            call()
        except ValueError:
            if fake.calls:
                failures.append("%s: raised after calling %s" % (name, fake.calls))
            continue
        failures.append("%s: accepted (called %s)" % (name, fake.calls))
    assert not failures, "\n".join(failures)


POOL_SMEM_MAX = 227 * 1024           # the opt-in shared memory of one H100 CTA
POOL_MAX_N = 17706                   # the largest scene the pool takes at nsample 512 and c_info 128


def test_region_pool_shared_memory_limit():
    """The pool stages the scene's xyz in shared memory: at nsample 512 and c_info 128 it takes scenes of up to
    POOL_MAX_N points (tests/test_pointrcnn_rcnn_gpu.py runs that one), and one point more is rejected by the C ABI
    before any CUDA call, so also on a machine without a GPU."""
    pkg = importlib.import_module("3dssd_b200")
    L = pkg.lib()
    assert L.ssd3d_region_pool_smem(POOL_MAX_N, 512, 128) <= POOL_SMEM_MAX < L.ssd3d_region_pool_smem(POOL_MAX_N + 1, 512, 128)
    assert L.ssd3d_region_pool_smem(POOL_MAX_N, 512, 128) == (POOL_MAX_N * 3 + 7 * 128 + 8 * 512) * 4
    null = ctypes.c_void_p(None)
    pool = lambda n, p: L.ssd3d_region_pool(1, n, p, 512, 128, 128, *[null] * 4, 9, null, 1.0, 0.5, *[null] * 8)
    assert pool(POOL_MAX_N, 0) == 0                                         # accepted: no proposal, nothing to launch
    assert pool(POOL_MAX_N + 1, 0) == -1 and "shared memory" in L.ssd3d_last_error().decode()
    assert pool(POOL_MAX_N + 1, 100) == -1 and "shared memory" in L.ssd3d_last_error().decode()


def test_stage2_sa_route_plan():
    """rcnn_layer1 / rcnn_layer2 at inference, from parameter shapes alone: the tensor-core route (K = 64 is a pooling
    width of its epilogue) with the first conv hoisted (c = 256 + 3 at layer 1, 128 + 3 at layer 2) and unit lists; the
    ball query takes the exhaustive kernel (512 and 128 candidates, below tf_ops.BQ_GRID_MIN_N)."""
    L = importlib.import_module("3dssd_b200.layers_util")
    T = importlib.import_module("3dssd_b200.tf_ops")
    pp = P.prepare(P.init_rcnn_params(128), "cpu")
    for spec, c in zip(C.ARCH_POINTRCNN_RCNN[:2], (256, 128)):
        plan = L._route_plan(pp, spec[12], spec[3], spec[4], True, c, False, "tc", True, True, 2)
        assert plan.tc and plan.agg is None and plan.hoisted == [0] and plan.compact
        assert [sc.route for sc in plan.scales] == ["hoisted"]
    assert 64 in T.TC_POOL_WIDTHS and 512 < T.BQ_GRID_MIN_N
