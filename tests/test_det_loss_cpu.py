"""Targets and detection losses without a GPU: the numpy oracle of csrc/det_loss.cu (oracle/det_loss.py) against the
reference's own numpy target functions (tests/golden/det_targets.npz, make_golden_det_targets.py), the float64 loss of a
literal restatement of the TF graph against the oracle, and the host-side helpers (label padding, synthetic boxes, the
constants of loss.py against the kernel's)."""
import os
import re

import numpy as np
import pytest
import torch

from oracle import det_loss as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "det_targets.npz")
FACE_TOL = 1e-4     # points nearer a face than this may land on either side of it after a float32 rounding


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


@pytest.fixture(scope="module")
def oracle_targets(golden):
    return O.assign(golden["base_xyz"], golden["vote_base"], golden["gt_boxes"], golden["gt_labels"])


def test_golden_holds_the_edge_cases(golden):
    z = golden
    assert (z["face_dist"] == 0).sum() >= 10                                          # points exactly on faces
    assert ((z["pmask"] == 0) & (z["nmask"] == 0)).sum() >= 1                        # inside but beyond 10 m
    near = z["vote_face_dist"] < 0.1
    assert (z["vote_mask"][near] == 1).any()
    per = 2 * np.pi / 12
    ry = z["gt_boxes"][..., 6][np.any(z["gt_boxes"] != 0, -1)]
    assert np.isclose(np.abs(ry), np.float32(np.pi)).any() and np.isclose(ry, np.float32(per / 2)).any()
    assert not np.any(z["gt_boxes"][-1]) and (z["nmask"][-1] == 1).all() and not z["vote_mask"][-1].any()
    assert (z["gt_labels"] == 2).any()                                               # a box of another class


def test_oracle_matches_reference_targets(golden, oracle_targets):
    z, t = golden, oracle_targets
    far, vfar = z["face_dist"] > FACE_TOL, z["vote_face_dist"] > FACE_TOL
    for k in ("assigned_idx", "pmask", "nmask"):
        np.testing.assert_array_equal(t[k][far], z[k][far], err_msg=k)
    np.testing.assert_array_equal(t["vote_mask"][vfar], z["vote_mask"][vfar])
    np.testing.assert_array_equal(t["angle_bin"], z["angle_bin"])
    np.testing.assert_allclose(t["angle_res"], z["angle_res"], atol=1e-6)            # TF's float32 formula vs numpy's float64
    enc = np.concatenate([z["encoded_ctr"], z["encoded_half"]], -1)
    assert np.array_equal(t["offset_target"][far].view(np.uint32), enc[far].view(np.uint32))
    assert np.array_equal(t["vote_target"][vfar].view(np.uint32), z["vote_target"][vfar].view(np.uint32))
    bx = t["assigned_box"].reshape(-1, 7).astype(np.float64)
    gc = O.corners(bx[:, :3], bx[:, 3:6], bx[:, 6]).reshape(z["corners"].shape)
    np.testing.assert_allclose(gc[:-1], z["corners"][:-1], atol=2e-5)
    assert np.isfinite(t["cls_label"]).all() and (t["cls_label"][t["pmask"] == 0] == 0).all()


def test_face_test_is_strict(golden, oracle_targets):
    """A point exactly on a face (axis-aligned box, exact corners) is outside: sign >= 0."""
    on = golden["face_dist"] == 0
    assert on.any()
    assert (oracle_targets["assigned_idx"][on] == golden["assigned_idx"][on]).all()
    n, d = O.box_planes(np.array([0, 0, 0, 2, 1, 2, 0], np.float32))
    assert not O.inside(np.array([[1.0, -0.5, 0.0]], np.float32), n, d)[0]
    assert O.inside(np.array([[0.999, -0.5, 0.0]], np.float32), n, d)[0]


def tf_graph_losses(base_xyz, pred_cls, pred_offset, pred_angle_cls, pred_angle_res, vote_offset, tg, nbins=12):
    """float64 torch restatement of the TF graph (single_stage_detector.train_forward, EncoderDecoder.encode,
    LossBuilder.forward) on given targets.  TF's tie rules are written as explicit masks: tf.minimum / tf.maximum route a
    tie to their first input, torch's split it evenly.  Returns the six losses (6,)."""
    d = lambda t: torch.as_tensor(np.asarray(t), dtype=torch.float64)
    pm, nm = d(tg["pmask"]), d(tg["nmask"])
    box = d(tg["assigned_box"])

    def huber(e):
        a = e.abs()
        q = torch.where(a <= 1.0, a, torch.ones_like(a))                     # tf.minimum(abs, delta)
        return 0.5 * q ** 2 + (a - q)

    def tmin(a, b):
        return torch.where(a <= b, a, b)

    def tmax(a, b):
        return torch.where(a >= b, a, b)

    # classification with the centre-ness label (loss_builder.py:56-137); base_xyz under tf.stop_gradient
    bx = base_xyz.detach()
    ab = box * pm[..., None]
    e = bx - ab[..., :3]
    ry = ab[..., 6]
    c, s = torch.cos(ry), torch.sin(ry)
    cx, cy, cz = c * e[..., 0] - s * e[..., 2], e[..., 1], s * e[..., 0] + c * e[..., 2]
    fr, bk = ab[..., 3] / 2 - cx, cx + ab[..., 3] / 2
    bo, tp = -cy, cy + ab[..., 4]
    le, ri = ab[..., 5] / 2 - cz, cz + ab[..., 5] / 2
    safe = pm > 0                                             # the reference's 0/0 of a negative is multiplied by gt_cls 0
    r = lambda a, b: torch.where(safe, tmin(a, b) / torch.where(safe, tmax(a, b), torch.ones_like(a)), torch.zeros_like(a)) * pm
    ctr = torch.pow(tmax(r(fr, bk) * r(bo, tp) * r(le, ri), torch.full_like(fr, 1e-6)), 1 / 3.0)
    lab = torch.as_tensor(np.asarray(tg["gt_cls"]), dtype=torch.float64) * pm
    z = (lab == 1).double() * ctr
    x = pred_cls[..., 0]
    cm = pm + nm
    cls = ((torch.clamp_min(x, 0) - x * z + torch.log1p(torch.exp(-x.abs()))) * cm).sum() / tmax(cm.sum(), d(1.0))
    norm = tmax(pm.sum(), d(1.0))
    # encode (anchor_encoder.py:151-173): the translation target depends on base_xyz
    half = box[..., 3:6] / 2
    enc = torch.stack([box[..., 0] - base_xyz[..., 0], box[..., 1] - half[..., 1] - base_xyz[..., 1],
                       box[..., 2] - base_xyz[..., 2]], -1)
    target = torch.cat([enc, half], -1)
    off = pred_offset.reshape(target.shape)
    offset = (huber(off - target).sum(-1) * pm).sum() / norm
    lg = pred_angle_cls.reshape(*pm.shape, nbins)
    rs = pred_angle_res.reshape(*pm.shape, nbins)
    onehot = torch.nn.functional.one_hot(torch.as_tensor(np.asarray(tg["angle_bin"]), dtype=torch.long), nbins).double()
    bin_loss = ((torch.logsumexp(lg, -1) - (lg * onehot).sum(-1)) * pm).sum() / norm
    res = (rs * onehot).sum(-1)
    res_loss = huber((res - d(tg["angle_res"])) * pm).sum() / norm
    # corner loss: decode with the GT bin (anchor_decoder.py:86-112), corners (box_3d_utils.py:89-130)
    interval = float(np.float32(2 * np.pi / nbins))
    ang = (torch.as_tensor(np.asarray(tg["angle_bin"]), dtype=torch.float64) + res) * interval
    pc = base_xyz + off[..., :3]
    pc = pc + torch.stack([torch.zeros_like(off[..., 4]), off[..., 4], torch.zeros_like(off[..., 4])], -1)
    two = off[..., 3:6] * 2
    lhw = tmax(two, torch.full_like(two, float(np.float32(0.1))))

    def corners(ctr3, size, a):
        sx = d([1, 1, -1, -1, 1, 1, -1, -1])
        sz = d([1, -1, -1, 1, 1, -1, -1, 1])
        xc = sx * size[..., :1] / 2
        yc = torch.cat([torch.zeros_like(size[..., 1:2]).expand(*size.shape[:-1], 4), -size[..., 1:2].expand(*size.shape[:-1], 4)], -1)
        zc = sz * size[..., 2:3] / 2
        cc, ss = torch.cos(a)[..., None], torch.sin(a)[..., None]
        return torch.stack([cc * xc + ss * zc + ctr3[..., :1], yc + ctr3[..., 1:2], -ss * xc + cc * zc + ctr3[..., 2:3]], -1)

    corner = (huber(corners(pc, lhw, ang) - corners(box[..., :3], box[..., 3:6], box[..., 6])).sum((-1, -2)) * pm).sum() / norm
    vm = d(tg["vote_mask"])
    vote = (huber(d(tg["vote_target"]) - vote_offset).sum(-1) * vm).sum() / tmax(vm.sum(), d(1.0))
    return torch.stack([cls, offset, bin_loss, res_loss, corner, vote])


def random_preds(rng, b, n, nv, nbins=12, scale=1.0):
    """Head outputs as box_regression_head returns them (float32 numpy): cls (b, n, 1), offset (b, n, 1, 6) with some
    half sizes on the 0.05 floor, angle logits / residuals (b, n, 1, nbins), raw vote offsets (b, nv, 3)."""
    cls = (rng.standard_normal((b, n, 1)) * 2 * scale).astype(np.float32)
    off = (rng.standard_normal((b, n, 1, 6)) * scale).astype(np.float32)
    off[..., 3:6] = np.abs(off[..., 3:6]) + 0.3
    off[:, ::17, 0, 3] = np.float32(0.05)                     # 2 * half == 0.1: the tie of tf.maximum
    off[:, ::13, 0, 5] = np.float32(0.01)                     # below the floor
    acls = rng.standard_normal((b, n, 1, nbins)).astype(np.float32)
    ares = (rng.standard_normal((b, n, 1, nbins)) * 0.5).astype(np.float32)
    vote = (rng.standard_normal((b, nv, 3)) * 1.5 * scale).astype(np.float32)
    return cls, off, acls, ares, vote


def with_gt_cls(tg, gt_labels):
    out = dict(tg)
    out["gt_cls"] = np.take_along_axis(gt_labels, tg["assigned_idx"].astype(np.int64), 1) if gt_labels.shape[1] else \
        np.zeros_like(tg["assigned_idx"])
    return out


def test_tf_graph_restatement_agrees_with_oracle(golden, oracle_targets):
    rng = np.random.default_rng(5)
    z = golden
    b, n = z["base_xyz"].shape[:2]
    preds = random_preds(rng, b, n, z["vote_base"].shape[1])
    tg = with_gt_cls(oracle_targets, z["gt_labels"])
    want, norm = O.losses(z["base_xyz"], *preds, oracle_targets)
    t = [torch.tensor(p, dtype=torch.float64, requires_grad=True) for p in (z["base_xyz"],) + preds]
    got = tf_graph_losses(*t, tg)
    np.testing.assert_allclose(got.detach().numpy(), want, rtol=1e-8)     # the oracle's centre-ness label is float32
    assert norm[1] == oracle_targets["pmask"].sum() and norm[2] == oracle_targets["vote_mask"].sum()
    got.sum().backward()
    for x in t:
        assert torch.isfinite(x.grad).all()
    neg = oracle_targets["pmask"] == 0
    assert (t[0].grad.numpy()[neg] == 0).all()               # a non-positive point: no corner / offset gradient


def test_make_label_batch_pads_with_zeros(pkg):
    samples = [{"label_boxes_3d": np.arange(14, dtype=np.float32).reshape(2, 7) + 1, "label_classes": np.array([1, 1])},
               {"label_boxes_3d": np.zeros((0, 7), np.float32), "label_classes": np.zeros((0,), np.int64)},
               {"label_boxes_3d": np.ones((3, 7), np.float32), "label_classes": np.array([1, 2, 1])}]
    boxes, labels = pkg.kitti_io.make_label_batch(samples)
    assert boxes.shape == (3, 3, 7) and boxes.dtype == np.float32 and labels.shape == (3, 3) and labels.dtype == np.int32
    np.testing.assert_array_equal(boxes[0, :2], samples[0]["label_boxes_3d"])
    assert not boxes[0, 2].any() and not boxes[1].any() and not labels[1].any()
    np.testing.assert_array_equal(labels, [[1, 1, 0], [0, 0, 0], [1, 2, 1]])
    empty_b, empty_l = pkg.kitti_io.make_label_batch(samples[1:2])
    assert empty_b.shape == (1, 0, 7) and empty_l.shape == (1, 0)


def test_synthetic_scenes_with_boxes(pkg):
    synth = __import__("importlib").import_module("3dssd_b200.synth")
    pts, boxes, labels = synth.kitti_like_with_boxes(3, 4096, 40, seed=3)
    assert pts.shape == (3, 4096, 4) and boxes.shape == (3, 40, 7) and labels.shape == (3, 40) and labels.dtype == np.int32
    valid = np.any(boxes != 0, -1)
    assert ((labels == 1) == valid).all() and (~valid).any()
    ry = boxes[..., 6][valid]
    assert np.isclose(np.abs(ry), np.pi).any()
    edges = np.arange(12) * (np.pi / 6) - np.pi / 12
    assert np.isclose(ry[:, None], edges[None]).any()
    t = O.assign(pts[:, ::16, :3], pts[:, 1::16, :3], boxes, labels)
    assert t["pmask"].sum() > 0 and t["vote_mask"].sum() > 0


def test_loss_constants_match_the_kernel(pkg):
    src = open(os.path.join(ROOT, "3dssd_b200", "csrc", "det_loss.cu")).read()
    val = lambda name: float(re.search(r"\b%s = ([0-9.e-]+)f?;" % name, src).group(1))
    L = pkg.loss
    assert val("kExpand") == L.EXPAND_DIMS_LENGTH and val("kSampleRange") == L.SOFTMAX_SAMPLE_RANGE
    assert val("kCtrEps") == L.CENTER_NESS_EPS and L.CENTER_NESS_LABEL_RANGE == (0.0, 1.0)
    assert L.ANGLE_CLS_NUM == pkg.head.ANGLE_CLS_NUM
