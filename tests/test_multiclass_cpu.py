"""Several classes on the CPU (DESIGN.md section 3.17): the per-class NMS as the reference's class loop over the numpy
NMS oracle; the class-count oracle (tests/oracle_multiclass.py) against the reference's class targets
(tests/golden/multiclass_targets.npz) and against a float64 restatement of loss_builder.cls_loss with its autograd
gradient; the multi-class tf_ops wrappers' checks and C-call packing (pinned in tests/golden/multiclass_abi_trace.json,
recorded like tests/test_tf_ops_abi_cpu.py), the class-list checks and a three-class head's variables."""
import importlib
import json
import os

import numpy as np
import pytest
import torch

from oracle import det_loss as odl
from oracle import head as ohead
import oracle_multiclass as OM

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "multiclass_abi_trace.json")


def nms_classes(boxes, scores, thr, max_out):
    """postprocessor.py:49-120 on the numpy NMS oracle: per class c the NMS of scores[..., c] over the shared boxes,
    the kept rows concatenated class-major with column 8 = c, zero padded to C * max_out rows."""
    b, n, c = scores.shape
    blk = np.zeros((b, c * max_out, 9), np.float32)
    cnt = np.zeros((b,), np.int32)
    for k in range(c):
        bk, ck = ohead.bev_nms(boxes, np.ascontiguousarray(scores[..., k]), thr, max_out, k)
        for s in range(b):
            blk[s, cnt[s]:cnt[s] + ck[s]] = bk[s, :ck[s]]
            cnt[s] += ck[s]
    return blk, cnt


def _box(x, z, l=2.0, w=2.0):
    return np.array([x, 1.0, z, l, 1.5, w, 0.0], np.float32)


def test_nms_classes_hand_scenes():
    # box 0 and 1 overlap (IoU > 0.1), box 2 stands alone; 4 classes
    boxes = np.stack([_box(0, 0), _box(0.5, 0), _box(10, 10), _box(20, 20, 0.0)])[None]
    scores = np.array([[[0.9, 0.0, 0.5, 0.7],
                        [0.8, 0.0, 0.5, 0.2],
                        [0.1, 0.0, 0.5, 0.7],
                        [0.0, 0.0, 0.5, 0.1]]], np.float32)
    blk, cnt = nms_classes(boxes, scores, 0.1, 2)
    # class 0: 0 suppresses 1, then 2 -> fills max_output = 2
    assert blk[0, 0, 7] == np.float32(0.9) and blk[0, 1, 0] == 10 and list(blk[0, :2, 8]) == [0, 0]
    # class 1: every score equal (0): ties to the lower index -> boxes 0 and 2
    assert list(blk[0, 2:4, 0]) == [0, 10] and list(blk[0, 2:4, 8]) == [1, 1]
    # class 2: equal scores across classes, same decisions as class 1
    assert np.array_equal(blk[0, 4:6, :8], np.stack([np.r_[_box(0, 0), 0.5], np.r_[_box(10, 10), 0.5]]))
    # class 3: boxes 0 and 2 tie at 0.7; box 0 is kept in classes 0..3
    assert list(blk[0, 6:8, 0]) == [0, 10] and cnt[0] == 8 and np.all(blk[0, :, 8] == np.repeat(np.arange(4), 2))
    # a class whose candidates are all suppressed but the first keeps exactly one row; the tail stays zero
    one = nms_classes(np.stack([_box(0, 0), _box(0.1, 0)])[None], np.array([[[1.0], [0.5]]], np.float32), 0.1, 5)
    assert one[1][0] == 1 and not one[0][0, 1:].any()


def test_nms_classes_at_one_class_is_the_single_nms():
    rng = np.random.default_rng(1)
    boxes = np.concatenate([rng.uniform(-8, 8, (2, 200, 3)), rng.uniform(0.5, 4, (2, 200, 3)), rng.uniform(-3, 3, (2, 200, 1))],
                           -1).astype(np.float32)
    sc = rng.uniform(0, 1, (2, 200)).astype(np.float32)
    blk, cnt = nms_classes(boxes, sc[..., None], 0.1, 100)
    eb, ec = ohead.bev_nms(boxes, sc, 0.1, 100)
    assert np.array_equal(blk, eb) and np.array_equal(cnt, ec)


FACE_TOL = 1e-4     # points nearer a face than this may land on either side of it after a float32 rounding


@pytest.fixture(scope="module")
def golden_mc():
    return dict(np.load(os.path.join(HERE, "golden", "multiclass_targets.npz")))


def test_multiclass_golden_holds_every_class_and_an_out_of_list_label(golden_mc):
    z = golden_mc
    pos = z["pmask"] > 0
    for k in (1, 2, 3, 4):
        assert (pos & (z["assigned_label"] == k)).sum() >= 10, k
    assert not z["cls_label"][pos & (z["assigned_label"] == 4)].any()


def test_oracle_class_targets_match_the_reference(golden_mc):
    """The class-count oracle at C = 3 against the reference's mask assignment and its one_hot(label - 1) x centre-ness
    classification target (tests/golden/make_golden_multiclass.py): the class-agnostic targets equal the reference's,
    every class column matches, and a label of 4 gives a zero row on a point that stays a positive."""
    z = golden_mc
    t = OM.assign(z["base_xyz"], z["vote_base"], z["gt_boxes"], z["gt_labels"], 3)
    far = z["face_dist"] > FACE_TOL
    for k in ("assigned_idx", "pmask", "nmask"):
        np.testing.assert_array_equal(t[k][far], z[k][far], err_msg=k)
    assert t["cls_label"].shape == z["cls_label"].shape == z["pmask"].shape + (3,)
    np.testing.assert_array_equal(t["cls_label"][far] > 0, z["one_hot"][far] > 0)
    np.testing.assert_allclose(t["cls_label"][far], z["cls_label"][far], rtol=2e-6, atol=1e-7)   # float32 vs float64
    out = far & (z["pmask"] > 0) & (z["assigned_label"] == 4)
    assert out.any() and (t["pmask"][out] == 1).all() and not t["cls_label"][out].any()


def test_oracle_one_class_path_is_the_single_class_oracle(golden_mc):
    z = golden_mc
    one = odl.assign(z["base_xyz"], z["vote_base"], z["gt_boxes"], z["gt_labels"])
    t = OM.assign(z["base_xyz"], z["vote_base"], z["gt_boxes"], z["gt_labels"], 1)
    for k in one:
        got = t[k][..., 0] if k == "cls_label" else t[k]
        assert np.array_equal(np.asarray(got).view(np.uint8), np.asarray(one[k]).view(np.uint8)), k


def loss_builder_cls_loss(pred_cls, gt_label, pmask, nmask, centerness, c):
    """LossBuilder.cls_loss for a sigmoid 'Center-ness' head (loss_builder.py:58-96) in float64 torch, op for op:
    gt_cls = one_hot(label - 1, C) * centre-ness, sigmoid_cross_entropy_with_logits, reduce_mean over the classes,
    reduce_sum(loss * cls_mask) / max(1, reduce_sum(cls_mask)).  Differentiable w.r.t. pred_cls."""
    cm = pmask + nmask
    norm = torch.clamp_min(cm.sum(), 1.0)
    onehot = torch.nn.functional.one_hot(torch.where((gt_label >= 1) & (gt_label <= c), gt_label - 1, c), c + 1)[..., :c]
    gt = onehot.double() * centerness[..., None]
    loss = torch.nn.functional.binary_cross_entropy_with_logits(pred_cls, gt, reduction="none").mean(-1)
    return (loss * cm).sum() / norm


@pytest.mark.parametrize("c", [1, 2, 3, 8])
def test_oracle_cls_loss_and_gradient_match_loss_builder(c):
    """The class-count oracle's classification loss and its gradient (the recipe of ssd3d_det_loss_classes /
    _grad_classes) against the float64 restatement of loss_builder.cls_loss and torch autograd of it; the other five
    losses and the norms are the single-class oracle's, and at C = 1 so is the classification loss."""
    rng = np.random.default_rng(c)
    B, N, NV = 2, 60, 10
    pm = (rng.uniform(size=(B, N)) < 0.4).astype(np.float32)
    nm = ((rng.uniform(size=(B, N)) < 0.7) & (pm == 0)).astype(np.float32)
    lab = np.where(pm > 0, rng.integers(1, c + 2, (B, N)), 0)                   # c + 1: a label outside the list
    ctr = np.where(pm > 0, rng.uniform(0.01, 1.0, (B, N)), 0.0).astype(np.float32)
    z = np.where((lab[..., None] - 1) == np.arange(c), ctr[..., None], 0).astype(np.float32)
    box = np.concatenate([rng.uniform(-5, 5, (B, N, 3)), rng.uniform(1, 3, (B, N, 3)), rng.uniform(-3, 3, (B, N, 1))], -1)
    tg = dict(pmask=pm, nmask=nm, cls_label=z, assigned_box=box.astype(np.float32), angle_bin=rng.integers(0, 12, (B, N)).astype(np.int32),
              angle_res=rng.uniform(-0.5, 0.5, (B, N)).astype(np.float32), offset_target=np.zeros((B, N, 6), np.float32),
              vote_mask=(rng.uniform(size=(B, NV)) < 0.5).astype(np.float32), vote_target=rng.normal(size=(B, NV, 3)).astype(np.float32))
    base = rng.uniform(-5, 5, (B, N, 3)).astype(np.float32)
    x = (3 * rng.standard_normal((B, N, c))).astype(np.float32)
    heads = [rng.normal(size=(B, N, k)).astype(np.float32) for k in (6, 12, 12)]
    vo = rng.normal(size=(B, NV, 3)).astype(np.float32)
    loss, norm = OM.losses(base, x, *heads, vo, tg, c)
    xt = torch.tensor(x, dtype=torch.float64, requires_grad=True)
    ref = loss_builder_cls_loss(xt, torch.as_tensor(lab), torch.as_tensor(pm, dtype=torch.float64),
                                torch.as_tensor(nm, dtype=torch.float64), torch.as_tensor(ctr, dtype=torch.float64), c)
    (gref,) = torch.autograd.grad(ref * 1.5, [xt])
    assert abs(loss[0] - ref.item()) <= 1e-12 * max(1.0, abs(ref.item()))
    np.testing.assert_allclose(OM.cls_grad(x, tg, c, 1.5, norm[0]), gref.numpy(), rtol=1e-10, atol=1e-15)
    one, one_norm = odl.losses(base, x[..., :1], *heads, vo, dict(tg, cls_label=z[..., 0]))
    assert np.array_equal(loss[1:], one[1:]) and np.array_equal(norm, one_norm)
    if c == 1:
        assert loss[0] == one[0]


# ---- the wrappers: checks before any launch and the C-call packing ---------------------------------------------------

def _abi():
    return importlib.import_module("test_tf_ops_abi_cpu")


@pytest.fixture()
def abi(monkeypatch):
    A = _abi()
    T = importlib.import_module("3dssd_b200.tf_ops")
    fake = A._FakeLib()
    monkeypatch.setattr(T, "lib", lambda: fake)
    monkeypatch.setattr(T, "_stream", lambda: A._STREAM)
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    return T, fake, A


def test_multiclass_abi_trace(abi):
    T, fake, A = abi
    rec = A._Recorder(fake)
    f, i = A._f, A._i
    blk, bc = f(2, 15, 9), i(2)
    rec("bev_nms_classes", T.bev_nms, f(2, 30, 7), f(2, 30, 3), 0.1, 5, cls_num=3)
    rec("bev_nms_classes_out", T.bev_nms, f(2, 30, 7), f(2, 30, 3), 0.1, 5, out=(blk, bc), cls_num=3)
    rec("decode_classes", T.decode_dist_anchor_free, f(2, 20, 3), f(2, 20, 30), f(2, 20, 3), cls_num=3)
    b, n, nv, g = 2, 12, 10, 4
    base = f(b, n, 3)
    tg = rec("det_assign_classes", T.det_assign, base, f(b, nv, 3), f(b, g, 7), i(b, g), cls_num=3)
    reg, cls, vo = f(b, n, 1, 30), f(b, n, 1, 3), f(b, nv, 8)[..., 2:5]
    rec("det_loss_classes", T.det_loss, base, cls, reg[..., :6], reg[..., 6:18], reg[..., 18:], vo, tg, cls_num=3)
    rec("det_loss_grad_classes", T.det_loss_grad, base, cls, reg[..., :6], reg[..., 6:18], reg[..., 18:], vo, tg, f(6), f(3),
        cls_num=3)

    def det_fb(base, reg, cls, vo, go):
        loss = T.det_loss_train(base, cls, reg[..., :6], reg[..., 6:18], reg[..., 18:], vo, tg, cls_num=3)
        return (loss,) + torch.autograd.grad(loss, [base, reg, cls, vo], go)

    leaf = lambda *s: f(*s).requires_grad_()
    rec("det_loss_train_classes", det_fb, leaf(b, n, 3), leaf(b, n, 1, 30), leaf(b, n, 1, 3), leaf(b, nv, 3), f(6))
    got = json.loads(json.dumps(rec.trace))
    path = os.environ.get("SSD3D_RECORD_MULTICLASS_ABI")
    if path:
        with open(path, "w") as fh:
            json.dump(got, fh, indent=0, sort_keys=True)
        return
    with open(GOLDEN) as fh:
        exp = json.load(fh)
    assert sorted(got) == sorted(exp)
    for case in sorted(exp):
        assert got[case] == exp[case], case


def test_multiclass_wrappers_reject_malformed_input(abi):
    T, fake, A = abi
    f, i = A._f, A._i
    b, n, nv, g = 2, 12, 10, 4
    tg = T.det_assign(f(b, n, 3), f(b, nv, 3), f(b, g, 7), i(b, g), cls_num=3)
    reg, vo = f(b, n, 1, 30), f(b, nv, 3)
    loss = lambda cls, c, t=tg: T.det_loss(f(b, n, 3), cls, reg[..., :6], reg[..., 6:18], reg[..., 18:], vo, t, cls_num=c)
    cases = {
        "nms_width": lambda: T.bev_nms(f(2, 30, 7), f(2, 30, 2), 0.1, 5, cls_num=3),
        "nms_flat_scores": lambda: T.bev_nms(f(2, 30, 7), f(2, 30), 0.1, 5, cls_num=1),
        "nms_c0": lambda: T.bev_nms(f(2, 30, 7), f(2, 30, 0), 0.1, 5, cls_num=0),
        "nms_c9": lambda: T.bev_nms(f(2, 30, 7), f(2, 30, 9), 0.1, 5, cls_num=9),
        "nms_bool": lambda: T.bev_nms(f(2, 30, 7), f(2, 30, 1), 0.1, 5, cls_num=True),
        "nms_block_rows": lambda: T.bev_nms(f(2, 30, 7), f(2, 30, 3), 0.1, 5, out=(f(2, 5, 9), i(2)), cls_num=3),
        "nms_block_cols": lambda: T.bev_nms(f(2, 30, 7), f(2, 30, 3), 0.1, 5, out=(f(2, 15, 8), i(2)), cls_num=3),
        "decode_width": lambda: T.decode_dist_anchor_free(f(2, 20, 3), f(2, 20, 30), f(2, 20, 4), cls_num=3),
        "decode_c9": lambda: T.decode_dist_anchor_free(f(2, 20, 3), f(2, 20, 30), f(2, 20, 9), cls_num=9),
        "assign_c0": lambda: T.det_assign(f(b, n, 3), f(b, nv, 3), f(b, g, 7), i(b, g), cls_num=0),
        "assign_label_dtype": lambda: T.det_assign(f(b, n, 3), f(b, nv, 3), f(b, g, 7), i(b, g).long(), cls_num=3),
        "assign_label_float": lambda: T.det_assign(f(b, n, 3), f(b, nv, 3), f(b, g, 7), f(b, g), cls_num=3),
        "loss_width": lambda: loss(f(b, n, 1, 2), 3),
        "loss_c9": lambda: loss(f(b, n, 1, 9), 9),
        "loss_label_shape": lambda: loss(f(b, n, 1, 2), 2),
        "loss_label_dtype": lambda: loss(f(b, n, 1, 3), 3, dict(tg, cls_label=tg["cls_label"].double())),
        "grad_width": lambda: T.det_loss_grad(f(b, n, 3), f(b, n, 1, 2), reg[..., :6], reg[..., 6:18], reg[..., 18:], vo, tg,
                                              f(6), f(3), cls_num=3),
    }
    failures = []
    for name, op in cases.items():
        fake.calls.clear()
        try:
            op()
        except ValueError:
            if fake.calls:
                failures.append("%s: raised after calling %s" % (name, [c[0] for c in fake.calls]))
            continue
        failures.append("%s: accepted" % name)
    assert not failures, "\n".join(failures)


# ---- names, import and tools -----------------------------------------------------------------------------------------

def test_class_list_checks():
    C = importlib.import_module("3dssd_b200.config")
    assert C.CLS_LIST == ("Car",)
    assert C.check_cls_list("Car, Pedestrian,Cyclist") == ("Car", "Pedestrian", "Cyclist")
    assert C.check_cls_list(list(C.CLASS_MEAN_SIZE)) == tuple(C.CLASS_MEAN_SIZE)
    for bad in ("Car,Bus", "Car,Car", "", list(C.CLASS_MEAN_SIZE) + ["Car"], "car"):
        with pytest.raises(ValueError):
            C.check_cls_list(bad)


@pytest.mark.parametrize("tool,extra", [("train.py", ["--steps", "1"]), ("eval_kitti.py", ["--samples", "x", "--labels", "y",
                                                                                               "--weights", "z"]),
                                         ("prepare_kitti.py", None), ("build_mixup_db.py", ["--out", "x.npz", "--synthetic", "1"])])
def test_tools_reject_bad_class_lists(tool, extra):
    import subprocess
    import sys
    root = os.path.dirname(HERE)
    if extra is None:
        extra = ["--root", "x", "--list", "y", "--out", "z"]
    r = subprocess.run([sys.executable, os.path.join(root, "tools", tool)] + extra + ["--classes", "Car,Truck,Car"],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode != 0 and "class" in (r.stdout + r.stderr).lower(), r.stdout[-2000:] + r.stderr[-2000:]


def test_three_class_head_variables_and_import():
    P = importlib.import_module("3dssd_b200.params")
    io = importlib.import_module("3dssd_b200.kitti_io")
    H = importlib.import_module("3dssd_b200.head")
    d = P.init_head_params(512, cls_channels=3, seed=4)
    assert d["pred_cls/weights"].shape == (128, 3) and d["pred_cls/biases"].shape == (3,)
    assert d["pred_reg/weights"].shape == (128, 30) and d["conv1d_0/weights"].shape == (512, 128)
    tf = {k + ":0": (v.reshape((1,) + v.shape) if k.endswith("/weights") else v) for k, v in d.items()}
    back = io.params_from_tf_variables(tf)
    assert np.asarray(back["pred_cls/weights"]).reshape(-1, 3).shape == (128, 3)
    head = H.DetectionHead(params=back, device="cpu")
    assert head.cls_num == 3 and head.max_output == 300
    with pytest.raises(ValueError):
        H.DetectionHead(params=back, device="cpu", cls_num=2)
    assert H.DetectionHead(params=P.init_head_params(512, seed=4), device="cpu").max_output == 100
