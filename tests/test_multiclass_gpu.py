"""Several classes on the GPU (-m gpu, DESIGN.md section 3.17): the per-class NMS cluster kernel against C calls of the
single-class NMS, the class forms of the decode, the target assignment and the losses against the single-class kernels
and float64, three-class inference and training end to end, and the class column through the KITTI evaluator."""
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import oracle_multiclass as OM

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
synth = importlib.import_module("3dssd_b200.synth")
CLS3 = ("Car", "Pedestrian", "Cyclist")


def _scene(rng, b, n, c, spread=None):
    """Clustered boxes (so that the NMS suppresses) and per-class scores with ties inside and across the classes."""
    spread = spread if spread is not None else max(4.0, np.sqrt(n) * 0.8)
    ctr = rng.uniform(-spread, spread, (b, n, 3)).astype(np.float32)
    lhw = rng.uniform(0.5, 4.5, (b, n, 3)).astype(np.float32)
    ry = rng.uniform(-np.pi, np.pi, (b, n, 1)).astype(np.float32)
    boxes = np.concatenate([ctr, lhw, ry], -1)
    scores = rng.uniform(0, 1, (b, n, c)).astype(np.float32)
    scores[:, 5:9] = scores[:, 4:5]                                  # ties within a class
    if c > 1:
        scores[:, 20:40, 1] = scores[:, 20:40, 0]                    # equal scores across classes
    return boxes, scores


def _per_class(pkg, boxes, scores, thr, max_out):
    """The reference's class loop: one single-class NMS per class on the shared boxes, concatenated in class order."""
    b, n, c = scores.shape
    blk = torch.zeros((b, c * max_out, 9), dtype=torch.float32, device=boxes.device)
    cnt = torch.zeros((b,), dtype=torch.int32, device=boxes.device)
    for k in range(c):
        bk, ck = pkg.tf_ops.bev_nms(boxes, scores[..., k].contiguous(), thr, max_out, cls_id=k)
        for s in range(b):
            m = int(ck[s])
            blk[s, int(cnt[s]):int(cnt[s]) + m] = bk[s, :m]
            cnt[s] += m
    return blk, cnt


def _bits(t):
    return t.detach().cpu().contiguous().view(torch.int32).numpy() if t.dtype == torch.float32 else t.detach().cpu().numpy()


@pytest.mark.parametrize("c", [1, 2, 3, 8])
def test_bev_nms_classes_equals_the_class_loop(pkg, cuda, c):
    rng = np.random.default_rng(c)
    for b in (1, 8):
        for n in (64, 256, 513, 4096, 16384):
            boxes, scores = (torch.from_numpy(a).to(cuda) for a in _scene(rng, b, n, c))
            got_b, got_c = pkg.tf_ops.bev_nms(boxes, scores, 0.1, 100, cls_num=c)
            exp_b, exp_c = _per_class(pkg, boxes, scores, 0.1, 100)
            assert np.array_equal(_bits(got_c), _bits(exp_c)), (b, n)
            assert np.array_equal(_bits(got_b), _bits(exp_b)), (b, n)
            if c == 1:
                sb, sc = pkg.tf_ops.bev_nms(boxes, scores[..., 0].contiguous(), 0.1, 100)
                assert np.array_equal(_bits(got_b), _bits(sb)) and np.array_equal(_bits(got_c), _bits(sc))
            for s in range(b):
                assert not got_b[s, int(got_c[s]):].any()
    # degenerate boxes are never suppressed: every class fills max_output, and a box is kept in all three classes
    boxes, scores = _scene(rng, 2, 300, 3, spread=200.0)
    boxes[:, :, 3] = np.where(np.arange(300) % 2 == 0, boxes[:, :, 3], 0.0)
    bt, st = torch.from_numpy(boxes).to(cuda), torch.from_numpy(scores).to(cuda)
    got_b, got_c = pkg.tf_ops.bev_nms(bt, st, 0.1, 10, cls_num=3)
    exp_b, exp_c = _per_class(pkg, bt, st, 0.1, 10)
    assert np.array_equal(_bits(got_b), _bits(exp_b)) and np.array_equal(_bits(got_c), _bits(exp_c))
    assert int(got_c.max()) == 30                                     # every class fills max_output


def test_bev_nms_classes_graph_replay_and_largest_launch(pkg, cuda):
    rng = np.random.default_rng(11)
    boxes, scores = (torch.from_numpy(a).to(cuda) for a in _scene(rng, 8, 16384, 8))
    eager = [t.clone() for t in pkg.tf_ops.bev_nms(boxes, scores, 0.1, 100, cls_num=8)]
    out = (torch.empty((8, 800, 9), dtype=torch.float32, device=cuda), torch.empty((8,), dtype=torch.int32, device=cuda))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        pkg.tf_ops.bev_nms(boxes, scores, 0.1, 100, out=out, cls_num=8)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        pkg.tf_ops.bev_nms(boxes, scores, 0.1, 100, out=out, cls_num=8)
    out[0].fill_(7.0)
    out[1].fill_(-1)
    g.replay()
    torch.cuda.synchronize()
    assert np.array_equal(_bits(out[0]), _bits(eager[0])) and np.array_equal(_bits(out[1]), _bits(eager[1]))


def test_decode_classes(pkg, cuda):
    rng = np.random.default_rng(3)
    ctr = torch.from_numpy(rng.uniform(-30, 30, (4, 500, 3)).astype(np.float32)).to(cuda)
    reg = torch.from_numpy(rng.standard_normal((4, 500, 30)).astype(np.float32)).to(cuda)
    for c in (1, 2, 3, 8):
        cls = torch.from_numpy((4 * rng.standard_normal((4, 500, c))).astype(np.float32)).to(cuda)
        boxes, scores = pkg.tf_ops.decode_dist_anchor_free(ctr, reg, cls, 12, cls_num=c)
        assert tuple(scores.shape) == (4, 500, c)
        for k in range(c):
            b1, s1 = pkg.tf_ops.decode_dist_anchor_free(ctr, reg, cls[..., k:k + 1].contiguous(), 12)
            assert np.array_equal(_bits(boxes), _bits(b1)) and np.array_equal(_bits(scores[..., k].contiguous()), _bits(s1))


def _targets_case(rng, b=3, n=512, nv=600, g=12):
    pts, boxes, labels = synth.kitti_like_multiclass(b, 4096, g, CLS3, seed=int(rng.integers(1 << 20)))
    labels[:, 1] = np.where(labels[:, 1] > 0, 4, 0)                   # a label outside 1..3: a positive with a zero row
    sel = lambda m: np.stack([pts[s, rng.choice(4096, m, replace=False), :3] for s in range(b)])
    return sel(n), sel(nv), boxes, labels


def test_det_assign_classes_on_the_reference_golden(pkg, cuda):
    """The kernel at C = 3 on the scenes of tests/golden/multiclass_targets.npz (the reference's mask assignment and
    one_hot(label - 1) x centre-ness, with a label of 4) and the class-count oracle on them, bit for bit."""
    z = dict(np.load(os.path.join(ROOT, "tests", "golden", "multiclass_targets.npz")))
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    got = pkg.tf_ops.det_assign(T(z["base_xyz"]), T(z["vote_base"]), T(z["gt_boxes"]), T(z["gt_labels"]), 12, cls_num=3)
    ref = OM.assign(z["base_xyz"], z["vote_base"], z["gt_boxes"], z["gt_labels"], 3)
    for k in ref:
        assert np.array_equal(_bits(got[k]).view(np.uint8), np.asarray(ref[k]).view(np.uint8)), k
    far = z["face_dist"] > 1e-4
    lab = got["cls_label"].cpu().numpy()
    np.testing.assert_allclose(lab[far], z["cls_label"][far], rtol=2e-6, atol=1e-7)
    out = far & (z["pmask"] > 0) & (z["assigned_label"] == 4)
    assert out.any() and (got["pmask"].cpu().numpy()[out] == 1).all() and not lab[out].any()


def test_det_assign_classes(pkg, cuda):
    rng = np.random.default_rng(5)
    base, vb, boxes, labels = _targets_case(rng)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    got = pkg.tf_ops.det_assign(T(base), T(vb), T(boxes), T(labels), 12, cls_num=3)
    one = pkg.tf_ops.det_assign(T(base), T(vb), T(boxes), T(labels), 12)
    for k in pkg.tf_ops.DET_TARGETS:
        if k != "cls_label":
            assert np.array_equal(_bits(got[k]), _bits(one[k])), k
    assert tuple(got["cls_label"].shape) == (3, 512, 3)
    lab = got["cls_label"].cpu().numpy()
    ref = OM.assign(base, vb, boxes, labels, 3)["cls_label"]                 # the class-count oracle, bit for bit
    assert np.array_equal(lab.view(np.int32), ref.view(np.int32))
    for c in range(3):
        col = pkg.tf_ops.det_assign(T(base), T(vb), T(boxes), T((labels == c + 1).astype(np.int32)), 12)["cls_label"]
        assert np.array_equal(_bits(got["cls_label"][..., c].contiguous()), _bits(col)), c
    idx = got["assigned_idx"].cpu().numpy()
    pm = got["pmask"].cpu().numpy()
    out_of_range = (np.take_along_axis(labels, idx, 1) == 4) & (pm > 0)
    assert out_of_range.any() and not lab[out_of_range].any()


def _loss_inputs(pkg, cuda, c, seed=7):
    rng = np.random.default_rng(seed)
    base, vb, boxes, labels = _targets_case(rng)
    labels = np.where(labels > c, c, labels).astype(np.int32) if c < 3 else labels
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    tg = pkg.tf_ops.det_assign(T(base), T(vb), T(boxes), T(labels), 12, cls_num=c)
    b, n, nv = base.shape[0], base.shape[1], vb.shape[1]
    reg = T((0.5 * rng.standard_normal((b, n, 1, 30))).astype(np.float32))
    cls = T((2 * rng.standard_normal((b, n, 1, c))).astype(np.float32))
    vo = T((0.3 * rng.standard_normal((b, nv, 3))).astype(np.float32))
    return T(base), cls, reg, vo, tg


def test_det_loss_classes_at_one_class_is_det_loss(pkg, cuda):
    base, cls, reg, vo, tg = _loss_inputs(pkg, cuda, 1)
    tg1 = dict(tg, cls_label=tg["cls_label"][..., 0].contiguous())
    args = (base, cls, reg[..., :6], reg[..., 6:18], reg[..., 18:], vo)
    l1, n1 = pkg.tf_ops.det_loss(*args, tg1)
    lc, nc = pkg.tf_ops.det_loss(*args, tg, cls_num=1)
    assert np.array_equal(_bits(l1), _bits(lc)) and np.array_equal(_bits(n1), _bits(nc))
    gl = torch.tensor([1.0, 0.5, 2.0, 0.25, 1.5, 0.75], device=cuda)
    g1 = pkg.tf_ops.det_loss_grad(*args, tg1, gl, n1)
    gc = pkg.tf_ops.det_loss_grad(*args, tg, gl, nc, cls_num=1)
    for a, b in zip(g1, gc):
        assert np.array_equal(_bits(a), _bits(b))


@pytest.mark.parametrize("c", [2, 3, 8])
def test_det_loss_classes_against_float64(pkg, cuda, c):
    base, cls, reg, vo, tg = _loss_inputs(pkg, cuda, c, seed=10 + c)
    args = (base, cls, reg[..., :6], reg[..., 6:18], reg[..., 18:], vo)
    loss, norm = pkg.tf_ops.det_loss(*args, tg, cls_num=c)
    # the five other losses are the single-class kernel's, bit for bit
    tg0 = dict(tg, cls_label=tg["cls_label"][..., 0].contiguous())
    l1, n1 = pkg.tf_ops.det_loss(base, cls[..., :1], *args[2:], tg0)
    assert np.array_equal(_bits(loss[1:]), _bits(l1[1:])) and np.array_equal(_bits(norm), _bits(n1))
    # loss_builder.cls_loss in float64: the class mean of the sigmoid cross-entropy, masked, over the mask's sum
    x = cls.double().reshape(cls.shape[0], cls.shape[1], c).requires_grad_()
    z = tg["cls_label"].double()
    cm = (tg["pmask"] + tg["nmask"]).double()
    ce = torch.nn.functional.binary_cross_entropy_with_logits(x, z, reduction="none").mean(-1)
    ref = (ce * cm).sum() / torch.clamp_min(cm.sum(), 1.0)
    ref = ref.detach()
    assert abs(float(loss[0]) - float(ref)) <= 1e-6 * max(1.0, abs(float(ref)))
    gl = torch.tensor([1.5, 0.5, 2.0, 0.25, 1.5, 0.75], device=cuda)
    (gref,) = torch.autograd.grad((ce * cm).sum() / torch.clamp_min(cm.sum(), 1.0) * 1.5, [x])
    grads = pkg.tf_ops.det_loss_grad(*args, tg, gl, norm, cls_num=c)
    assert tuple(grads[1].shape) == (cls.shape[0], cls.shape[1], c)
    assert float((grads[1].double() - gref).abs().max()) <= 1e-5 * max(1.0, float(gref.abs().max()))
    g1 = pkg.tf_ops.det_loss_grad(base, cls[..., :1], *args[2:], tg0, gl, n1)
    for k in (0, 2, 3):
        assert np.array_equal(_bits(grads[k]), _bits(g1[k])), k
    # the class-count oracle (float64)
    npy = lambda t: t.detach().cpu().numpy()
    oloss, onorm = OM.losses(npy(base), npy(cls), npy(reg[..., :6]), npy(reg[..., 6:18]), npy(reg[..., 18:]), npy(vo),
                             {k: npy(v) for k, v in tg.items()}, c)
    assert abs(float(loss[0]) - oloss[0]) <= 1e-6 * max(1.0, abs(oloss[0]))
    og = OM.cls_grad(npy(cls), {k: npy(v) for k, v in tg.items()}, c, 1.5, float(norm[0]))
    assert np.abs(npy(grads[1]).astype(np.float64) - og).max() <= 1e-5 * max(1.0, np.abs(og).max())
    again = pkg.tf_ops.det_loss(*args, tg, cls_num=c)[0], pkg.tf_ops.det_loss_grad(*args, tg, gl, norm, cls_num=c)[1]
    assert np.array_equal(_bits(again[0]), _bits(loss)) and np.array_equal(_bits(again[1]), _bits(grads[1]))


def _weights(pkg, c, seed=0):
    arch = pkg.config.ARCH_3DSSD
    d = pkg.params.init_params(arch, 1, seed=seed, random_bias=True)
    d.update(pkg.params.init_head_params(pkg.config.layer_channels(arch, 1)[-1], cls_channels=c, seed=seed + 1))
    return d


def test_three_class_inference(pkg, cuda):
    w = _weights(pkg, 3)
    head = pkg.DetectionHead(params=w, device=cuda)
    assert head.cls_num == 3 and head.max_output == 300
    with pytest.raises(ValueError):
        pkg.DetectionHead(params=w, device=cuda, cls_num=1)
    net = pkg.SABackbone(params=w, in_channels=1, device=cuda, head=head)
    pts = torch.from_numpy(synth.kitti_like_multiclass(8, 16384, 20, CLS3, seed=3)[0]).to(cuda)
    xyz, feat = net.forward(pts)[:2]
    block, cnt, raw = head(xyz, feat, return_raw=True)
    assert tuple(block.shape) == (8, 300, 9) and raw["score"].shape[-1] == 3
    exp_b, exp_c = _per_class(pkg, raw["boxes"][:, :, 0].contiguous(), raw["score"].contiguous(), 0.1, 100)
    assert np.array_equal(_bits(block), _bits(exp_b)) and np.array_equal(_bits(cnt), _bits(exp_c))
    assert set(np.unique(block[..., 8].cpu().numpy()).tolist()) <= {0.0, 1.0, 2.0}
    eager = [t.clone() for t in net.detections(xyz, feat)]
    gather = pkg.dist.DetectionGather(8, cuda, max_output=head.max_output)
    replay = net.capture(pts, gather=gather)
    _, (gb, gc) = replay(pts)
    torch.cuda.synchronize()
    assert np.array_equal(_bits(gb), _bits(eager[0])) and np.array_equal(_bits(gc), _bits(eager[1]))
    rb, rc = gather.result()
    assert tuple(rb.shape) == (8, 300, 9) and np.array_equal(_bits(rb), _bits(eager[0])) and np.array_equal(_bits(rc), _bits(eager[1]))
    with pytest.raises(ValueError):
        net.capture(pts, gather=pkg.dist.DetectionGather(8, cuda))


def _scenes(pkg, cuda, batch, npoints, seed):
    p, b, l = synth.kitti_like_multiclass(batch, npoints, 20, CLS3, seed=seed)
    xyz, feat = pkg.tf_ops.split_points(torch.from_numpy(p).to(cuda))
    return xyz, feat, torch.from_numpy(b).to(cuda), torch.from_numpy(l).to(cuda)


def test_three_class_training(pkg, cuda, tmp_path):
    S = pkg.solver
    arch = pkg.config.ARCH_3DSSD
    mk = lambda: S.Trainer(arch, pkg.params.TrainableParams(_weights(pkg, 3), cuda), S.Solver())
    tr = mk()
    assert tr.cls_num == 3
    scene = _scenes(pkg, cuda, 2, 2048, seed=4)
    first = tr.step(*scene)
    totals = [float(first["total"])]
    for _ in range(30):
        out = tr.step(*scene)
        assert all(np.isfinite(float(v)) for v in out.values())
        totals.append(float(out["total"]))
    assert totals[-1] < totals[0], totals
    path = str(tmp_path / "ckpt.npz")
    tr.save(path)
    other = mk()
    other.load(path)
    state = lambda t: [t.adam.param, t.adam.m, t.adam.v, t.adam.state, t.tp.stats_flat]
    for x, y in zip(state(tr), state(other)):
        assert np.array_equal(_bits(x), _bits(y))
    # the next step: the same losses; its backward accumulates with float atomics, so the update is compared from one
    # injected gradient (as tests/test_solver_gpu.py does)
    nxt = _scenes(pkg, cuda, 2, 2048, seed=5)
    a, b = tr.step(*nxt), other.step(*nxt)
    for k in a:
        assert np.array_equal(_bits(a[k].reshape(1)), _bits(b[k].reshape(1))), k
    g = torch.randn(tr.adam.grad.shape, generator=torch.Generator(device=cuda).manual_seed(4), device=cuda) * 0.05
    for name in ("param", "m", "v"):
        getattr(other.adam, name).copy_(getattr(tr.adam, name))
    for t in (tr, other):
        t.adam.grad.copy_(g)
        t.adam.step()
    for x, y in zip(state(tr)[:4], state(other)[:4]):
        assert np.array_equal(_bits(x), _bits(y))
    weights = pkg.kitti_io.params_from_tf_variables(dict(np.load(path)))
    head = pkg.DetectionHead(params=weights, device=cuda)
    assert head.cls_num == 3 and weights["pred_cls/weights"].shape[-1] == 3


def test_class_column_through_the_evaluator(pkg, cuda, tmp_path):
    """GT boxes of a three-class batch through the per-class NMS, scored on their own class only (distinct scores, so
    that the precision curve has a point at each of the 41 recall samples): every class and difficulty reaches AP 100 %
    (kitti_ap 1.0) in bird's-eye view and 3-D.  The boxes are whole in the image, at least 45 px tall (easy), apart from
    each other, and every class has more than 41 of them."""
    ev, io = pkg.evaluation, pkg.kitti_io
    b, g = 80, 30
    _, boxes, labels = synth.kitti_like_multiclass(b, 4096, g, CLS3, seed=12)
    p2 = np.array([[721.5377, 0.0, 609.5593, 44.85728], [0.0, 721.5377, 172.854, 0.2163791], [0.0, 0.0, 1.0, 0.002745884]],
                  np.float32)
    keep = np.zeros_like(labels, bool)
    names = []
    for s in range(b):
        lines = []
        for j in range(g):
            x, y, z, l, h, w, ry = boxes[s, j].astype(np.float64)
            if labels[s, j] == 0 or not 6 <= z <= 25:
                continue
            if any(keep[s, k] and np.hypot(boxes[s, k, 0] - x, boxes[s, k, 2] - z) < 6.0 for k in range(j)):
                continue
            x1, y1, x2, y2 = io.project_boxes_to_image(boxes[s, j:j + 1], p2, io.KITTI_IMG_SHAPE)[0]
            if x1 <= 0 or x2 >= io.KITTI_IMG_SHAPE[1] - 1 or y2 - y1 < 45:
                continue
            keep[s, j] = True
            lines.append("%s 0.00 0 0.00 %.2f %.2f %.2f %.2f %.4f %.4f %.4f %.4f %.4f %.4f %.4f"
                         % (CLS3[labels[s, j] - 1], x1, y1, x2, y2, h, w, l, x, y, z, ry))
        path = tmp_path / ("%06d.txt" % s)
        path.write_text("\n".join(lines) + "\n")
        names.append(str(path))
    lab = np.where(keep, labels, 0)
    assert all((lab == c + 1).sum() > 41 for c in range(3))
    bx = np.where(keep[..., None], boxes, 0).astype(np.float32)
    rank = np.linspace(1.0, 0.5, b * g, dtype=np.float32).reshape(b, g)
    scores = np.stack([np.where(lab == c + 1, rank, 0.0) for c in range(3)], -1).astype(np.float32)
    block, cnt = pkg.tf_ops.bev_nms(torch.from_numpy(bx).to(cuda), torch.from_numpy(scores).to(cuda), 0.1, 100, cls_num=3)
    assert set(np.unique(block[..., 8].cpu().numpy()).tolist()) <= {0.0, 1.0, 2.0}
    acc = ev.EvalAccumulator(cls_list=CLS3, cls_thresh=0.3)
    acc.add(block, cnt, [p2] * b, names)
    res = [r.cpu().numpy() for r in acc.evaluate(cuda)]
    for k in (2, 4):                                                  # bird's-eye view and 3-D: the boxes are the GT
        ap = np.asarray(ev.kitti_ap(res[k]))
        assert np.allclose(ap, 1.0, atol=1e-6), (k, ap)


def test_train_and_evaluate_three_classes_with_the_tools(tmp_path):
    """tools/train.py --classes Car,Pedestrian,Cyclist --steps 50 on synthetic scenes writes a checkpoint;
    tools/eval_kitti.py --classes Car,Pedestrian,Cyclist on it, over sample dicts and label files of three-class scenes,
    prints the AP tables of all three classes; the same checkpoint with --classes Car is refused."""
    io = importlib.import_module("3dssd_b200.kitti_io")
    ckpt, samples, labels = tmp_path / "ckpt", tmp_path / "samples", tmp_path / "label_2"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "train.py"), "--classes", "Car,Pedestrian,Cyclist",
                        "--steps", "50", "--batch", "2", "--log-interval", "25", "--ckpt", str(ckpt)],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and r.stdout.count("Total Loss") == 3, r.stdout[-3000:] + r.stderr[-3000:]
    weights = sorted(ckpt.glob("model-*.npz"))[-1]
    assert np.load(weights)["pred_cls/weights"].shape[-1] == 3
    samples.mkdir()
    labels.mkdir()
    pts, boxes, lab = synth.kitti_like_multiclass(8, 16384, 20, CLS3, seed=77)
    p2 = np.array([[721.5377, 0.0, 609.5593, 44.85728], [0.0, 721.5377, 172.854, 0.2163791], [0.0, 0.0, 1.0, 0.002745884]],
                  np.float32)
    for i in range(8):
        lines = []
        for j in np.nonzero((lab[i] > 0) & (boxes[i, :, 2] >= 6))[0]:
            x1, y1, x2, y2 = io.project_boxes_to_image(boxes[i, j:j + 1], p2, io.KITTI_IMG_SHAPE)[0]
            x, y, z, l, h, w, ry = boxes[i, j]
            lines.append("%s 0.00 0 0.00 %.2f %.2f %.2f %.2f %.4f %.4f %.4f %.4f %.4f %.4f %.4f"
                         % (CLS3[lab[i, j] - 1], x1, y1, x2, y2, h, w, l, x, y, z, ry))
        (labels / ("%06d.txt" % i)).write_text("\n".join(lines) + "\n")
        np.save(samples / ("%06d.npy" % i), np.array({io.KEY_POINT_CLOUD: pts[i], io.KEY_STEREO_CALIB: p2, io.KEY_SAMPLE_NAME: i},
                                                    dtype=object), allow_pickle=True)
    ev = [sys.executable, os.path.join(ROOT, "tools", "eval_kitti.py"), "--samples", str(samples), "--labels", str(labels),
          "--weights", str(weights), "--batch", "4", "--cls-thresh", "0.0"]
    r = subprocess.run(ev + ["--classes", "Car,Pedestrian,Cyclist"], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "evaluated 8 frames" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    for title in ("precision_image:", "precision_ground:", "precision_3d:"):
        i = r.stdout.index(title)
        table = r.stdout[i:].split("\n")[1:4]                        # one row per class: Car, Pedestrian, Cyclist
        assert all(len(row.replace("[", " ").replace("]", " ").split()) == 3 for row in table), table
    r = subprocess.run(ev + ["--classes", "Car"], capture_output=True, text=True, timeout=900)
    assert r.returncode != 0 and "pred_cls has 3 class column(s)" in r.stdout + r.stderr
