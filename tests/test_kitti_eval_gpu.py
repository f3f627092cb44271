"""The GPU KITTI evaluator (csrc/box_eval.cu, DESIGN.md section 3.10) bit for bit against its C twin
(oracle/kitti_eval_twin.c): calc_iou / calc_iou_match, and the six Evaluate arrays on the rule frames, a synthetic
3,769-frame validation set, perfect and hopeless detections, frames at the per-frame limits, and the detector end to end."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import kitti_eval as K

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _boxes(rng, b, n):
    """Boxes clustered so that many pairs overlap: (x, y, z, l, h, w, ry)."""
    out = np.empty((b, n, 7), np.float32)
    out[..., 0] = rng.uniform(-4, 4, (b, n))
    out[..., 1] = rng.uniform(1, 2, (b, n))
    out[..., 2] = rng.uniform(16, 24, (b, n))
    out[..., 3:6] = rng.uniform(0.5, 4.5, (b, n, 3))
    out[..., 6] = rng.uniform(-np.pi, np.pi, (b, n))
    out[..., 6].flat[::7] = np.float32(np.pi)
    return out


@pytest.mark.parametrize("shape", [(8, 100, 40), (1, 512, 64), (3, 7, 5), (0, 4, 3), (2, 0, 3), (2, 4, 0)])
def test_calc_iou_equals_the_twin(pkg, cuda, shape):
    b, n, m = shape
    rng = np.random.default_rng(b * 1000 + n + m)
    d, g = _boxes(rng, b, n), _boxes(rng, b, m)
    bev, v3 = pkg.tf_ops.calc_iou(torch.from_numpy(d).to(cuda), torch.from_numpy(g).to(cuda))
    eb, e3 = K.twin_box_iou(d, g)
    np.testing.assert_array_equal(bev.cpu().numpy(), eb)
    np.testing.assert_array_equal(v3.cpu().numpy(), e3)
    if b * n * m:
        assert (eb > 0).mean() > 0.1


def test_calc_iou_match_equals_the_twin(pkg, cuda):
    rng = np.random.default_rng(9)
    d, g = _boxes(rng, 1, 100000)[0], _boxes(rng, 1, 100000)[0]
    bev, v3 = pkg.tf_ops.calc_iou_match(torch.from_numpy(d).to(cuda), torch.from_numpy(g).to(cuda))
    eb, e3 = K.twin_box_iou_matched(d, g)
    np.testing.assert_array_equal(bev.cpu().numpy(), eb)
    np.testing.assert_array_equal(v3.cpu().numpy(), e3)


def _gpu_eval(pkg, cuda, rows, labels, nl):
    return [a.cpu().numpy() for a in pkg.tf_ops.evaluate_labels(torch.from_numpy(rows).to(cuda), labels,
                                                                torch.from_numpy(np.asarray(nl, np.int32)).to(cuda))]


def _assert_equal(got, exp):
    for k, (a, b) in enumerate(zip(got, exp)):
        np.testing.assert_array_equal(a, b, err_msg="array %d" % k)


def test_evaluate_rule_frames(pkg, cuda):
    from test_kitti_eval_cpu import RULES, _frame
    rows, labels, nl = [], [], []
    for name in sorted(RULES):
        r, l, n, _ = _frame(name)
        rows.append(r)
        labels += l
        nl += list(n)
        _assert_equal(_gpu_eval(pkg, cuda, r, l, n), K.twin_evaluate(r, l, n))
    rows = np.concatenate(rows)
    _assert_equal(_gpu_eval(pkg, cuda, rows, labels, nl), K.twin_evaluate(rows, labels, nl))


def test_evaluate_synthetic_val_set(pkg, cuda):
    rows, labels, nl = K.synthetic_frames(3769, seed=11, max_labels=12)
    exp = K.twin_evaluate(rows, labels, nl)
    got = _gpu_eval(pkg, cuda, rows, labels, nl)
    _assert_equal(got, exp)
    _assert_equal(_gpu_eval(pkg, cuda, rows, labels, nl), got)          # two calls, the same bits
    for m in (0, 2, 4):
        assert np.all(got[m] >= 0) and np.any(got[m][:, :, 1:] > 0)      # every class evaluated, something found
    for m in (1, 3, 5):
        assert np.all(got[m] == -1)


def _separated(labels):
    """Frames whose non-DontCare labels overlap no other label, in the image or in BEV."""
    for lab in labels:
        obj = [r for r in lab if int(r[0]) != K.DONTCARE]
        for i in range(len(obj)):
            for j in range(i + 1, len(obj)):
                if K.image_overlap(obj[i][4:8], obj[j][4:8]) > 0 or K.box_overlaps(K.label_box7(obj[i]), K.label_box7(obj[j]))[0] > 0:
                    return False
    return True


def test_perfect_and_hopeless_detections(pkg, cuda):
    rows, labels, nl = [], [], []
    seed = 0
    while len(labels) < 1500:
        r, l, n = K.synthetic_frames(1, seed=5000 + seed, max_labels=3, perfect=True)
        seed += 1
        if _separated(l):
            rows.append(r)
            labels += l
            nl += list(n)
    rows = np.concatenate(rows)
    got = _gpu_eval(pkg, cuda, rows, labels, nl)
    _assert_equal(got, K.twin_evaluate(rows, labels, nl))
    for m in range(3):
        for c in range(3):
            for d in range(3):
                n_gt = sum(K.ignored_gt(r, c, d) == 0 for lab in labels for r in lab)
                p = got[2 * m][c, d]
                k = int(np.sum(p == 1))
                assert np.all(p[:k] == 1) and np.all(p[k:] == 0), (m, c, d, p)
                assert k == 41 if n_gt >= 41 else 0 < k <= 41, (m, c, d, n_gt, k)
    rows, labels, nl = K.synthetic_frames(300, seed=12, max_labels=6, miss_all=True)
    got = _gpu_eval(pkg, cuda, rows, labels, nl)
    _assert_equal(got, K.twin_evaluate(rows, labels, nl))
    for m in (0, 2, 4):
        assert np.all(got[m] == 0)


def test_frames_at_the_per_frame_limits(pkg, cuda):
    rng = np.random.default_rng(13)
    rows, labels, nl = K.synthetic_frames(2, seed=14, max_labels=10)
    assert len(rows) > 0
    big_lab = np.concatenate([K.synthetic_frames(1, seed=15 + i, max_labels=12)[1][0] for i in range(60)])[:256]
    big_det = np.tile(rows, (-(-1024 // len(rows)), 1))[:1024].copy()
    big_det[:, 13] = rng.uniform(0.3, 1, 1024)
    assert big_lab.shape[0] == 256 and big_det.shape[0] == 1024
    r = np.concatenate([rows, big_det])
    l = labels + [big_lab]
    n = list(nl) + [1024]
    _assert_equal(_gpu_eval(pkg, cuda, r, l, n), K.twin_evaluate(r, l, n))
    with pytest.raises(ValueError, match="1024 detections"):
        _gpu_eval(pkg, cuda, np.concatenate([r, r[:1]]), l, n[:-1] + [1025])
    with pytest.raises(ValueError, match="256 label rows"):
        _gpu_eval(pkg, cuda, r, l[:-1] + [np.concatenate([big_lab, big_lab[:1]])], n)


def _label_text(lab):
    names = {0: "Car", 1: "Pedestrian", 2: "Cyclist", 3: "Van", 4: "Person_sitting", 5: "DontCare", 6: "Misc"}
    return "".join("%s %s %d %s\n" % (names[int(r[0])], repr(float(r[1])), int(r[2]), " ".join(repr(float(v)) for v in r[3:]))
                   for r in lab)


def test_detector_end_to_end(pkg, cuda, tmp_path):
    synth = __import__("importlib").import_module("3dssd_b200.synth")
    io, ev = pkg.kitti_io, pkg.evaluation
    arch = pkg.config.ARCH_3DSSD
    weights = pkg.params.init_params(arch, 1, seed=21)
    weights.update(pkg.params.init_head_params(pkg.config.layer_channels(arch, 1)[-1], seed=22))
    pts = synth.kitti_like(8, 16384, seed=23)
    p2 = np.array([[721.5, 0, 609.6, 44.9], [0, 721.5, 172.9, 0.2], [0, 0, 1, 0.003]], np.float32)
    _, labels, _ = K.synthetic_frames(8, seed=24, max_labels=8)
    (tmp_path / "label_2").mkdir()
    (tmp_path / "samples").mkdir()
    names = []
    for i, lab in enumerate(labels):
        path = tmp_path / "label_2" / ("%06d.txt" % i)
        path.write_text(_label_text(lab))
        names.append(str(path))
        np.save(tmp_path / "samples" / ("%06d.npy" % i),
                np.array({io.KEY_POINT_CLOUD: pts[i], io.KEY_STEREO_CALIB: p2, io.KEY_SAMPLE_NAME: i}, dtype=object),
                allow_pickle=True)
    head = pkg.DetectionHead(params=weights, device=cuda)
    net = pkg.SABackbone(arch, weights, in_channels=1, device=cuda, head=head)
    xyz, feat = net.forward(torch.from_numpy(pts).to(cuda))[:2]
    block, count = net.detections(xyz, feat)
    rows, nl = ev.detection_rows(block, count, [p2] * 8, cls_thresh=0.0)
    assert rows.shape[0] > 0
    got = [a.cpu().numpy() for a in pkg.tf_ops.evaluate(torch.from_numpy(rows).to(cuda), names, torch.from_numpy(nl).to(cuda))]
    parsed = [ev.read_label_file(n) for n in names]
    for a, b in zip(parsed, labels):
        np.testing.assert_array_equal(a, b)
    _assert_equal(got, K.twin_evaluate(rows, parsed, nl))
    assert np.all(got[0][0] >= 0) and np.all(got[0][1:] == -1)
    acc = ev.EvalAccumulator(cls_thresh=0.0)
    acc.add(block[:4], count[:4], [p2] * 4, names[:4])
    acc.add(block[4:], count[4:], [p2] * 4, names[4:])
    _assert_equal([a.cpu().numpy() for a in acc.evaluate(cuda)], got)
    assert len(ev.format_ap_tables(got)) == 7

    np.savez(tmp_path / "weights.npz", **weights)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "eval_kitti.py"), "--samples", str(tmp_path / "samples"),
                          "--labels", str(tmp_path / "label_2"), "--weights", str(tmp_path / "weights.npz"), "--batch", "4",
                          "--cls-thresh", "0.0"], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "precision_3d:" in out.stdout and "evaluated 8 frames" in out.stdout


def test_recall(pkg, cuda):
    rng = np.random.default_rng(25)
    g = _boxes(rng, 1, 6)[0]
    p = np.concatenate([g[:4], g[:1], _boxes(rng, 1, 3)[0] + np.float32([30, 0, 30, 0, 0, 0, 0])])
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    det, tot = pkg.evaluation.recall([to(p), to(p[:0])], [to(g), to(g)], 0.7)
    _, iou3 = K.twin_box_iou(p[None], g[None])
    best = iou3[0].max(1)
    assert (det, tot) == (len(np.unique(iou3[0].argmax(1)[best >= 0.7])), 12)
    assert det >= 4
