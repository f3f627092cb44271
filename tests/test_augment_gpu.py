"""The augmentation kernels (csrc/augment.cu) against their numpy twin (oracle/augment.py), bit for bit, and the
Augmentor in front of the training step."""
import glob
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import augment as OA
from test_backbone_gpu import scaled_arch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
synth = importlib.import_module("3dssd_b200.synth")
A = importlib.import_module("3dssd_b200.augment")
GOLDEN = os.path.join(ROOT, "tests", "golden", "augment.npz")


def ragged_scenes(sizes, max_boxes, seed):
    """KITTI-like scenes of the given point counts packed one after the other."""
    pts, boxes, labels = [], np.zeros((len(sizes), max_boxes, 7), np.float32), np.zeros((len(sizes), max_boxes), np.int32)
    for s, n in enumerate(sizes):
        p, b, l = synth.kitti_like_with_boxes(1, n, max_boxes, seed=seed + 31 * s)
        pts.append(p[0])
        boxes[s], labels[s] = b[0], l[0]
    offsets = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    return np.concatenate(pts), offsets, boxes, labels


def run_gpu(cuda, pts, offsets, sem, boxes, labels, draws, m):
    dbg = {}
    block, ob, ol = A.Augmentor(m, cuda)(torch.from_numpy(pts), torch.from_numpy(offsets),
                                         None if sem is None else torch.from_numpy(sem), torch.from_numpy(boxes),
                                         torch.from_numpy(labels), draws, debug=dbg)
    torch.cuda.synchronize()
    out = {k: v.cpu().numpy() for k, v in dbg.items()}
    out.update(block=block.cpu().numpy(), boxes=ob.cpu().numpy(), labels=ol.cpu().numpy())
    return out


def host_draws(d):
    return tuple(t.cpu().numpy() for t in d)


def same_bits(got, exp, what):
    got, exp = np.ascontiguousarray(got), np.ascontiguousarray(exp)
    assert got.shape == exp.shape, (what, got.shape, exp.shape)
    if got.dtype.kind == "f":
        got, exp = got.view(np.uint32 if got.itemsize == 4 else np.uint64), exp.astype(got.dtype).view(
            np.uint32 if got.itemsize == 4 else np.uint64)
    bad = np.flatnonzero((got != exp).reshape(-1))
    assert bad.size == 0, "%s: %d of %d differ, first at %d" % (what, bad.size, got.size, bad[0])


def check_against_twin(cuda, pts, offsets, sem, boxes, labels, draws, m):
    got = run_gpu(cuda, pts, offsets, sem, boxes, labels, draws, m)
    block, ob, rec = OA.augment(pts, offsets, sem, boxes, labels, host_draws(draws), m)
    same_bits(got["sem_labels"], rec["sem"], "sem labels")
    same_bits(got["chosen_try"], rec["chosen"], "chosen tries")
    same_bits(got["boxes"], ob, "boxes")
    same_bits(got["points"], rec["points"], "points")
    same_bits(got["moved_by"], rec["moved_by"], "moving box")
    same_bits(got["sort_keys"].view(np.uint64), rec["sort_keys"], "sort keys")
    same_bits(got["survivors"], rec["survivors"], "survivor counts")
    same_bits(got["block"], block, "chosen points")
    same_bits(got["labels"], labels, "labels")
    return got, rec


def test_ragged_scenes_equal_the_twin(cuda):
    """8 ragged scenes, 9k..40k points (both branches of the choice), up to 40 boxes, every draw outcome."""
    sizes = [9000, 40000, 16384, 12000, 33000, 16385, 20000, 9500]
    pts, off, boxes, labels = ragged_scenes(sizes, 40, seed=5)
    gen = torch.Generator(device=cuda).manual_seed(11)
    d = A.draw(len(sizes), boxes.shape[1], off[-1], 16384, gen, cuda)
    u = d.scene_u.cpu().numpy()
    u[:, :4] = [[0.7, 0.2, 0.3, 0.4], [0.1, 0.6, 0.2, 0.9], [0.5, 0.5, 0.5, 0.5], [0.9, 0.9, 0.9, 0.1],
                [0.2, 0.1, 0.8, 0.3], [0.6, 0.3, 0.3, 0.6], [0.4, 0.7, 0.1, 0.1], [0.8, 0.4, 0.6, 0.2]]
    d = d._replace(scene_u=torch.from_numpy(u).to(cuda))
    got, rec = check_against_twin(cuda, pts, off, None, boxes, labels, d, 16384)
    n = rec["survivors"]
    assert (n < 16384).any() and (n > 16384).any(), n
    assert (rec["chosen"] >= 0).any() and (got["moved_by"] >= 0).any()


def test_given_sem_labels_and_small_choice(cuda):
    pts, off, boxes, labels = ragged_scenes([3000, 700, 1], 12, seed=9)
    sem = np.concatenate([OA.sem_labels(pts[off[s]:off[s + 1]], boxes[s], labels[s]) for s in range(3)])
    sem[::7] = 0                                        # positives and negatives the boxes do not decide
    sem[5::11] = 3
    gen = torch.Generator(device=cuda).manual_seed(3)
    d = A.draw(3, 12, off[-1], 1024, gen, cuda)
    d = d._replace(scene_u=torch.tensor([[0.5, 0.5, 0.5, 0.5, 0.1, 0.9]] * 3, dtype=torch.float64, device=cuda))
    check_against_twin(cuda, pts, off, sem, boxes, labels, d, 1024)


def test_limits_equal_the_twin(cuda):
    """256 boxes in a packed grid (many exhausted searches) and 131072 points in one scene."""
    pts, off, boxes, labels = ragged_scenes([131072], 40, seed=2)
    g = 256
    bx = np.zeros((1, g, 7), np.float32)
    k = np.arange(g)
    bx[0, :, 0] = (k % 16) * 4.0 - 30.0
    bx[0, :, 1] = 1.65
    bx[0, :, 2] = (k // 16) * 4.0 + 5.0
    bx[0, :, 3:6] = (3.9, 1.6, 1.7)
    bx[0, :, 6] = np.linspace(-np.pi, np.pi, g).astype(np.float32)
    lb = np.ones((1, g), np.int32)
    gen = torch.Generator(device=cuda).manual_seed(7)
    d = A.draw(1, g, off[-1], 16384, gen, cuda)
    d = d._replace(scene_u=torch.tensor([[0.7, 0.1, 0.2, 0.3, 0.8, 0.2]], dtype=torch.float64, device=cuda))
    got, rec = check_against_twin(cuda, pts, off, None, bx, lb, d, 16384)
    assert (rec["chosen"] < 0).any() and (rec["chosen"] >= 0).any()


def test_two_runs_give_the_same_bits(cuda):
    pts, off, boxes, labels = ragged_scenes([20000, 10000], 30, seed=4)
    gen = torch.Generator(device=cuda).manual_seed(5)
    d = A.draw(2, 30, off[-1], 16384, gen, cuda)
    d = d._replace(scene_u=torch.tensor([[0.6, 0.2, 0.2, 0.2, 0.3, 0.7]] * 2, dtype=torch.float64, device=cuda))
    a = run_gpu(cuda, pts, off, None, boxes, labels, d, 16384)
    b = run_gpu(cuda, pts, off, None, boxes, labels, d, 16384)
    for k in a:
        same_bits(a[k], b[k], k)


@pytest.mark.skipif(not os.path.exists(GOLDEN), reason="tests/golden/augment.npz not generated")
def test_golden_scenes_equal_the_twin(cuda):
    """The scenes of the reference's own run: kernels and twin agree bit for bit on the recorded draws."""
    from test_augment_cpu import golden_inputs
    for case in golden_inputs():
        pts, off, sem, boxes, labels, draws, m = case
        dd = A.Draws(*(torch.from_numpy(np.ascontiguousarray(x)).to(cuda) for x in draws))
        check_against_twin(cuda, pts, off, sem, boxes, labels, dd, m)


def test_augmented_training_steps(pkg, cuda):
    """Augmentor -> Trainer.step on the 1/8-scale model: finite losses and positives."""
    S = importlib.import_module("3dssd_b200.solver")
    arch = scaled_arch(pkg, 8)
    d = pkg.params.init_params(arch, 1, seed=0)
    d.update(pkg.params.init_head_params(pkg.config.layer_channels(arch, 1)[-1], seed=1))
    tr = S.Trainer(arch, pkg.params.TrainableParams(d, cuda), S.Solver(), None)
    aug = A.Augmentor(2048, cuda)
    for step in range(3):
        pts, off, boxes, labels = ragged_scenes([3000, 2500], 12, seed=100 + step)
        for a in (pts, boxes):                            # squeezed like compact_scene: the density of the 1/8 radii
            a[..., 0] *= 0.2
            a[..., 2] *= 0.2
        boxes[..., [3, 5]] *= 0.2
        gen = torch.Generator(device=cuda).manual_seed(A.draw_seed(0, step))
        dr = A.draw(2, 12, off[-1], 2048, gen, cuda)
        block, gb, gl = aug(torch.from_numpy(pts), torch.from_numpy(off), None, torch.from_numpy(boxes),
                            torch.from_numpy(labels), dr)
        xyz, feat = pkg.tf_ops.split_points(block)
        losses = tr.step(xyz, feat, gb, gl)
        vals = {k: float(v) for k, v in losses.items()}
        assert all(np.isfinite(v) for v in vals.values()), vals
    tg = pkg.tf_ops.det_assign(xyz, xyz, gb, gl)                   # the augmented points lie in the augmented boxes
    assert float(tg["pmask"].sum()) > 0


@pytest.mark.parametrize("source", ["synthetic", "files"])
def test_train_tool_with_augment(tmp_path, source):
    args = [sys.executable, os.path.join(ROOT, "tools", "train.py"), "--augment", "--steps", "3", "--batch", "2",
            "--log-interval", "1"]
    if source == "files":
        p, b, l = synth.kitti_like_with_boxes(3, 20000, 10, seed=8)
        for i in range(3):
            n = 15000 + 2000 * i
            d = {"point_cloud": p[i, :n], "label_boxes_3d": b[i, l[i] > 0], "label_classes": l[i, l[i] > 0],
                 "sample_name": i}
            if i != 1:
                d["label_sem_seg"] = OA.sem_labels(p[i, :n], b[i], l[i])
            np.save(tmp_path / ("%06d.npy" % i), np.array(d, dtype=object), allow_pickle=True)
        args += ["--data", str(tmp_path)]
        assert len(glob.glob(str(tmp_path / "*.npy"))) == 3
    r = subprocess.run(args, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.count("Total Loss") == 3, r.stdout[-3000:]
