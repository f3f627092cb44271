"""The mixup kernels (csrc/mixup.cu) against their numpy twin (oracle/mixup.py), bit for bit, and the Augmentor with
mixup in front of the training step."""
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import augment as OA
from oracle import mixup as OM
from test_augment_gpu import ragged_scenes, same_bits

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "mixup.npz")
synth = importlib.import_module("3dssd_b200.synth")
A = importlib.import_module("3dssd_b200.augment")
MX = importlib.import_module("3dssd_b200.mixup")


def gpu_db(cuda, pts, off, boxes, labels):
    return MX.ObjectDatabase.build(torch.from_numpy(pts), off, boxes, labels, device=cuda)


def check_db(cuda, pts, off, boxes, labels):
    db = gpu_db(cuda, pts, off, boxes, labels)
    tw = OM.build_db(pts, off, boxes, labels)
    same_bits(db.host_offsets, tw["offsets"], "object offsets")
    same_bits(db.offsets.cpu().numpy(), tw["offsets"], "device offsets")
    same_bits(db.points.cpu().numpy(), tw["points"], "object points")
    same_bits(db.boxes.cpu().numpy(), tw["boxes"], "object boxes")
    same_bits(db.classes.cpu().numpy(), tw["classes"], "object classes")
    same_bits(np.stack([db.frames.cpu().numpy(), db.rows.cpu().numpy()], 1), np.stack([tw["frames"], tw["rows"]], 1), "sources")
    return db, tw


def twin_db(db):
    return dict(points=db.points.cpu().numpy(), offsets=db.host_offsets, boxes=db.boxes.cpu().numpy(), classes=db.classes.cpu().numpy())


def check_paste(cuda, db, pts, off, sem, boxes, labels, ids, planes):
    mix = MX.Mixup(db, ids, planes)
    d = torch.device(cuda)
    m = MX.paste(mix, torch.from_numpy(pts).to(d), off, torch.from_numpy(off).to(d), torch.from_numpy(sem).to(d),
                 torch.from_numpy(boxes).to(d), torch.from_numpy(labels).to(d))
    torch.cuda.synchronize()
    tp, toff, tsem, tb, tl, tacc = OM.paste(pts, off, sem, boxes, labels, ids, twin_db(db), planes)
    same_bits(m.layout.offsets, toff, "pasted offsets")
    same_bits(m.points.cpu().numpy(), tp, "pasted points")
    same_bits(m.sem_labels.cpu().numpy(), tsem, "pasted labels")
    same_bits(m.boxes.cpu().numpy(), tb, "pasted boxes")
    same_bits(m.labels.cpu().numpy(), tl, "pasted box labels")
    same_bits(m.accepted.cpu().numpy(), tacc, "accepted")
    return m, tacc


def tilted(rng, b):
    p = np.stack([rng.uniform(-0.05, 0.05, b), -rng.uniform(0.95, 1.05, b), rng.uniform(-0.05, 0.05, b), rng.uniform(1.5, 1.8, b)], 1)
    return p / np.linalg.norm(p[:, :3], axis=1, keepdims=True)


def source_db(cuda, seed=40, frames=6, max_boxes=20):
    pts, off, boxes, labels = ragged_scenes([20000 + 1000 * k for k in range(frames)], max_boxes, seed=seed)
    return gpu_db(cuda, pts, off, boxes, labels)


def test_database_equals_the_twin(cuda):
    z = np.load(GOLDEN)
    check_db(cuda, z["db_frame_points"], z["db_frame_offsets"], z["db_frame_boxes"], z["db_frame_labels"])
    sizes = [131072, 9000, 20000, 1, 15000, 33000, 700, 18000]
    pts, off, boxes, labels = ragged_scenes(sizes, 40, seed=21)
    g = 256
    bx, lb = np.zeros((8, g, 7), np.float32), np.zeros((8, g), np.int32)
    bx[:, :40], lb[:, :40] = boxes, labels
    rng = np.random.default_rng(3)
    k = np.arange(g - 40)                                               # frame 0: 256 rows
    bx[0, 40:, 0], bx[0, 40:, 1], bx[0, 40:, 2] = (k % 18) * 3.5 - 30, 1.65, (k // 18) * 4.5 + 5
    bx[0, 40:, 3:6] = (3.9, 1.6, 1.7)
    bx[0, 40:, 6] = rng.uniform(-np.pi, np.pi, g - 40)
    lb[0, 40:] = 1
    lb[2, :5] = 2                                                       # another class
    db, _ = check_db(cuda, pts, off, bx, lb)
    assert len(db) > 100 and (db.frames.cpu().numpy() == 0).sum() > 40


def test_golden_scenes_paste_equals_the_twin(cuda):
    z = np.load(GOLDEN)
    db, _ = check_db(cuda, z["db_frame_points"], z["db_frame_offsets"], z["db_frame_boxes"], z["db_frame_labels"])
    _, acc = check_paste(cuda, db, z["points"], z["offsets"], z["sem_labels"], z["gt_boxes"], z["gt_labels"], z["ids"], z["ref_planes"])
    same_bits(acc, z["ref_accepted"], "accepted vs the reference")


def test_ragged_scenes_paste_equals_the_twin(cuda):
    db = source_db(cuda)
    pts, off, boxes, labels = ragged_scenes([9000, 40000, 16384, 12000, 33000, 16385, 20000, 9500], 40, seed=5)
    rng = np.random.default_rng(8)
    sem = np.concatenate([OA.sem_labels(pts[off[s]:off[s + 1]], boxes[s], labels[s]) for s in range(8)])
    ids = MX.Sampler(db, seed=1).ids(3, 8)
    m, acc = check_paste(cuda, db, pts, off, sem, boxes, labels, ids, tilted(rng, 8))
    assert acc[ids >= 0].any() and not acc[ids >= 0].all()
    # every point of a kept object lies inside its pasted box grown by 0.1
    mp, mb, lay = m.points.cpu().numpy(), m.boxes.cpu().numpy(), m.layout
    for s in range(8):
        kept = np.flatnonzero(acc[s])
        nv = int(OA.valid_rows(boxes[s]).sum())
        for r, i in enumerate(kept):
            p = mp[lay.offsets[s] + lay.slot_start[s, i]:lay.offsets[s] + lay.slot_start[s, i + 1]]
            n, d = OA.planes(mb[s, nv + r:nv + r + 1], OA.EXPAND)
            assert OA.inside(p[:, 0], p[:, 1], p[:, 2], n[0], d[0]).all(), (s, i)


def test_paste_limits_equal_the_twin(cuda):
    db = source_db(cuda)
    rng = np.random.default_rng(9)
    n_obj = len(db)
    sizes = np.diff(db.host_offsets)
    # G + S = 256: 241 rows and 15 draws
    pts, off, boxes, labels = ragged_scenes([20000, 5000], 40, seed=6)
    g = 241
    bx, lb = np.zeros((2, g, 7), np.float32), np.zeros((2, g), np.int32)
    bx[:, :40], lb[:, :40] = boxes, labels
    k = np.arange(g - 40)
    bx[0, 40:, 0], bx[0, 40:, 1], bx[0, 40:, 2], bx[0, 40:, 3:6] = (k % 15) * 4.0 - 30, 1.65, (k // 15) * 4.5 + 5, (3.9, 1.6, 1.7)
    lb[0, 40:] = 1
    sem = np.zeros(off[-1], np.int32)
    ids = rng.integers(0, n_obj, (2, 15)).astype(np.int32)
    check_paste(cuda, db, pts, off, sem, bx, lb, ids, tilted(rng, 2))
    # a scene of exactly 131072 slots
    first = rng.integers(0, n_obj, 15).astype(np.int32)
    n0 = 131072 - int(sizes[first].sum())
    pts, off, boxes, labels = ragged_scenes([n0, 3000], 20, seed=7)
    ids = np.stack([first, rng.integers(0, n_obj, 15).astype(np.int32)])
    m, _ = check_paste(cuda, db, pts, off, np.zeros(off[-1], np.int32), boxes, labels, ids, tilted(rng, 2))
    assert m.layout.max_slots == 131072
    # every id -1
    check_paste(cuda, db, pts, off, np.zeros(off[-1], np.int32), boxes, labels, np.full((2, 15), -1, np.int32), tilted(rng, 2))
    # every object dropped: each scene holds the drawn boxes themselves
    ids = rng.integers(0, n_obj, (2, 15)).astype(np.int32)
    bx = db.boxes.cpu().numpy()[ids]
    _, acc = check_paste(cuda, db, pts, off, np.zeros(off[-1], np.int32), bx, np.ones((2, 15), np.int32), ids, tilted(rng, 2))
    assert not acc.any()


def run_chain(cuda, db, pts, off, sem, boxes, labels, ids, planes, m, seed):
    lay = MX.layout(off, ids, db.host_offsets, boxes.shape[1])
    gen = torch.Generator(device=cuda).manual_seed(seed)
    d = A.draw(len(off) - 1, lay.rows, lay.total, m, gen, cuda)
    d = d._replace(scene_u=d.scene_u.clone().fill_(0.25))
    dbg = {}
    block, ob, ol = A.Augmentor(m, cuda)(torch.from_numpy(pts).pin_memory(), torch.from_numpy(off).pin_memory(),
                                         None if sem is None else torch.from_numpy(sem), torch.from_numpy(boxes).pin_memory(),
                                         torch.from_numpy(labels).pin_memory(), d, debug=dbg, mixup=MX.Mixup(db, ids, planes))
    return block, ob, ol, dbg, d


def test_augmentor_with_mixup_equals_the_twin_chain(cuda):
    db = source_db(cuda)
    pts, off, boxes, labels = ragged_scenes([9000, 40000, 16384, 12000], 30, seed=15)
    rng = np.random.default_rng(10)
    ids = MX.Sampler(db, seed=2).ids(0, 4)
    planes = tilted(rng, 4)
    block, ob, ol, dbg, d = run_chain(cuda, db, pts, off, None, boxes, labels, ids, planes, 16384, 5)
    torch.cuda.synchronize()
    tb, tob, tol, rec = OM.augment(pts, off, None, boxes, labels, ids, twin_db(db), planes, tuple(t.cpu().numpy() for t in d), 16384)
    same_bits(dbg["input_sem_labels"].cpu().numpy(), rec["sem"], "sem labels")
    same_bits(dbg["pasted_points"].cpu().numpy(), rec["pasted_points"], "pasted points")
    same_bits(dbg["sem_labels"].cpu().numpy(), rec["pasted_sem"], "pasted labels")
    same_bits(dbg["chosen_try"].cpu().numpy(), rec["chosen"], "chosen tries")
    same_bits(ob.cpu().numpy(), tob, "boxes")
    same_bits(ol.cpu().numpy(), tol, "labels")
    same_bits(dbg["points"].cpu().numpy(), rec["points"], "points")
    same_bits(dbg["moved_by"].cpu().numpy(), rec["moved_by"], "moving box")
    same_bits(dbg["sort_keys"].cpu().numpy().view(np.uint64), rec["sort_keys"], "sort keys")
    same_bits(dbg["survivors"].cpu().numpy(), rec["survivors"], "survivors")
    same_bits(block.cpu().numpy(), tb, "block")
    absent = rec["pasted_sem"] < 0
    assert absent.any() and (rec["sort_keys"][absent] == OA.ALL_ONES).all()


def test_mixup_call_does_not_synchronise(cuda):
    db = source_db(cuda)
    pts, off, boxes, labels = ragged_scenes([20000, 18000], 30, seed=16)
    ids = MX.Sampler(db, seed=3).ids(1, 2)
    planes = np.tile(np.array(MX.FLAT_PLANE), (2, 1))
    run_chain(cuda, db, pts, off, None, boxes, labels, ids, planes, 16384, 6)             # warm-up: loads the modules
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        run_chain(cuda, db, pts, off, None, boxes, labels, ids, planes, 16384, 7)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


@pytest.mark.parametrize("source", ["synthetic", "files"])
def test_train_tool_with_mixup(tmp_path, source):
    db_path = tmp_path / "db.npz"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "build_mixup_db.py"), "--synthetic", "4", "--out", str(db_path)],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "objects" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    args = [sys.executable, os.path.join(ROOT, "tools", "train.py"), "--augment", "--mixup", str(db_path), "--steps", "3",
            "--batch", "2", "--log-interval", "1"]
    if source == "files":
        p, b, l = synth.kitti_like_with_boxes(3, 20000, 10, seed=8)
        data, planes = tmp_path / "data", tmp_path / "planes"
        data.mkdir()
        planes.mkdir()
        for i in range(3):
            d = {"point_cloud": p[i, :15000 + 2000 * i], "label_boxes_3d": b[i, l[i] > 0], "label_classes": l[i, l[i] > 0],
                 "sample_name": i}
            np.save(data / ("%06d.npy" % i), np.array(d, dtype=object), allow_pickle=True)
            (planes / ("%06d.txt" % i)).write_text("# Plane\nWidth 4\nHeight 1\n0.01 -0.99 0.02 1.66\n")
        args += ["--data", str(data), "--planes", str(planes)]
    r = subprocess.run(args, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert r.stdout.count("Total Loss") == 3, r.stdout[-3000:]
