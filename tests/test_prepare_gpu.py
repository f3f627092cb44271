"""The preprocessing kernel (csrc/prepare.cu) against its numpy twin (oracle/prepare.py) bit for bit, tools/prepare_kitti.py
on the golden's raw tree against the twin and the reference, and the raw KITTI -> train -> eval sequence."""
import glob
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import prepare as OP
from test_augment_gpu import same_bits
from test_prepare_cpu import COORD_TOL, FACE_TOL, GOLDEN, png, twin_frames, write_tree

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T = importlib.import_module("3dssd_b200.tf_ops")
IO = importlib.import_module("3dssd_b200.kitti_io")
MX = importlib.import_module("3dssd_b200.mixup")
KITTI = ("7.215377e+02 0.000000e+00 6.095593e+02 4.485728e+01 0.000000e+00 7.215377e+02 1.728540e+02 2.163791e-01 "
         "0.000000e+00 0.000000e+00 1.000000e+00 2.745884e-03",
         "9.999239e-01 9.837760e-03 -7.445048e-03 -9.869795e-03 9.999421e-01 -4.278459e-03 7.402527e-03 4.351614e-03 9.999631e-01",
         "7.533745e-03 -9.999714e-01 -6.166020e-04 -4.069766e-03 1.480249e-02 7.280733e-04 -9.998902e-01 -7.631618e-02 "
         "9.998621e-01 7.523790e-03 1.480755e-02 -2.717806e-01")


def kitti_block(rng=None):
    p2, r0, tr = (np.array([float(v) for v in s.split()]) for s in KITTI)
    if rng is not None:
        tr = tr + rng.normal(0, 1e-3, 12)
        p2 = p2 * (1 + rng.normal(0, 1e-3, 12))
    return np.concatenate([tr, r0, p2])


def sweep(rng, n):
    """A seeded 360-degree velodyne sweep of n points (x forward, y left, z up, reflectance)."""
    az = rng.uniform(-np.pi, np.pi, n)
    r = 2 + rng.exponential(18, n)
    el = rng.uniform(-0.43, 0.03, n)
    return np.stack([r * np.cos(az) * np.cos(el), r * np.sin(az) * np.cos(el), 1.73 + r * np.sin(el), rng.uniform(0, 1, n)],
                    1).astype(np.float32)


def check_kernel(cuda, pts, off, calib, hw):
    kept, koff = T.prepare_points(torch.from_numpy(pts).to(cuda), off, torch.from_numpy(calib).to(cuda), hw)
    torch.cuda.synchronize()
    tk, toff = OP.prepare_points(pts, off, calib, hw)
    same_bits(koff.cpu().numpy(), toff, "kept offsets")
    same_bits(kept[:int(toff[-1])].cpu().numpy(), tk, "kept points")
    return tk, toff


def test_golden_frames_equal_the_twin(cuda, tmp_path):
    z = dict(np.load(GOLDEN))
    write_tree(z, str(tmp_path))
    fr = twin_frames(z, str(tmp_path)) + twin_frames(z, str(tmp_path), "testing", gt=False)
    off = np.concatenate([[0], np.cumsum([len(f[1]) for f in fr])])
    _, toff = check_kernel(cuda, np.concatenate([f[1] for f in fr]), off, np.stack([f[2] for f in fr]), np.array([f[3] for f in fr]))
    assert (np.diff(toff) > 0).all()


def test_ragged_sweeps_equal_the_twin(cuda):
    rng = np.random.default_rng(31)
    sizes = rng.integers(60000, 130001, 16)
    sizes[5] = 0                                                        # an empty frame
    pts = np.concatenate([sweep(rng, n) for n in sizes])
    off = np.concatenate([[0], np.cumsum(sizes)])
    calib = np.stack([kitti_block(rng) for _ in sizes])
    hw = np.tile([375, 1242], (16, 1))
    hw[3] = (370, 1224)
    calib[9, 29:33] = 0                                                 # P2's last row zero: h_2 = 0 everywhere, none kept
    _, toff = check_kernel(cuda, pts, off, calib, hw)
    n = np.diff(toff)
    assert n[5] == 0 and n[9] == 0 and (np.delete(n, [5, 9]) > 5000).all()


def test_frame_limit_equals_the_twin(cuda):
    rng = np.random.default_rng(32)
    big = T.PREP_MAX_FRAME_POINTS
    pts = np.concatenate([sweep(rng, big), sweep(rng, 1000)])
    check_kernel(cuda, pts, np.array([0, big, big + 1000]), np.stack([kitti_block(), kitti_block(rng)]), np.array([[375, 1242]] * 2))
    with pytest.raises(ValueError):
        T.prepare_points(torch.zeros((big + 1, 4), device=cuda), [0, big + 1], torch.zeros((1, 33), dtype=torch.float64, device=cuda),
                         [[375, 1242]])


def run_tool(*args):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "prepare_kitti.py")] + [str(a) for a in args],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def test_tool_on_the_golden_tree(cuda, tmp_path):
    z = dict(np.load(GOLDEN))
    train_list, test_list = write_tree(z, str(tmp_path))
    out, db_path = tmp_path / "train", tmp_path / "db.npz"
    log = run_tool("--root", tmp_path, "--split", "training", "--list", train_list, "--out", out, "--mixup-db", db_path, "--batch", 4)
    assert "frames read 6, kept 4, skipped 2" in log, log
    frames = twin_frames(z, str(tmp_path))
    dicts, _, lines, tdb = OP.prepare(frames, mixup=True)
    assert (out / "train_list.txt").read_text().split() == lines == [str(s) for s in z["ref_train_list"]]
    assert sorted(os.listdir(out)) == sorted(lines + ["train_list.txt"])
    po, bo = z["ref_point_offsets"], z["ref_box_offsets"]
    for r, i in enumerate(sorted(dicts)):
        got = IO.read_sample(str(out / ("%06d.npy" % i)))
        assert set(got) == set(dicts[i]), i
        for k, v in dicts[i].items():
            assert type(got[k]) is type(v), (i, k)
            if isinstance(v, np.ndarray):
                same_bits(got[k], v, "%d %s" % (i, k))
                assert got[k].dtype == v.dtype, (i, k)
            else:
                assert got[k] == v, (i, k)
        # against the reference
        assert np.abs(got["point_cloud"] - z["ref_points"][po[r]:po[r + 1]]).max() <= COORD_TOL
        face = z["face_margin"][po[r]:po[r + 1]] < FACE_TOL
        assert np.array_equal(got["label_sem_seg"][~face], z["ref_sem"][po[r]:po[r + 1]][~face])
        assert np.array_equal(got["label_boxes_3d"], z["ref_boxes"][bo[r]:bo[r + 1]]) and got["sample_name"] == z["ref_names"][r]
    db = MX.ObjectDatabase.load(str(db_path))
    for k in ("points", "offsets", "boxes", "classes", "frames", "rows"):
        same_bits(getattr(db, k).numpy(), tdb[k], "database " + k)
    same_bits(db.points.numpy(), z["ref_db_points"].astype(np.float32), "database vs the reference")
    # tools/build_mixup_db.py over the written files: the same database, its frames numbering the files in name order
    db2_path = tmp_path / "db2.npz"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "build_mixup_db.py"), "--data", str(out), "--out", str(db2_path),
                        "--batch", "3"], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    db2 = MX.ObjectDatabase.load(str(db2_path))
    for k in ("points", "offsets", "boxes", "classes", "rows"):
        same_bits(getattr(db, k).numpy(), getattr(db2, k).numpy(), "build_mixup_db " + k)
    files = np.array([int(s[:6]) for s in lines])
    same_bits(db.frames.numpy(), files[db2.frames.numpy()], "frames as file numbers")
    # the testing split without GT
    out_t = tmp_path / "test"
    run_tool("--root", tmp_path, "--split", "testing", "--list", test_list, "--out", out_t)
    got = IO.read_sample(str(out_t / "000000.npy"))
    assert set(got) == {"point_cloud", "label_sem_seg", "label_dist", "stereo_calib", "sample_name"}
    assert np.abs(got["point_cloud"] - z["ref_nogt_points"]).max() <= COORD_TOL and (got["label_sem_seg"] == 1).all()


def synthetic_tree(root, rng, ids):
    """A raw KITTI training tree of sweeps with Cars on them, their ground planes, and a train / val list."""
    d = os.path.join(root, "training")
    for sub in ("velodyne", "calib", "image_2", "label_2", "planes"):
        os.makedirs(os.path.join(d, sub), exist_ok=True)
    calib = "P2: %s\nR0_rect: %s\nTr_velo_to_cam: %s\n" % KITTI
    blk = kitti_block()
    V, R0 = blk[:12].reshape(3, 4), blk[12:21].reshape(3, 3)
    M, t = R0 @ V[:, :3], R0 @ V[:, 3]
    for fid in ids:
        f = "%06d" % fid
        pts, lines = [sweep(rng, 60000)], []
        for _ in range(4):
            x, zc, ry = rng.uniform(-12, 12), rng.uniform(8, 40), rng.uniform(-np.pi, np.pi)
            lines.append("Car 0.00 0 -1.57 100 150 300 250 1.56 1.70 3.90 %.2f 1.65 %.2f %.2f" % (x, zc, ry))
            u = rng.uniform(-0.45, 0.45, (300, 3)) * (3.9, 0.9, 1.7)
            c, s = np.cos(ry), np.sin(ry)
            rect = np.stack([c * u[:, 0] + s * u[:, 2] + x, 1.65 - 0.8 + u[:, 1], -s * u[:, 0] + c * u[:, 2] + zc], 1)
            velo = np.linalg.solve(M, (rect - t).T).T                 # the velodyne points whose rect image is rect
            pts.append(np.concatenate([velo, rng.uniform(0, 1, (300, 1))], 1).astype(np.float32))
        lines.append("DontCare -1 -1 -10 503.89 169.71 590.61 190.13 -1 -1 -1 -1000 -1000 -1000 -10")
        np.concatenate(pts).astype(np.float32).tofile(os.path.join(d, "velodyne", f + ".bin"))
        open(os.path.join(d, "calib", f + ".txt"), "w").write(calib)
        open(os.path.join(d, "image_2", f + ".png"), "wb").write(png(1242, 375))
        open(os.path.join(d, "label_2", f + ".txt"), "w").write("\n".join(lines) + "\n")
        open(os.path.join(d, "planes", f + ".txt"), "w").write("# Plane\nWidth 4\nHeight 1\n0.0 -1.0 0.0 1.65\n")
    return d


def test_raw_tree_prepare_train_eval(cuda, tmp_path):
    rng = np.random.default_rng(40)
    ids = [3, 11, 4, 20, 8, 15]
    d = synthetic_tree(str(tmp_path), rng, ids)
    (tmp_path / "train.txt").write_text("\n".join("%06d" % i for i in ids[:4]) + "\n")
    (tmp_path / "val.txt").write_text("\n".join("%06d" % i for i in ids[4:]) + "\n")
    train, val, db = tmp_path / "train_out", tmp_path / "val_out", tmp_path / "db.npz"
    log = run_tool("--root", tmp_path, "--list", tmp_path / "train.txt", "--out", train, "--mixup-db", db)
    assert "kept 4" in log and "mixup database" in log, log
    run_tool("--root", tmp_path, "--list", tmp_path / "val.txt", "--out", val)
    assert len(glob.glob(str(val / "*.npy"))) == 2
    ckpt = tmp_path / "ckpt"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "train.py"), "--data", str(train), "--augment", "--mixup", str(db),
                        "--planes", os.path.join(d, "planes"), "--steps", "3", "--batch", "2", "--log-interval", "1", "--ckpt", str(ckpt)],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and r.stdout.count("Total Loss") == 3, r.stdout[-3000:] + r.stderr[-3000:]
    weights = sorted(glob.glob(str(ckpt / "model-*.npz")))[-1]
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "eval_kitti.py"), "--samples", str(val), "--labels",
                        os.path.join(d, "label_2"), "--weights", weights, "--batch", "2"], capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "evaluated 2 frames" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    assert "AP" in r.stdout or "precision" in r.stdout, r.stdout[-3000:]
