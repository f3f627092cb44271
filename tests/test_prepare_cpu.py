"""The KITTI preprocessing twin (oracle/prepare.py) and the raw-frame readers (kitti_io) against the reference's own
preprocessing (tests/golden/prepare.npz, tests/golden/make_golden_prepare.py), the host checks and the C-boundary call of
tf_ops.prepare_points."""
import importlib
import os
import zlib

import numpy as np
import pytest
import torch

from oracle import prepare as OP
from test_tf_ops_abi_cpu import _Recorder, abi  # noqa: F401  (abi is a fixture)

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "prepare.npz")
FILTER_TOL = 1e-7          # a point this close to a filter bound may fall on either side (sum order, DESIGN 3.14)
FACE_TOL = 1e-4            # metres: float32 semantic labels near a grown face (DESIGN 3.12)
COORD_TOL = 1e-12          # metres
EXACT_FRAME = 2            # the power-of-two frame: every operation exact
IO = importlib.import_module("3dssd_b200.kitti_io")


def png(w, h):
    def chunk(t, data):
        return len(data).to_bytes(4, "big") + t + data + (zlib.crc32(t + data) & 0xFFFFFFFF).to_bytes(4, "big")
    return b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", w.to_bytes(4, "big") + h.to_bytes(4, "big") + bytes([8, 2, 0, 0, 0])) + chunk(b"IEND", b"")


def write_tree(z, root):
    """The golden's raw KITTI tree under root -> (training list path, testing list path)."""
    off = z["velodyne_offsets"]
    lists = {"training": [], "testing": []}
    for k, fid in enumerate(z["frame_ids"]):
        split = str(z["frame_split"][k])
        d = os.path.join(root, split)
        for sub in ("velodyne", "calib", "image_2", "label_2"):
            os.makedirs(os.path.join(d, sub), exist_ok=True)
        f = "%06d" % fid
        z["velodyne"][off[k]:off[k + 1]].astype(np.float32).tofile(os.path.join(d, "velodyne", f + ".bin"))
        open(os.path.join(d, "calib", f + ".txt"), "w").write(str(z["calib_texts"][k]))
        open(os.path.join(d, "image_2", f + ".png"), "wb").write(png(int(z["image_hw"][k][1]), int(z["image_hw"][k][0])))
        if split == "training":
            open(os.path.join(d, "label_2", f + ".txt"), "w").write(str(z["label_texts"][k]))
        lists[split].append("%06d" % fid)
    paths = []
    for split in ("training", "testing"):
        p = os.path.join(root, split + "_list.txt")
        open(p, "w").write("\n".join(lists[split]) + "\n")
        paths.append(p)
    return tuple(paths)


def twin_frames(z, root, split="training", gt=True):
    """oracle/prepare.py frames read back through kitti_io from the rebuilt tree."""
    out = []
    for k, fid in enumerate(z["frame_ids"]):
        if str(z["frame_split"][k]) != split:
            continue
        d, f = os.path.join(root, split), "%06d" % fid
        pts = IO.read_velodyne(os.path.join(d, "velodyne", f + ".bin"))
        calib = IO.calib_block(IO.read_calib(os.path.join(d, "calib", f + ".txt")))
        hw = IO.png_size(os.path.join(d, "image_2", f + ".png"))
        boxes = classes = None
        if gt:
            boxes, classes = IO.read_label(os.path.join(d, "label_2", f + ".txt"), ("Car",))
        out.append((int(fid), pts, calib, hw, boxes, classes))
    return out


@pytest.fixture(scope="module")
def golden(tmp_path_factory):
    z = dict(np.load(GOLDEN))
    root = str(tmp_path_factory.mktemp("kitti"))
    write_tree(z, root)
    return z, root


def test_readers_against_the_golden_text(golden):
    z, root = golden
    d = os.path.join(root, "training")
    cal = IO.read_calib(os.path.join(d, "calib", "000007.txt"))
    assert set(cal) >= {"P0", "P2", "R0_rect", "Tr_velo_to_cam", "Tr_imu_to_velo"} and "calib_time" not in cal
    assert all(v.dtype == np.float64 for v in cal.values())
    assert np.array_equal(cal["P2"].reshape(3, 4), z["ref_p2"][0])
    assert IO.png_size(os.path.join(d, "image_2", "000003.png")) == (370, 1224)
    v = IO.read_velodyne(os.path.join(d, "velodyne", "000007.bin"))
    assert v.dtype == np.float32 and v.shape == (10000, 4) and np.array_equal(v, z["velodyne"][:10000])
    boxes, classes = IO.read_label(os.path.join(d, "label_2", "000007.txt"), ("Car",))
    assert boxes.dtype == np.float64 and classes.dtype == np.int64
    assert np.array_equal(boxes, z["ref_boxes"][:3]) and np.array_equal(classes, z["ref_classes"][:3])
    b2, c2 = IO.read_label(os.path.join(d, "label_2", "000007.txt"), ("Car", "Van"))
    assert len(b2) == 4 and list(c2) == [1, 2, 1, 1]                     # DontCare is dropped, file order is kept
    assert IO.read_label(os.path.join(d, "label_2", "000005.txt"), ("Car",))[0].shape == (0, 7)


def test_malformed_files_raise(tmp_path):
    def put(name, data):
        p = tmp_path / name
        (p.write_bytes if isinstance(data, bytes) else p.write_text)(data)
        return str(p)
    with pytest.raises(ValueError, match="v.bin"):
        IO.read_velodyne(put("v.bin", np.zeros(7, np.float32).tobytes()))
    with pytest.raises(ValueError, match="c1.txt"):
        IO.read_calib(put("c1.txt", "P2: 1 2 3 4 5 6 7 8 9 10 11 12\nR0_rect: 1 0 0 0 1 0 0 0 1\n"))        # no Tr_velo_to_cam
    with pytest.raises(ValueError, match="c2.txt"):
        IO.read_calib(put("c2.txt", "P2: 1 2 3\nR0_rect: 1 0 0 0 1 0 0 0 1\nTr_velo_to_cam: 0 0 0 0 0 0 0 0 0 0 0 0\n"))
    with pytest.raises(ValueError, match="c3.txt"):
        IO.read_calib(put("c3.txt", "P2 1 2 3\n"))
    with pytest.raises(ValueError, match="l1.txt"):
        IO.read_label(put("l1.txt", "Car 0.00 0 -1.57 1 2 3 4 1.5 1.6 3.9 1 2 x 0.1\n"))
    with pytest.raises(ValueError, match="l2.txt"):
        IO.read_label(put("l2.txt", "Car 0.00 0 -1.57 1 2 3 4 1.5 1.6 3.9 1 2\n"))
    with pytest.raises(ValueError, match="l3.txt"):
        IO.read_label(put("l3.txt", "Car  0.00 0 -1.57 1 2 3 4 1.5 1.6 3.9 1 2 3 0.1\n"))    # a double space: an empty field
    with pytest.raises(ValueError, match="p1.png"):
        IO.png_size(put("p1.png", b"GIF89a" + bytes(30)))
    with pytest.raises(ValueError, match="p2.png"):
        IO.png_size(put("p2.png", png(10, 10)[:20]))
    with pytest.raises(FileNotFoundError):
        IO.png_size(str(tmp_path / "missing.png"))
    assert IO.read_label(put("l4.txt", "Car 0.00 0 -1.57 1 2 3 4 1.5 1.6 3.9 1 2 3 0.1 0.93\n"))[0].shape == (1, 7)   # with score


def near_filter(z, k):
    off = z["velodyne_offsets"]
    return z["filter_margin"][off[k]:off[k + 1]] < FILTER_TOL


def test_twin_equals_the_reference(golden):
    """Every kept/skipped decision, the list, boxes, classes, names and the mixup objects equal; coordinates within
    1e-12 m; kept masks and semantic labels equal except the marked near-ties."""
    z, root = golden
    frames = twin_frames(z, root)
    dicts, skipped, lines, db = OP.prepare(frames, mixup=True)
    assert [int(i in dicts) for i in range(len(frames))] == list(z["ref_kept"])
    assert skipped == {3: "no_objects", 4: "no_points"}
    assert lines == [str(s) for s in z["ref_train_list"]]
    po, bo = z["ref_point_offsets"], z["ref_box_offsets"]
    near_any = 0
    for r, i in enumerate(sorted(dicts)):
        d = dicts[i]
        assert d["sample_name"] == z["ref_names"][r] and d["label_num"] == bo[r + 1] - bo[r]
        assert np.array_equal(d["label_boxes_3d"], z["ref_boxes"][bo[r]:bo[r + 1]])
        assert np.array_equal(d["label_classes"], z["ref_classes"][bo[r]:bo[r + 1]])
        assert np.array_equal(d["stereo_calib"], z["ref_p2"][r])
        assert d["label_dist"].dtype == np.float32 and (d["label_dist"] == 1).all()
        ref = z["ref_points"][po[r]:po[r + 1]]
        near = near_filter(z, i)
        near_any += int(near.sum())
        pts, calib, hw = frames[i][1], frames[i][2], frames[i][3]
        rect, u, v = OP.transform(pts, calib)
        mine = OP.keep_mask(rect, u, v, hw)
        assert not near.any() or i == EXACT_FRAME
        assert len(ref) == int(mine.sum()), i
        assert np.abs(d["point_cloud"] - ref).max() <= COORD_TOL, i
        face = z["face_margin"][po[r]:po[r + 1]] < FACE_TOL
        assert np.array_equal(d["label_sem_seg"][~face], z["ref_sem"][po[r]:po[r + 1]][~face]), i
        assert d["label_sem_seg"].dtype == np.int64 and d["point_cloud"].dtype == np.float64
    assert near_any > 5                                                    # the boundary frame holds points on the bounds
    assert np.array_equal(db["offsets"], z["ref_db_offsets"])
    assert np.array_equal(np.stack([db["frames"], db["rows"]], 1), z["ref_db_src"])
    assert np.array_equal(db["boxes"], z["ref_db_boxes"].astype(np.float32))
    assert np.array_equal(db["points"], z["ref_db_points"].astype(np.float32))
    assert (db["counts"] == 3).any()                                       # the three-point Car is not an object


def test_boundary_frame_is_bit_exact(golden):
    z, root = golden
    frames = twin_frames(z, root)
    dicts, _, _, _ = OP.prepare(frames)
    r = sorted(dicts).index(EXACT_FRAME)
    po = z["ref_point_offsets"]
    got, ref = dicts[EXACT_FRAME]["point_cloud"], z["ref_points"][po[r]:po[r + 1]]
    assert got.shape == ref.shape and np.array_equal(got.view(np.uint64), ref.view(np.uint64))
    assert np.array_equal(dicts[EXACT_FRAME]["label_sem_seg"], z["ref_sem"][po[r]:po[r + 1]])


def test_no_gt_frame_equals_the_reference(golden):
    z, root = golden
    frames = twin_frames(z, root, "testing", gt=False)
    dicts, skipped, lines, db = OP.prepare(frames)
    d = dicts[0]
    assert not skipped and lines == ["000000.npy"] and db is None
    assert set(d) == {"point_cloud", "label_sem_seg", "label_dist", "stereo_calib", "sample_name"}
    assert d["sample_name"] == z["ref_nogt_name"] and np.array_equal(d["stereo_calib"], z["ref_nogt_p2"])
    assert np.array_equal(d["label_sem_seg"], z["ref_nogt_sem"]) and (d["label_sem_seg"] == 1).all()
    assert np.abs(d["point_cloud"] - z["ref_nogt_points"]).max() <= COORD_TOL


def test_host_checks_raise(abi):  # noqa: F811
    T, fake = abi
    f = lambda *s: torch.zeros(s, dtype=torch.float32)
    d = lambda *s: torch.zeros(s, dtype=torch.float64)
    hw = np.array([[375, 1242], [370, 1224]])
    big = T.PREP_MAX_FRAME_POINTS
    bad = [lambda: T.prepare_points(f(30, 3), [0, 10, 30], d(2, 33), hw),                  # points not [T, 4]
           lambda: T.prepare_points(d(30, 4), [0, 10, 30], d(2, 33), hw),                  # float64 points
           lambda: T.prepare_points(f(30, 4), [0, 10, 30], f(2, 33), hw),                  # float32 calibration
           lambda: T.prepare_points(f(30, 4), [0, 10, 30], d(2, 32), hw),
           lambda: T.prepare_points(f(30, 4), [0, 10, 30], d(3, 33), hw),
           lambda: T.prepare_points(f(30, 4), [0, 10, 31], d(2, 33), hw),                  # offsets do not end at T
           lambda: T.prepare_points(f(30, 4), [0, 20, 10, 30], d(3, 33), np.ones((3, 2))),  # falling offsets
           lambda: T.prepare_points(f(30, 4), [0, 10, 30], d(2, 33), np.array([[375, 1242], [0, 1224]])),
           lambda: T.prepare_points(f(30, 4), [0, 10, 30], d(2, 33), np.array([[375, -1], [370, 1224]])),
           lambda: T.prepare_points(f(30, 4), [0, 10, 30], d(2, 33), hw[:1]),
           lambda: T.prepare_points(f(30, 4), [0, 10, 30], d(2, 33), hw, (-40, 40, -5, 3, 0)),
           lambda: T.prepare_points(f(30, 4), [30], d(0, 33), np.zeros((0, 2))),            # no frame
           lambda: T.prepare_points(f(big + 1, 4), [0, big + 1], d(1, 33), hw[:1])]        # over the per-frame limit
    for k, call in enumerate(bad):
        fake.calls.clear()
        with pytest.raises(ValueError):
            call()
        assert not fake.calls, k
    fake.calls.clear()
    T.prepare_points(f(big, 4), [0, big], d(1, 33), hw[:1])                               # at the limit
    assert fake.calls[-1][0] == "ssd3d_prepare_points" and fake.calls[-1][1][1] == big


def test_wrapper_abi_trace(abi):  # noqa: F811
    """The entry points, scalars and pointer placements of tf_ops.prepare_points."""
    T, fake = abi
    rec = _Recorder(fake)
    pts, calib = torch.zeros((50, 4), dtype=torch.float32), torch.zeros((3, 33), dtype=torch.float64)
    rec("prep", T.prepare_points, pts, np.array([0, 20, 20, 50]), calib, np.array([[375, 1242], [370, 1224], [256, 512]]))
    t = rec.trace["prep"][0]
    assert t["calls"] == [["ssd3d_prepare_workspace", 3, 30],
                          ["ssd3d_prepare_points", 3, 30, 50, ["a.0", 0], "scratch", ["a.2", 0], "scratch", "scratch", 0, ["r.0", 0],
                           ["r.1", 0], "stream"]]
    assert [r[1:3] for r in t["returns"]] == [[[50, 4], "torch.float64"], [[4], "torch.int32"]]
