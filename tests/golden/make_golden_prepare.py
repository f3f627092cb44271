"""Generates tests/golden/prepare.npz by executing the REFERENCE's own KITTI preprocessing on a written raw tree.

Pulled out of their source files with `ast` (make_golden_augment.pull / make_golden_mixup.pull_method; nothing is copied
into this repo) and executed as they are:
  lib/utils/kitti_util.py                    Calibration, inverse_rigid_trans, Object3d, read_label, load_velo_scan
  lib/utils/points_filter.py                 get_point_filter, get_point_filter_in_image
  lib/utils/box_3d_utils.py                  object_label_to_box_3d
  lib/utils/voxelnet_aug.py                  check_inside_points and its corner / surface chain
  lib/dataset/dataloader/kitti_dataloader.py KittiDataset.preprocess_samples and generate_mixup_sample on an instance
                                             made without __init__
  lib/dataset/maps_dict.py                   executed whole (key constants)
Stubs: cfg (POINT_CLOUD_RANGE, CLS_LIST ('Car',), EXPAND_DIMS_LENGTH, MIN_POINTS_NUM, TEST.WITH_GT), a kitti_object over
the written tree, cv2 (imread gives the recorded (H, W, 3) shape, cvtColor is the identity) and numba (identity
decorators).  The numpy of this project has no np.int, so the executed code gets a numpy proxy whose `int` is the
builtin.  preprocess_batch's loop (kitti_dataloader.py:294-311) is restated: preprocess_samples([i]) per list position,
'%06d.npy' % i for every frame it returns, generate_mixup_sample on each of those.

Frames (training list, in list order; KITTI ids differ from positions):
  0, 1  a 10000-point subsample of mayavi/kitti_sample_scan.txt (the reference's one real scan, U(0,1) intensity) with
        a KITTI calibration, Car / Van / DontCare rows, at 1242 x 375 and 1224 x 370
  2     power-of-two calibration, points exactly on u = 0, u = W, v = 0, v = H, rect_z = 0 (h_2 = 0, 0 / 0 too) and
        every extents bound: all arithmetic exact, so BLAS order cannot matter
  3     no Car (Van and DontCare only): skipped
  4     Cars holding no kept point: skipped
  5     a Car holding 3 points (not in the database) and one holding 40
and one frame of the testing split processed without GT.
Recorded per point: the float64 margin to the nearest filter bound (u, v, rect_z, extents) and, for the kept points,
to the nearest face of a grown class box, to mark near-ties.
Needs a reference checkout (path in $REFERENCE):   REFERENCE=<checkout> python tests/golden/make_golden_prepare.py
"""
import os
import sys
import tempfile
import types
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_augment as MGA  # noqa: E402
import make_golden_mixup as MGM  # noqa: E402

REF = MGA.REF
EXTENTS = (-40, 40, -5, 3, 0, 70)
KITTI_CALIB = {
    "P0": "7.215377e+02 0.000000e+00 6.095593e+02 0.000000e+00 0.000000e+00 7.215377e+02 1.728540e+02 0.000000e+00 "
          "0.000000e+00 0.000000e+00 1.000000e+00 0.000000e+00",
    "P2": "7.215377e+02 0.000000e+00 6.095593e+02 4.485728e+01 0.000000e+00 7.215377e+02 1.728540e+02 2.163791e-01 "
          "0.000000e+00 0.000000e+00 1.000000e+00 2.745884e-03",
    "R0_rect": "9.999239e-01 9.837760e-03 -7.445048e-03 -9.869795e-03 9.999421e-01 -4.278459e-03 7.402527e-03 "
               "4.351614e-03 9.999631e-01",
    "Tr_velo_to_cam": "7.533745e-03 -9.999714e-01 -6.166020e-04 -4.069766e-03 1.480249e-02 7.280733e-04 -9.998902e-01 "
                      "-7.631618e-02 9.998621e-01 7.523790e-03 1.480755e-02 -2.717806e-01",
    "Tr_imu_to_velo": "9.999976e-01 7.553071e-04 -2.035826e-03 -8.086759e-01 -7.854027e-04 9.998898e-01 -1.482298e-02 "
                      "3.195559e-01 2.024406e-03 1.482454e-02 9.998881e-01 -7.997231e-01",
}
EXACT_CALIB = {"P2": "256 0 256 0 0 256 128 0 0 0 1 0", "R0_rect": "1 0 0 0 1 0 0 0 1",
               "Tr_velo_to_cam": "0 -1 0 0 0 0 -1 0 1 0 0 0"}


class NumpyProxy(types.ModuleType):
    """numpy with np.int = the builtin int (the reference predates its removal)."""

    def __init__(self):
        super().__init__("numpy")
        self.int = int

    def __getattr__(self, k):
        return getattr(np, k)


def png_bytes(w, h):
    def chunk(t, data):
        return len(data).to_bytes(4, "big") + t + data + (zlib.crc32(t + data) & 0xFFFFFFFF).to_bytes(4, "big")
    ihdr = w.to_bytes(4, "big") + h.to_bytes(4, "big") + bytes([8, 2, 0, 0, 0])
    return b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", ihdr) + chunk(b"IEND", b"")


def calib_text(d):
    return "".join("%s: %s\n" % kv for kv in d.items()) + "calib_time: 09-Jan-2012 13:57:47\n"


def label_line(t, box, trunc=0.0, occ=0):
    x, y, z, l, h, w, ry = box
    return "%s %.2f %d %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f" % (t, trunc, occ, -1.57, 100.0, 150.0, 300.0,
                                                                                     250.0, h, w, l, x, y, z, ry)


DONTCARE = "DontCare -1 -1 -10 503.89 169.71 590.61 190.13 -1 -1 -1 -1000 -1000 -1000 -10"


def velo_of_rect(r):
    """Velodyne coordinates whose exact-calibration rect image is r (x_r = -y_v, y_r = -z_v, z_r = x_v)."""
    r = np.asarray(r, np.float32).reshape(-1, 3)
    return np.stack([r[:, 2], -r[:, 0], -r[:, 1]], 1)


def with_i(v, rng):
    return np.concatenate([v, rng.uniform(0, 1, (len(v), 1))], 1).astype(np.float32)


def cluster(centre, n, rng, spread=(0.6, 0.4, 1.2)):
    return centre + rng.uniform(-1, 1, (n, 3)) * np.asarray(spread)


def build_frames(rng):
    """[(kitti id, split, velodyne [N, 4] float32, calib text, (H, W), label text or None)]"""
    scan = np.loadtxt(os.path.join(os.path.dirname(REF), "mayavi", "kitti_sample_scan.txt"), dtype=np.float32)
    scan = scan[np.sort(rng.choice(len(scan), 10000, replace=False))]
    real = with_i(scan, rng)
    frames = []
    # 0, 1: the real scan; Car rows on clusters of the scan in front of the camera, a Van and a DontCare
    rect = np.stack([-scan[:, 1], -scan[:, 2], scan[:, 0]], 1)            # roughly, to place the boxes
    front = np.flatnonzero((rect[:, 2] > 6) & (rect[:, 2] < 35) & (np.abs(rect[:, 0]) < 0.6 * rect[:, 2]))
    for fid, hw in ((7, (375, 1242)), (3, (370, 1224))):
        pick = rect[rng.choice(front, 3, replace=False)]
        lines = [label_line("Car", (p[0], p[1] + 0.8, p[2], 3.9, 1.6, 1.7, rng.uniform(-3, 3))) for p in pick]
        q = rect[rng.choice(front)]
        lines.insert(1, label_line("Van", (q[0], q[1] + 1.0, q[2], 5.0, 2.0, 1.9, 0.3)))
        lines.append(DONTCARE)
        frames.append((fid, "training", real, calib_text(KITTI_CALIB), hw, "\n".join(lines) + "\n"))
    # 2: exact boundaries (W = 512, H = 256: u = 256 x / z + 256, v = 256 y / z + 128)
    on = [(-8, 1, 8), (8, 1, 8), (0, -4, 8), (0, 4, 8), (0, 0, 0), (1, 1, 0), (3, 1, -0.0),   # u = 0, u = W, v = 0, v = H, z = 0
          (-40, 1, 64), (40, 1, 64), (-39.999996, 1, 64), (39.999996, 1, 64),               # x extents (and just inside)
          (0, -5, 16), (0, 3, 16), (0, -4.9999995, 16), (0, 2.9999998, 16),                  # y extents
          (0, 1, 70), (0, 1, 69.99999), (-8.000001, 1, 8), (7.999999, 1, 8)]
    box = (2.0, 1.5, 20.0, 4.0, 1.5, 2.0, 0.0)
    inside = cluster(np.array([2.0, 0.8, 20.0]), 30, rng, (1.5, 0.5, 0.7))
    frames.append((12, "training", with_i(velo_of_rect(np.concatenate([np.asarray(on, np.float64), inside])), rng),
                   calib_text(EXACT_CALIB), (256, 512), label_line("Car", box) + "\n" + DONTCARE + "\n"))
    # 3: no Car
    pts = with_i(velo_of_rect(cluster(np.array([0.0, 0.8, 15.0]), 50, rng)), rng)
    frames.append((5, "training", pts, calib_text(EXACT_CALIB), (256, 512),
                   label_line("Van", (0.0, 1.5, 15.0, 5.0, 2.0, 1.9, 0.0)) + "\n" + DONTCARE + "\n"))
    # 4: Cars that hold no kept point (one behind the camera)
    pts = with_i(velo_of_rect(np.concatenate([cluster(np.array([0.0, 0.8, 15.0]), 50, rng),
                                              cluster(np.array([0.0, 0.8, -10.0]), 20, rng)])), rng)
    frames.append((9, "training", pts, calib_text(EXACT_CALIB), (256, 512),
                   label_line("Car", (6.0, 1.5, 30.0, 3.9, 1.6, 1.7, 0.4)) + "\n" +
                   label_line("Car", (0.0, 1.5, -10.0, 3.9, 1.6, 1.7, 0.0)) + "\n"))
    # 5: a Car with 3 points (below MIN_POINTS_NUM) and one with 40
    pts = with_i(velo_of_rect(np.concatenate([cluster(np.array([-5.0, 0.8, 25.0]), 3, rng, (0.5, 0.3, 0.5)),
                                              cluster(np.array([5.0, 0.8, 25.0]), 40, rng), cluster(np.array([0.0, 0.0, 50.0]), 60, rng,
                                                                                                     (20, 1, 15))])), rng)
    frames.append((1, "training", pts, calib_text(EXACT_CALIB), (256, 512),
                   label_line("Car", (-5.0, 1.5, 25.0, 3.9, 1.6, 1.7, 0.2)) + "\n" +
                   label_line("Car", (5.0, 1.5, 25.0, 3.9, 1.6, 1.7, -0.3)) + "\n"))
    # testing split, no GT: the real scan again
    frames.append((4, "testing", real, calib_text(KITTI_CALIB), (375, 1242), None))
    return frames


def write_tree(root, frames):
    for fid, split, pts, calib, hw, label in frames:
        d = os.path.join(root, split)
        for sub in ("velodyne", "calib", "image_2", "label_2"):
            os.makedirs(os.path.join(d, sub), exist_ok=True)
        pts.astype(np.float32).tofile(os.path.join(d, "velodyne", "%06d.bin" % fid))
        open(os.path.join(d, "calib", "%06d.txt" % fid), "w").write(calib)
        open(os.path.join(d, "image_2", "%06d.png" % fid), "wb").write(png_bytes(hw[1], hw[0]))
        if label is not None:
            open(os.path.join(d, "label_2", "%06d.txt" % fid), "w").write(label)


def reference_env(root, split, shapes):
    npx = NumpyProxy()
    env = {"np": npx, "numba": types.SimpleNamespace(jit=MGA._jit, njit=MGA._jit), "os": os}
    maps = {}
    exec(compile(open(os.path.join(REF, "dataset", "maps_dict.py")).read(), "maps_dict.py", "exec"), maps)
    env["maps_dict"] = types.SimpleNamespace(**{k: v for k, v in maps.items() if k.startswith("KEY_")})
    MGA.pull(os.path.join(REF, "utils", "kitti_util.py"), {"Calibration", "inverse_rigid_trans", "Object3d", "read_label",
                                                          "load_velo_scan"}, env)
    MGA.pull(os.path.join(REF, "utils", "points_filter.py"), {"get_point_filter", "get_point_filter_in_image"}, env)
    MGA.pull(os.path.join(REF, "utils", "voxelnet_aug.py"), MGM.CORNER_CHAIN, env)
    b3 = {"np": npx}
    MGA.pull(os.path.join(REF, "utils", "box_3d_utils.py"), {"object_label_to_box_3d"}, b3)
    env["box_3d_utils"] = types.SimpleNamespace(object_label_to_box_3d=b3["object_label_to_box_3d"])
    env["cv2"] = types.SimpleNamespace(COLOR_BGR2RGB=4, cvtColor=lambda img, code: img)
    ns = types.SimpleNamespace
    env["cfg"] = ns(TRAIN=ns(AUGMENTATIONS=ns(EXPAND_DIMS_LENGTH=0.1)), DATASET=ns(MIN_POINTS_NUM=5, POINT_CLOUD_RANGE=EXTENTS),
                    TEST=ns(WITH_GT=True))
    sd = os.path.join(root, split)
    env["kitti_object"] = ns(
        get_image=lambda i: np.zeros(shapes[i] + (3,), np.uint8),
        get_calibration=lambda i: env["Calibration"](os.path.join(sd, "calib", "%06d.txt" % i)),
        get_lidar=lambda i: env["load_velo_scan"](os.path.join(sd, "velodyne", "%06d.bin" % i)),
        get_label_objects=lambda i: env["read_label"](os.path.join(sd, "label_2", "%06d.txt" % i)))
    path = os.path.join(REF, "dataset", "dataloader", "kitti_dataloader.py")
    pre = MGM.pull_method(path, "KittiDataset", "preprocess_samples", env)
    gen = MGM.pull_method(path, "KittiDataset", "generate_mixup_sample", env)
    return env, pre, gen


def instance(env, ids, img_list):
    me = object.__new__(type("KittiDataset", (), {}))
    me.idx_list = ["%06d" % i for i in ids]
    me.kitti_object = env["kitti_object"]
    me.extents = np.reshape(EXTENTS, [3, 2])
    me.img_list = img_list
    me.cls_list = ("Car",)
    me.idx2cls_dict = {1: "Car"}
    me.cls2idx_dict = {"Car": 1}
    return me


def margins(env, pts, calib_path, hw, boxes):
    """float64 margins of each point to the nearest filter bound and (for boxes) to the nearest grown box face."""
    cal = env["Calibration"](calib_path)
    rect = cal.project_velo_to_rect(pts[:, :3])
    with np.errstate(divide="ignore", invalid="ignore"):
        uv = cal.project_rect_to_image(rect)
    H, W = hw
    e = np.asarray(EXTENTS, np.float64)
    d = np.stack([uv[:, 0], uv[:, 0] - W, uv[:, 1], uv[:, 1] - H, rect[:, 2], rect[:, 0] - e[0], rect[:, 0] - e[1],
                  rect[:, 1] - e[2], rect[:, 1] - e[3], rect[:, 2] - e[4], rect[:, 2] - e[5]], 1)
    filt = np.nan_to_num(np.abs(d), nan=0.0).min(1)
    face = np.full(len(pts), np.inf)
    for b in boxes:
        l, h, w = b[3] + 0.1, b[4] + 0.1, b[5] + 0.1
        c, s = np.cos(b[6]), np.sin(b[6])
        q = rect - b[:3]
        cx, cz = c * q[:, 0] - s * q[:, 2], s * q[:, 0] + c * q[:, 2]
        face = np.minimum(face, np.abs(np.stack([cx - l / 2, cx + l / 2, q[:, 1], q[:, 1] + h, cz - w / 2, cz + w / 2], 1)).min(1))
    return filt, face


def main():
    rng = np.random.default_rng(2028)
    frames = build_frames(rng)
    root = tempfile.mkdtemp()
    write_tree(root, frames)
    train = [f for f in frames if f[1] == "training"]
    test = [f for f in frames if f[1] == "testing"]
    out = dict(extents=np.asarray(EXTENTS, np.float64))
    rec = {k: [] for k in ("points", "sem", "boxes", "classes", "p2", "filter_margin", "face_margin")}
    kept_flags, names, lines, db_pts, db_off, db_boxes, db_src = [], [], [], [], [0], [], []
    env, pre, gen = reference_env(root, "training", {f[0]: f[4] for f in train})
    me = instance(env, [f[0] for f in train], "train")
    for i, (fid, _, pts, calib, hw, label) in enumerate(train):
        dicts, _ = pre(me, [i])
        K = env["maps_dict"]
        filt, _ = margins(env, pts, os.path.join(root, "training", "calib", "%06d.txt" % fid), hw, [])
        rec["filter_margin"].append(filt)
        if dicts is None:
            kept_flags.append(0)
            print("frame %d (id %d): skipped" % (i, fid))
            continue
        d = dicts[0]
        kept_flags.append(1)
        lines.append("%06d.npy" % i)
        names.append(d[K.KEY_SAMPLE_NAME])
        _, face = margins(env, pts, os.path.join(root, "training", "calib", "%06d.txt" % fid), hw, d[K.KEY_LABEL_BOXES_3D])
        cal = env["Calibration"](os.path.join(root, "training", "calib", "%06d.txt" % fid))
        keep = env["get_point_filter_in_image"](cal.project_velo_to_rect(pts[:, :3]), cal, hw[0], hw[1]) & \
            env["get_point_filter"](cal.project_velo_to_rect(pts[:, :3]), np.reshape(EXTENTS, [3, 2]))
        rec["face_margin"].append(face[keep])
        rec["points"].append(d[K.KEY_POINT_CLOUD])
        rec["sem"].append(d[K.KEY_LABEL_SEMSEG])
        rec["boxes"].append(d[K.KEY_LABEL_BOXES_3D])
        rec["classes"].append(d[K.KEY_LABEL_CLASSES])
        rec["p2"].append(d[K.KEY_STEREO_CALIB].P)
        assert d[K.KEY_LABEL_NUM] == len(d[K.KEY_LABEL_BOXES_3D]) and np.all(d[K.KEY_LABEL_DIST] == 1)
        for obj in gen(me, d) or []:
            db_pts.append(obj[K.KEY_SAMPLED_GT_POINTS])
            db_off.append(db_off[-1] + len(obj[K.KEY_SAMPLED_GT_POINTS]))
            db_boxes.append(obj[K.KEY_SAMPLED_GT_LABELS_3D])
            row = [j for j, b in enumerate(d[K.KEY_LABEL_BOXES_3D]) if np.array_equal(b, obj[K.KEY_SAMPLED_GT_LABELS_3D])][0]
            db_src.append((i, row))
        print("frame %d (id %d): %d -> %d points, %d boxes, %d positive" % (i, fid, len(pts), len(d[K.KEY_POINT_CLOUD]),
                                                                            len(d[K.KEY_LABEL_BOXES_3D]), int((d[K.KEY_LABEL_SEMSEG] > 0).sum())))
    # the testing frame without GT
    env_t, pre_t, _ = reference_env(root, "testing", {f[0]: f[4] for f in test})
    env_t["cfg"].TEST.WITH_GT = False
    dt, _ = pre_t(instance(env_t, [f[0] for f in test], "test"), [0])
    K = env_t["maps_dict"]
    cat = lambda a: np.concatenate(a) if a else np.zeros(0)
    off = lambda a: np.concatenate([[0], np.cumsum([len(x) for x in a])]).astype(np.int64)
    out.update(
        frame_ids=np.asarray([f[0] for f in frames]), frame_split=np.asarray([f[1] for f in frames]),
        velodyne=np.concatenate([f[2] for f in frames]), velodyne_offsets=off([f[2] for f in frames]),
        calib_texts=np.asarray([f[3] for f in frames]), image_hw=np.asarray([f[4] for f in frames], np.int64),
        label_texts=np.asarray([f[5] or "" for f in frames]),
        ref_kept=np.asarray(kept_flags, np.int32), ref_train_list=np.asarray(lines), ref_names=np.asarray(names, np.int64),
        ref_points=cat(rec["points"]), ref_point_offsets=off(rec["points"]), ref_sem=cat(rec["sem"]).astype(np.int64),
        ref_boxes=cat(rec["boxes"]).reshape(-1, 7), ref_box_offsets=off(rec["boxes"]), ref_classes=cat(rec["classes"]).astype(np.int64),
        ref_p2=np.stack(rec["p2"]), filter_margin=cat(rec["filter_margin"]), face_margin=cat(rec["face_margin"]),
        ref_db_points=np.concatenate(db_pts), ref_db_offsets=np.asarray(db_off, np.int64), ref_db_boxes=np.stack(db_boxes),
        ref_db_src=np.asarray(db_src, np.int32),
        ref_nogt_points=dt[0][K.KEY_POINT_CLOUD], ref_nogt_sem=np.asarray(dt[0][K.KEY_LABEL_SEMSEG], np.int64),
        ref_nogt_name=int(dt[0][K.KEY_SAMPLE_NAME]), ref_nogt_p2=dt[0][K.KEY_STEREO_CALIB].P)
    np.savez_compressed(os.path.join(HERE, "prepare.npz"), **out)
    print("wrote prepare.npz: %d frames, %d kept, %d database objects" % (len(frames), sum(kept_flags), len(db_boxes)))


if __name__ == "__main__":
    main()
