"""numpy restatement of the KITTI preprocessing pass (csrc/prepare.cu + 3dssd_b200/prepare.py, DESIGN.md section 3.14),
operation by operation: the velo -> rect -> image transform in the canonical order of include/ssd3d.h with elementwise
float64 products and sums (no matrix product, so no BLAS order), the image-FOV and extents filters, the semantic labels
of oracle/augment.py on the float32 cast, the two skip rules and the sample dicts, and the mixup database of
oracle/mixup.py.  The reference's own preprocessing is held to it by tests/golden/prepare.npz."""
import numpy as np

from oracle import augment as OA
from oracle import mixup as OM

f32, f64 = np.float32, np.float64
EXTENTS = (-40.0, 40.0, -5.0, 3.0, 0.0, 70.0)


def transform(points, calib):
    """points [N, 4] float32, calib [33] float64 -> (rect [N, 3], u [N], v [N]) float64."""
    p = np.asarray(points, f32).astype(f64)
    c = np.asarray(calib, f64)
    V, R, P = c[:12].reshape(3, 4), c[12:21].reshape(3, 3), c[21:].reshape(3, 4)
    x, y, z = p[:, 0], p[:, 1], p[:, 2]
    ref = [((x * V[j, 0] + y * V[j, 1]) + z * V[j, 2]) + V[j, 3] for j in range(3)]
    rect = [(R[i, 0] * ref[0] + R[i, 1] * ref[1]) + R[i, 2] * ref[2] for i in range(3)]
    h = [((rect[0] * P[k, 0] + rect[1] * P[k, 1]) + rect[2] * P[k, 2]) + P[k, 3] for k in range(3)]
    with np.errstate(divide="ignore", invalid="ignore"):
        u, v = h[0] / h[2], h[1] / h[2]
    return np.stack(rect, 1), u, v


def keep_mask(rect, u, v, hw, extents=EXTENTS):
    H, W = (f64(a) for a in hw)
    e = np.asarray(extents, f64)
    with np.errstate(invalid="ignore"):
        img = (u >= 0) & (u < W) & (v >= 0) & (v < H) & (rect[:, 2] >= 0)
        box = ((rect[:, 0] > e[0]) & (rect[:, 0] < e[1]) & (rect[:, 1] > e[2]) & (rect[:, 1] < e[3]) & (rect[:, 2] > e[4]) &
               (rect[:, 2] < e[5]))
    return img & box


def kept_points(points, calib, hw, extents=EXTENTS):
    """One frame's kept points [K, 4] float64 (rect x, y, z, intensity) in input order."""
    rect, u, v = transform(points, calib)
    m = keep_mask(rect, u, v, hw, extents)
    return np.concatenate([rect[m], np.asarray(points, f32)[m, 3:4].astype(f64)], 1)


def prepare_points(points, offsets, calib, image_hw, extents=EXTENTS):
    """The kernel's outputs on a batch: (kept [T', 4] float64, kept_offsets [B + 1] int32)."""
    off = np.asarray(offsets, np.int64)
    parts = [kept_points(points[off[s]:off[s + 1]], calib[s], image_hw[s], extents) for s in range(len(off) - 1)]
    return (np.concatenate(parts) if parts else np.zeros((0, 4), f64),
            np.concatenate([[0], np.cumsum([len(q) for q in parts])]).astype(np.int32))


def frame_dict(i, name, points, calib, hw, boxes=None, classes=None, extents=EXTENTS):
    """preprocess_samples of one frame at list position i (KITTI id `name`): the sample dict, or (None, reason) when
    it is skipped ('no_objects': no object of the class list, 'no_points': no positive semantic label)."""
    kept = kept_points(points, calib, hw, extents)
    if boxes is not None:
        if len(boxes) == 0:
            return None, "no_objects"
        sem = OA.sem_labels(kept.astype(f32), np.asarray(boxes, f32), np.asarray(classes, np.int32)).astype(np.int64)
    else:
        sem = np.ones(len(kept), np.int64)
    if sem.sum() == 0:
        return None, "no_points"
    d = {"point_cloud": kept, "label_sem_seg": sem, "label_dist": np.ones(len(kept), f32),
         "stereo_calib": np.asarray(calib, f64)[21:].reshape(3, 4).copy(), "sample_name": int(name)}
    if boxes is not None:
        d.update(label_boxes_3d=np.asarray(boxes, f64).reshape(-1, 7), label_classes=np.asarray(classes, np.int64),
                 label_num=len(boxes))
    return d, None


def prepare(frames, extents=EXTENTS, mixup=False):
    """frames: list of (name, points [N, 4] float32, calib [33], (H, W), boxes [G, 7] | None, classes [G] | None) in list
    order.  -> (dicts {position: sample dict}, skipped {position: reason}, train_list lines, mixup database dict or None
    with frames = the file number of each object)."""
    dicts, skipped = {}, {}
    for i, (name, pts, calib, hw, boxes, classes) in enumerate(frames):
        d, why = frame_dict(i, name, pts, calib, hw, boxes, classes, extents)
        if d is None:
            skipped[i] = why
        else:
            dicts[i] = d
    lines = ["%06d.npy" % i for i in sorted(dicts)]
    db = None
    if mixup:
        keys = sorted(dicts)
        if keys:
            pts = [dicts[k]["point_cloud"].astype(f32) for k in keys]
            off = np.concatenate([[0], np.cumsum([len(p) for p in pts])])
            G = max(len(dicts[k]["label_boxes_3d"]) for k in keys)
            bx, lb = np.zeros((len(keys), G, 7), f32), np.zeros((len(keys), G), np.int32)
            for r, k in enumerate(keys):
                g = len(dicts[k]["label_boxes_3d"])
                bx[r, :g], lb[r, :g] = dicts[k]["label_boxes_3d"], dicts[k]["label_classes"]
            db = OM.build_db(np.concatenate(pts), off, bx, lb)
            db["frames"] = np.asarray(keys, np.int32)[db["frames"]]
        else:
            db = OM.build_db(np.zeros((0, 4), f32), np.zeros(1, np.int64), np.zeros((0, 0, 7), f32), np.zeros((0, 0), np.int32))
    return dicts, skipped, lines, db
