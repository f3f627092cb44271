"""Deterministic synthetic inputs (there is no dataset in this environment).

kitti_like(): the "synthetic KITTI" distribution of SURVEY.md section 8d / BASELINE.md 2c -- rect camera frame,
range of /root/reference/configs/kitti/3dssd/3dssd.yaml:3, 16384 points per scene like the reference loader
(lib/dataset/dataloader/kitti_dataloader.py:137-147), INCLUDING its duplicate padding: the loader re-samples
with replacement when a scan has fewer points, so exact duplicates (FPS / ball-query ties) are part of the
input distribution.
"""
import numpy as np


def kitti_like(batch, npoints=16384, seed=1000, dup_frac=0.02):
    out = np.empty((batch, npoints, 4), np.float32)
    for s in range(batch):
        rng = np.random.default_rng(seed + s)
        x = rng.uniform(-40.0, 40.0, npoints)
        z = 70.0 * rng.uniform(0.0, 1.0, npoints) ** 2            # denser near the sensor
        ground = rng.uniform(0.0, 1.0, npoints) < 0.7
        y = np.where(ground, 1.65 + 0.05 * rng.standard_normal(npoints), rng.uniform(-1.0, 1.6, npoints))
        inten = rng.uniform(0.0, 1.0, npoints)
        pts = np.stack([x, y, z, inten], axis=1).astype(np.float32)
        ndup = int(round(dup_frac * npoints))
        if ndup:
            src = rng.integers(0, npoints - ndup, ndup)
            pts[npoints - ndup:] = pts[src]                       # duplicate padding at the tail
        out[s] = pts
    return out


def uniform_cube(batch, npoints, channels=0, seed=0):
    """U(0,1)^3 coordinates (+ N(0,1) features), the distribution of the reference's own op test
    (lib/utils/tf_ops/grouping/tf_grouping_op_test.py:11-14)."""
    rng = np.random.default_rng(seed)
    xyz = rng.uniform(0.0, 1.0, (batch, npoints, 3)).astype(np.float32)
    if channels == 0:
        return xyz
    feat = rng.standard_normal((batch, npoints, channels)).astype(np.float32)
    return np.concatenate([xyz, feat], axis=-1)


def lattice(batch, npoints, step=0.25, seed=0):
    """Points on a coarse lattice: many exactly equal distances and exact duplicates -- adversarial for
    arg-max tie-breaking (FPS) and for the d == 0 / d == r boundaries of the ball queries."""
    rng = np.random.default_rng(seed)
    g = rng.integers(0, 12, (batch, npoints, 3)).astype(np.float32) * np.float32(step)
    return g


CAR_SIZE = ((3.2, 4.7), (1.4, 1.8), (1.5, 1.9))     # (l, h, w) ranges in metres


def kitti_like_with_boxes(batch, npoints, max_boxes, seed=0, surface_frac=0.3):
    """KITTI-like scenes with car-sized boxes, for training: (points [B, npoints, 4] fp32, gt_boxes [B, max_boxes, 7]
    fp32 camera-frame (x, y, z, l, h, w, ry) with the box standing on the ground at y ~ 1.65, zero-padded past each
    scene's box count, gt_labels [B, max_boxes] int32, 1 for a box and 0 for padding).  About surface_frac of the points
    lie on the boxes' side and top faces, the way a scan hits a car, and a few inside them.  The angles mix uniform
    draws in [-pi, pi), the edges of the 12 angle bins and +-pi."""
    pts = kitti_like(batch, npoints, seed=seed)
    boxes = np.zeros((batch, max_boxes, 7), np.float32)
    labels = np.zeros((batch, max_boxes), np.int32)
    per = 2 * np.pi / 12
    edges = np.concatenate([np.arange(12) * per - per / 2, [np.pi, -np.pi]])
    for s in range(batch):
        rng = np.random.default_rng(seed + 7919 * (s + 1))
        g = int(rng.integers(max(1, max_boxes // 2), max_boxes + 1)) if max_boxes else 0
        for j in range(g):
            l, h, w = (rng.uniform(lo, hi) for lo, hi in CAR_SIZE)
            ry = edges[rng.integers(len(edges))] if rng.uniform() < 0.3 else rng.uniform(-np.pi, np.pi)
            boxes[s, j] = (rng.uniform(-30, 30), 1.65 + 0.05 * rng.standard_normal(), rng.uniform(4, 60), l, h, w, ry)
            labels[s, j] = 1
        if g == 0:
            continue
        k = int(round(surface_frac * npoints))
        owner = rng.integers(0, g, k)
        b = boxes[s, owner].astype(np.float64)
        u = rng.uniform(-0.5, 0.5, (k, 3))                    # canonical (x / l, y / h, z / w)
        face = rng.integers(0, 6, k)                          # 0..3: a side, 4: the top, 5: inside
        u[face == 0, 0], u[face == 1, 0] = 0.5, -0.5
        u[face == 2, 2], u[face == 3, 2] = 0.5, -0.5
        u[face == 4, 1] = -0.5
        u[face == 5] *= 0.9
        cx, cy, cz = u[:, 0] * b[:, 3], (u[:, 1] - 0.5) * b[:, 4], u[:, 2] * b[:, 5]
        c, sn = np.cos(b[:, 6]), np.sin(b[:, 6])              # get_box3d_corners_helper's rotation (box_3d_utils.py)
        at = rng.choice(npoints, k, replace=False)
        pts[s, at, 0] = c * cx + sn * cz + b[:, 0]
        pts[s, at, 1] = cy + b[:, 1]
        pts[s, at, 2] = -sn * cx + c * cz + b[:, 2]
    return pts, boxes, labels


def kitti_like_multiclass(batch, npoints, max_boxes, classes=("Car", "Pedestrian", "Cyclist"), seed=0, surface_frac=0.3):
    """kitti_like_with_boxes for several classes: each box draws a class of `classes` (names of config.CLASS_MEAN_SIZE)
    uniformly, its label is the class's 1-based place in `classes`, and its (l, h, w) lies within +-15 % of the class's
    mean size (g_type_mean_size, lib/utils/model_util.py:19-26).  Same points-on-the-boxes recipe; a random stream of its
    own (kitti_like_with_boxes is left as it is)."""
    from .config import CLASS_MEAN_SIZE, check_cls_list
    classes = check_cls_list(classes)
    pts = kitti_like(batch, npoints, seed=seed)
    boxes = np.zeros((batch, max_boxes, 7), np.float32)
    labels = np.zeros((batch, max_boxes), np.int32)
    for s in range(batch):
        rng = np.random.default_rng(seed + 104729 * (s + 1))
        g = int(rng.integers(max(1, max_boxes // 2), max_boxes + 1)) if max_boxes else 0
        for j in range(g):
            k = int(rng.integers(len(classes)))
            l, h, w = (m * rng.uniform(0.85, 1.15) for m in CLASS_MEAN_SIZE[classes[k]])
            boxes[s, j] = (rng.uniform(-30, 30), 1.65 + 0.05 * rng.standard_normal(), rng.uniform(4, 60), l, h, w,
                           rng.uniform(-np.pi, np.pi))
            labels[s, j] = k + 1
        if g == 0:
            continue
        kpts = int(round(surface_frac * npoints))
        owner = rng.integers(0, g, kpts)
        b = boxes[s, owner].astype(np.float64)
        u = rng.uniform(-0.5, 0.5, (kpts, 3))
        face = rng.integers(0, 6, kpts)                       # 0..3: a side, 4: the top, 5: inside
        u[face == 0, 0], u[face == 1, 0] = 0.5, -0.5
        u[face == 2, 2], u[face == 3, 2] = 0.5, -0.5
        u[face == 4, 1] = -0.5
        u[face == 5] *= 0.9
        cx, cy, cz = u[:, 0] * b[:, 3], (u[:, 1] - 0.5) * b[:, 4], u[:, 2] * b[:, 5]
        c, sn = np.cos(b[:, 6]), np.sin(b[:, 6])
        at = rng.choice(npoints, kpts, replace=False)
        pts[s, at, 0] = c * cx + sn * cz + b[:, 0]
        pts[s, at, 1] = cy + b[:, 1]
        pts[s, at, 2] = -sn * cx + c * cz + b[:, 2]
    return pts, boxes, labels
