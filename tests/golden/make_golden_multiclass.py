"""Generates tests/golden/multiclass_targets.npz: the reference's class-aware classification targets at C = 3.

The scenes are those of make_golden_det_targets.py with labels 1..3 on the valid rows and one row labelled 4 per scene
(outside the class list).  The class-agnostic targets come from the REFERENCE's own numpy functions, pulled out of their
source files with `ast` as make_golden_det_targets.py does (mask_assign_targets_anchors_np, vote_targets_np).  The
class target follows the reference's graph, whose TensorFlow ops are restated in numpy:
  assigned_gt_labels = gather(gt_labels, assigned_idx) * pmask         lib/builder/target_assigner.py:57-59
  gt_cls = one_hot(assigned_gt_labels - 1, depth=3)                   lib/builder/loss_builder.py:73-74 (tf.one_hot: an
                                                                      index outside 0..2 gives a row of zeros)
  ctr_ness = _generate_centerness_label(base_xyz, assigned boxes, pmask)   loss_builder.py:99-137 (float64 here)
  cls_label = gt_cls * ctr_ness                                       loss_builder.py:87-88
Each point's float64 distance to the nearest face plane is recorded so a test can leave out the points a float32
rounding may put on either side.
Needs a reference checkout (path in $REFERENCE):   REFERENCE=<checkout> python tests/golden/make_golden_multiclass.py
"""
import importlib.util
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
C = 3


def _targets_module():
    spec = importlib.util.spec_from_file_location("make_golden_det_targets", os.path.join(HERE, "make_golden_det_targets.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def centerness(base, boxes, pmask, eps=1e-6):
    """_generate_centerness_label (loss_builder.py:99-137) in float64, CENTER_NESS_LABEL_RANGE (0, 1)."""
    e = base.astype(np.float64) - boxes[..., :3].astype(np.float64)
    ry = -boxes[..., 6].astype(np.float64)                 # rotate_points(canonical, -ry)
    c, s = np.cos(ry), np.sin(ry)
    cx, cy, cz = c * e[..., 0] + s * e[..., 2], e[..., 1], -s * e[..., 0] + c * e[..., 2]
    l, h, w = (boxes[..., k].astype(np.float64) for k in (3, 4, 5))
    fr, bk, bo, tp, le, ri = l / 2 - cx, cx + l / 2, -cy, cy + h, w / 2 - cz, cz + w / 2
    with np.errstate(divide="ignore", invalid="ignore"):
        cl = np.minimum(fr, bk) / np.maximum(fr, bk) * pmask
        cw = np.minimum(le, ri) / np.maximum(le, ri) * pmask
        ch = np.minimum(bo, tp) / np.maximum(bo, tp) * pmask
    return np.power(np.maximum(np.nan_to_num(cl * ch * cw, nan=0.0), eps), 1.0 / 3.0)


def main():
    T = _targets_module()
    env = T.reference_env()
    base, vote, boxes, labels = T.scenes()
    B, N, G = base.shape[0], base.shape[1], boxes.shape[1]
    valid = np.any(boxes != 0, -1)
    labels = np.where(valid, 1 + np.arange(G)[None] % C, 0).astype(np.int32)
    labels[:, 3] = np.where(valid[:, 3], C + 1, 0)            # outside the class list (box 3 overlaps box 0)
    ref = slice(0, B - 1)
    idx, pm, nm = (np.zeros((B, N), t) for t in (np.int32, np.float32, np.float32))
    i, p, n = env["mask_assign_targets_anchors_np"](base[ref], base[ref][:, :, None, :], boxes[ref], labels[ref], -1, 0.5, 0.6, 0.45,
                                                   10.0, np.ones((B - 1, N, 1), np.float32))
    idx[ref], pm[ref], nm[ref] = i[..., 0], p[..., 0], n[..., 0]
    nm[B - 1] = 1.0                                           # padded rows only: all negatives (by hand, as det_targets.npz)
    assigned = np.take_along_axis(labels, idx.astype(np.int64), 1) * pm.astype(np.int32)
    onehot = (assigned[..., None] - 1 == np.arange(C)).astype(np.float32)
    abox = np.take_along_axis(boxes, idx[..., None].astype(np.int64), 1)
    ctr = centerness(base, abox, pm)
    fdist = np.stack([T.face_distance(base[s], boxes[s], 0.0) for s in range(B)])
    np.savez_compressed(os.path.join(HERE, "multiclass_targets.npz"), base_xyz=base, vote_base=vote, gt_boxes=boxes,
                        gt_labels=labels, assigned_idx=idx, pmask=pm, nmask=nm, assigned_label=assigned.astype(np.int32),
                        one_hot=onehot, centerness=ctr, cls_label=onehot * ctr[..., None], face_dist=fdist)
    print("wrote multiclass_targets.npz: pos %d, by class %s, out-of-list positives %d"
          % (pm.sum(), [int(((assigned == k + 1) & (pm > 0)).sum()) for k in range(C)], int(((assigned == C + 1) & (pm > 0)).sum())))


if __name__ == "__main__":
    main()
