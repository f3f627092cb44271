"""numpy restatement of the class-count forms of csrc/det_loss.cu (include/ssd3d.h: ssd3d_det_assign_classes,
ssd3d_det_loss_classes, ssd3d_det_loss_grad_classes), built on the single-class oracle oracle/det_loss.py, whose
functions it calls unchanged for everything the class count does not touch:
  assign        the class-agnostic targets of oracle/det_loss.assign, and cls_label [B, N, C]: for a positive whose
                assigned box has label k in 1..C, column k - 1 holds its centre-ness label (oracle/det_loss.centerness),
                every other entry is 0 (a label outside 1..C gives a zero row and the point stays a positive);
  losses        loss (6,) and norm (3,): the classification term is sum over rows of cls_mask * (sum over the classes in
                order of the sigmoid cross-entropy) / C over max(1, sum of cls_mask), in float64; the other five terms
                and the norms are oracle/det_loss.losses' (they do not read the class columns);
  cls_grad      the gradient of the classification term w.r.t. pred_cls [B, N, C] for a loss gradient g0:
                (sigmoid(x_c) - label_c) * cls_mask * (g0 / norm) / C, in float64.
At C = 1 each is the single-class oracle's recipe."""
import numpy as np

from oracle import det_loss as odl


def assign(base_xyz, vote_base, gt_boxes, gt_labels, cls_num, nbins=12):
    out = odl.assign(base_xyz, vote_base, gt_boxes, gt_labels, nbins)       # labels reach only cls_label, replaced below
    B, N = base_xyz.shape[:2]
    lab = np.zeros((B, N, cls_num), np.float32)
    idx, pos = out["assigned_idx"], out["pmask"] > 0
    for s in range(B):
        for p in np.nonzero(pos[s])[0]:
            k = int(gt_labels[s, idx[s, p]])
            if 1 <= k <= cls_num:
                lab[s, p, k - 1] = odl.centerness(base_xyz[s, p].astype(np.float32), gt_boxes[s, idx[s, p]].astype(np.float32))
    out["cls_label"] = lab
    return out


def _cls_term(pred_cls, tg, cls_num):
    B, N = tg["pmask"].shape
    x = np.asarray(pred_cls, np.float64).reshape(B, N, -1)[..., :cls_num]
    z = np.asarray(tg["cls_label"], np.float64).reshape(B, N, cls_num)
    cm = tg["pmask"].astype(np.float64) + tg["nmask"].astype(np.float64)
    return x, z, cm


def losses(base_xyz, pred_cls, pred_offset, pred_angle_cls, pred_angle_res, vote_offset, tg, cls_num, nbins=12):
    x, z, cm = _cls_term(pred_cls, tg, cls_num)
    ce = np.zeros(cm.shape)
    for c in range(cls_num):                                               # the classes in order
        ce += np.maximum(x[..., c], 0) - x[..., c] * z[..., c] + np.log1p(np.exp(-np.abs(x[..., c])))
    rest = dict(tg, cls_label=np.zeros(cm.shape, np.float32))             # the single-class oracle for the other terms
    loss, norm = odl.losses(base_xyz, np.zeros(cm.shape + (1,), np.float32), pred_offset, pred_angle_cls, pred_angle_res,
                            vote_offset, rest, nbins)
    loss = np.array(loss, np.float64)
    loss[0] = (ce / cls_num * cm).sum(1).sum(0) / norm[0]
    return loss, norm


def cls_grad(pred_cls, tg, cls_num, g0, norm0):
    x, z, cm = _cls_term(pred_cls, tg, cls_num)
    return (1.0 / (1.0 + np.exp(-x)) - z) * cm[..., None] * (np.float64(g0) / np.float64(norm0)) / cls_num
