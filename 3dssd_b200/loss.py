"""Training targets and the detection loss of the shipped 3DSSD configuration (DESIGN.md section 3.8).

The two seams of the reference's training step, on the GPU:
  assign_targets   TargetAssigner.assign ('Mask', MINIBATCH_NUM -1)   /root/reference/lib/builder/target_assigner.py:147
                   + vote_targets_np                                  /root/reference/lib/np_functions/gt_sampler.py:28-61
  detection_loss   EncoderDecoder.encode + LossBuilder.forward        /root/reference/lib/builder/encoder_builder.py:45-77,
                   (cls, offset, angle, corner and vote losses)       /root/reference/lib/builder/loss_builder.py
                   and the sum trainer.py takes of them               /root/reference/lib/core/trainer.py:133-134
Both take the tensors head.box_regression_head and vote_layer return; the work is csrc/det_loss.cu.

    outs = backbone.train_forward(arch, tp, xyz, feat)
    tg = assign_targets(outs.base_xyz, outs.vote_base, gt_boxes, gt_labels)
    losses = detection_loss(outs.base_xyz, *outs.head, outs.vote_offset, tg)
    losses["total"].backward()
"""
from typing import NamedTuple

import torch

from . import tf_ops

# The one configuration built (configs/kitti/3dssd/3dssd.yaml:69-80 and lib/core/config.py).  All but the bin count are
# compiled into csrc/det_loss.cu (kExpand, kSampleRange, kCtrEps, the huber of delta 1); a test pins the two to agree.
ANGLE_CLS_NUM = 12                     # MODEL.ANGLE_CLS_NUM (3dssd.yaml:38)
EXPAND_DIMS_LENGTH = 0.1               # TRAIN.AUGMENTATIONS.EXPAND_DIMS_LENGTH (lib/core/config.py:84)
SOFTMAX_SAMPLE_RANGE = 10.0            # FIRST_STAGE.CLASSIFICATION_LOSS.SOFTMAX_SAMPLE_RANGE (lib/core/config.py:329)
CENTER_NESS_LABEL_RANGE = (0.0, 1.0)   # FIRST_STAGE.CLASSIFICATION_LOSS.CENTER_NESS_LABEL_RANGE (lib/core/config.py:327)
CENTER_NESS_EPS = 1e-6                 # _generate_centerness_label(epsilon=1e-6) (lib/builder/loss_builder.py:99)
LOSS_NAMES = ("cls_loss", "offset_loss", "bin_angle_loss", "res_angle_loss", "corner_loss", "vote_loss")


class Targets(NamedTuple):
    """Per candidate point [b, n]: assigned_idx (int32), assigned_box [.., 7], pmask, nmask, cls_label (the centre-ness
    classification target), angle_bin (int32), angle_res, offset_target [.., 6]; per vote base point [b, nv]: vote_mask,
    vote_target [.., 3].  No gradient flows into any of them."""
    assigned_idx: torch.Tensor
    assigned_box: torch.Tensor
    pmask: torch.Tensor
    nmask: torch.Tensor
    cls_label: torch.Tensor
    angle_bin: torch.Tensor
    angle_res: torch.Tensor
    offset_target: torch.Tensor
    vote_mask: torch.Tensor
    vote_target: torch.Tensor


def assign_targets(base_xyz, vote_base, gt_boxes, gt_labels):
    """base_xyz (b, n, 3) candidate points (the CG layer's centres), vote_base (b, nv, 3) the vote layer's input points,
    gt_boxes (b, g, 7) camera-frame (x, y, z, l, h, w, ry) padded with rows of zeros, gt_labels (b, g) -> Targets.
    A scene without a valid box gives all negatives and zero targets (include/ssd3d.h, ssd3d_det_assign)."""
    labels = gt_labels if isinstance(gt_labels, torch.Tensor) and gt_labels.dtype == torch.int32 else torch.as_tensor(
        gt_labels, device=base_xyz.device).to(torch.int32)
    with torch.no_grad():
        t = tf_ops.det_assign(base_xyz.detach(), vote_base.detach(), gt_boxes, labels, ANGLE_CLS_NUM)
    return Targets(**t)


def detection_loss(base_xyz, pred_cls, pred_offset, pred_angle_cls, pred_angle_res, vote_offset, targets):
    """The six losses of the 3DSSD head on `targets` -> dict of 0-d device tensors named LOSS_NAMES plus "total", their
    sum.  Differentiable w.r.t. base_xyz, the four head outputs (read in place) and the raw vote offsets."""
    loss = tf_ops.det_loss_train(base_xyz, pred_cls, pred_offset, pred_angle_cls, pred_angle_res, vote_offset,
                                 targets._asdict(), ANGLE_CLS_NUM)
    out = {name: loss[i] for i, name in enumerate(LOSS_NAMES)}
    out["total"] = loss.sum()
    return out
