"""Detection head, box decoding and post-processing of the single-stage 3DSSD detector (SURVEY.md section 8f, rows f1/f2).

Mirrors, for inference with the shipped 3DSSD configuration (anchor-free 'Dist-Anchor-free' regression, sigmoid
classification over the classes of CLS_LIST (one by default), `HEAD: [[[6], [6], 'conv1d', [128,], True, 'Det', '']]`, configs/kitti/3dssd/3dssd.yaml:68):
  HeadBuilder.build_layer            /root/reference/lib/modeling/head_builder.py:81-114
  box_regression_head                /root/reference/lib/utils/head_util.py:26-59
  decode_dist_anchor_free            /root/reference/lib/utils/anchor_decoder.py:86-112
  decode_class2angle                 /root/reference/lib/utils/anchor_decoder.py:6-14
  SingleStageDetector.test_forward   /root/reference/lib/modeling/single_stage_detector.py:193-226 (sigmoid scores)
  PostProcessor.forward              /root/reference/lib/builder/postprocessor.py:52-120 (BEV NMS, IoU 0.1, max 100)
The convolutions run on the tensor-core path (tf_ops.linear_tc), the NMS on the GPU (tf_ops.bev_nms); the reference
runs tf.image.non_max_suppression on the CPU per scene and class.
"""
import math

import torch

from . import config as _cfg
from . import tf_ops
from .params import TrainableParams, prepare

ANGLE_CLS_NUM = 12          # MODEL.ANGLE_CLS_NUM (3dssd.yaml:38)
REG_CHANNELS = 6            # 'Dist-Anchor-free': distances to the 6 faces (head_builder.py:49-55)
MAX_OUTPUT_NUM = 100        # MODEL.FIRST_STAGE.MAX_OUTPUT_NUM (3dssd.yaml:70)
NMS_THRESH = 0.1            # MODEL.FIRST_STAGE.NMS_THRESH (3dssd.yaml:71)
HEAD_3DSSD = _cfg.HEAD_3DSSD


def reg_channels(stage):
    """pred_reg_channel_num of a regression method (head_builder.py:51-58), before the 2 * ANGLE_CLS_NUM angle channels."""
    if stage["REGRESSION"] == "Dist-Anchor-free":
        return REG_CHANNELS
    if stage["REGRESSION"] == "Bin-Anchor":
        return stage["BIN_CLASS_NUM"] * 4 + 4                 # bin_x / res_x / bin_z / res_z, res_y, 3 size residuals
    raise NotImplementedError("regression method %r" % (stage["REGRESSION"],))


def _scope(scope, name):
    return name if scope == '' else scope + "/" + name


def head_convs(pp, scope, bn, mlp, hi, lo, want_f32=False):
    """head_builder.py:93-113 at inference on the split features (hi, lo), on the tensor cores: one conv1d_i per width of
    `mlp`, then the pred_cls_base -> pred_cls and pred_reg_base -> pred_reg chains.  Returns (features, (cls, reg)):
    the last conv1d_i output in fp32 when want_f32 (None otherwise, or without conv1d_i), cls and reg in fp32."""
    y = None
    for i in range(len(mlp)):
        y, (hi, lo) = tf_ops.linear_tc(hi, lo, pp.conv(_scope(scope, "conv1d_%d" % i), bn), want_f32=want_f32, want_split=True)
    preds = []
    for name in ("pred_cls", "pred_reg"):
        _, (b_hi, b_lo) = tf_ops.linear_tc(hi, lo, pp.conv(_scope(scope, name + "_base"), bn), want_f32=False, want_split=True)
        preds.append(tf_ops.linear_tc(b_hi, b_lo, pp.conv(_scope(scope, name), False), relu=False)[0])
    return y, tuple(preds)


def box_regression_head(feature_input, pred_cls_channel, pred_reg_base_num, pred_reg_channel_num, bn, is_training, *,
                        params, scope='', bn_decay=None):
    """head_util.py:26-59 without the nuScenes attribute / velocity branches.  feature_input (bs, n, c) fp32.
    Returns (pred_cls (bs,n,cls), pred_offset (bs,n,base,6), pred_angle_cls (bs,n,base,12), pred_angle_res (...)).
    is_training=True needs params as a params.TrainableParams: both conv chains then run with batch-statistics BatchNorm
    through the differentiable tf_ops.conv_train, their BatchNorms with moving-statistics decay bn_decay (None: 0.9)."""
    bs, n, _ = feature_input.shape
    if is_training:
        if not isinstance(params, TrainableParams):
            raise NotImplementedError("is_training=True needs params.TrainableParams (the inference forms are folded)")
        chain = lambda base, pred: params.conv_train(_scope(scope, pred), params.conv_train(_scope(scope, base), feature_input, bn, bn_decay),
                                                     False, bn_decay, relu=False)
        pred_cls, pred_reg = chain("pred_cls_base", "pred_cls"), chain("pred_reg_base", "pred_reg")
    else:
        _, (pred_cls, pred_reg) = head_convs(prepare(params, feature_input.device), scope, bn, (),
                                             *tf_ops.split_rows(feature_input))
    pred_reg = pred_reg.view(bs, n, pred_reg_base_num, pred_reg_channel_num + ANGLE_CLS_NUM * 2)
    return (pred_cls, pred_reg[..., :pred_reg_channel_num],
            pred_reg[..., pred_reg_channel_num:pred_reg_channel_num + ANGLE_CLS_NUM],
            pred_reg[..., pred_reg_channel_num + ANGLE_CLS_NUM:])


def decode_class2angle(pred_cls, pred_res_norm, bin_size, bin_interval, bin_offset=0.0):
    """anchor_decoder.py:6-14: angle = (bin + residual[bin] + offset) * interval."""
    res = torch.gather(pred_res_norm, -1, pred_cls.unsqueeze(-1)).squeeze(-1)
    return (pred_cls.to(torch.float32) + res + bin_offset) * bin_interval


def decode_dist_anchor_free(center_xyz, det_forced_6_distance, det_angle_cls, det_angle_res, is_training=False):
    """anchor_decoder.py:86-112 -> boxes (bs, n, 7) = (x, y, z, l, h, w, ry)."""
    bins = torch.argmax(det_angle_cls, dim=-1)
    angle = decode_class2angle(bins, det_angle_res, ANGLE_CLS_NUM, 2 * math.pi / ANGLE_CLS_NUM).unsqueeze(-1)
    translate, half = det_forced_6_distance[..., :3], det_forced_6_distance[..., 3:6]
    ctr = center_xyz + translate
    pad = torch.zeros_like(half)
    pad[..., 1] = half[..., 1]                                   # move the centre down by the half height (:103-106)
    ctr = ctr + pad
    lhw = torch.clamp_min(half * 2.0, 0.1)
    return torch.cat([ctr, lhw, angle], dim=-1)


def postprocess(pred_anchors_3d, pred_score, max_output=MAX_OUTPUT_NUM, nms_threshold=NMS_THRESH):
    """PostProcessor.forward: pred_anchors_3d (bs, n, 1, 7), pred_score (bs, n, C) -> fixed-size block
    (bs, C * max_output, 9) + count (bs,).  One class: tf_ops.bev_nms; C > 1: the per-class NMS over the shared boxes
    (postprocessor.py:49-120), class-major rows tagged with the 0-based class in column 8."""
    boxes = pred_anchors_3d[:, :, 0, :].contiguous()
    c = pred_score.shape[-1]
    if c == 1:
        return tf_ops.bev_nms(boxes, pred_score[:, :, 0].contiguous(), nms_threshold, max_output, cls_id=0)
    return tf_ops.bev_nms(boxes, pred_score.contiguous(), nms_threshold, max_output, cls_num=c)


class DetectionHead:
    """HeadBuilder (head_builder.py) + test_forward + PostProcessor for a 'conv1d' / 'Det' head spec.  stage: the
    MODEL.FIRST_STAGE constants (config.STAGE_3DSSD, the default, or config.STAGE_POINTRCNN_RPN): REGRESSION selects the
    decode ('Dist-Anchor-free': tf_ops.decode_dist_anchor_free, 'Bin-Anchor': tf_ops.decode_bin_anchor on one anchor of
    ANCHOR_SIZE per point), MAX_OUTPUT_NUM and NMS_THRESH the post-processing.
    A 'Dist-Anchor-free' head has as many sigmoid classes C as its pred_cls/weights has columns (1..8); cls_num, when
    given, must agree.  C > 1 decodes C scores per point and runs the per-class NMS: the block is
    [bs, C * MAX_OUTPUT_NUM, 9] (max_output), class-major, column 8 the 0-based class."""

    def __init__(self, head_cfg=None, params=None, device="cuda", cls_num=None, stage=None):
        self.cfg = HEAD_3DSSD if head_cfg is None else head_cfg
        self.xyz_index, self.feature_index, self.op_type, self.mlp_list, self.bn, self.layer_type, self.scope = self.cfg
        if self.op_type != 'conv1d' or self.layer_type != 'Det':
            raise NotImplementedError("only 'conv1d' / 'Det' heads are built")
        self.stage = _cfg.STAGE_3DSSD if stage is None else stage
        self.reg_channels = reg_channels(self.stage)
        self.params = prepare(params, device)
        raw = self.params.raw
        key = _scope(self.scope, "pred_cls") + "/weights"
        width = None if raw is None or key not in raw else int(raw[key].shape[-1])
        if self.stage["REGRESSION"] == "Dist-Anchor-free" and width is not None:
            if cls_num is not None and int(cls_num) != width:
                raise ValueError("DetectionHead: cls_num=%d but %s has %d columns" % (cls_num, key, width))
            if not 1 <= width <= tf_ops.MAX_CLASSES:
                raise ValueError("DetectionHead: %s has %d columns; 1..%d classes are built" % (key, width, tf_ops.MAX_CLASSES))
            cls_num = width
        self.cls_num = 1 if cls_num is None else int(cls_num)
        self.multi = self.stage["REGRESSION"] == "Dist-Anchor-free" and self.cls_num > 1
        self.max_output = self.stage["MAX_OUTPUT_NUM"] * (self.cls_num if self.multi else 1)   # rows of the block

    def forward(self, xyz_list, feature_list, return_raw=False, out=None, split=None):
        """out=(block, count): preallocated outputs of the NMS (the send buffer of the multi-GPU gather).  split: the
        features' split operand (hi, lo) when the layer that produced them already wrote it."""
        xs = [xyz_list[i] for i in self.xyz_index]                                 # head_builder.py:82-85
        fs = [feature_list[i] for i in self.feature_index]
        xyz = xs[0] if len(xs) == 1 else torch.cat(xs, dim=1)
        feat = (fs[0] if len(fs) == 1 else torch.cat(fs, dim=1)).contiguous()
        y, (cls, reg) = head_convs(self.params, self.scope, self.bn, self.mlp_list,
                                   *(tf_ops.split_rows(feat) if split is None else split), want_f32=True)
        y = feat if y is None else y
        st = self.stage
        # decode + sigmoid (anchor_decoder.py:86-164, single_stage_detector.py:210-211): one kernel
        if st["REGRESSION"] == "Bin-Anchor":
            boxes, score = tf_ops.decode_bin_anchor(xyz, reg, cls, st["ANCHOR_SIZE"], st["HALF_BIN_SEARCH_RANGE"],
                                                    st["BIN_CLASS_NUM"], ANGLE_CLS_NUM)
        elif self.multi:
            boxes, score = tf_ops.decode_dist_anchor_free(xyz, reg, cls, ANGLE_CLS_NUM, cls_num=self.cls_num)
        else:
            boxes, score = tf_ops.decode_dist_anchor_free(xyz, reg, cls, ANGLE_CLS_NUM)
        if self.multi:                                                             # postprocessor.py:49-120, every class
            block, cnt = tf_ops.bev_nms(boxes, score, st["NMS_THRESH"], st["MAX_OUTPUT_NUM"], out=out, cls_num=self.cls_num)
        else:
            block, cnt = tf_ops.bev_nms(boxes, score, st["NMS_THRESH"], st["MAX_OUTPUT_NUM"], cls_id=0, out=out)   # postprocessor.py:52-120
        if return_raw:
            bs, n, _ = reg.shape
            r4 = reg.view(bs, n, 1, self.reg_channels + 2 * ANGLE_CLS_NUM)
            k = self.reg_channels
            return block, cnt, {"boxes": boxes.unsqueeze(2), "score": score if self.multi else score.unsqueeze(-1), "cls": cls, "reg": reg,
                                "offset": r4[..., :k], "angle_cls": r4[..., k:k + ANGLE_CLS_NUM],
                                "angle_res": r4[..., k + ANGLE_CLS_NUM:], "feat": y}
        return block, cnt

    __call__ = forward
