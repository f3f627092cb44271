"""Detection head, box decoding and post-processing of the single-stage 3DSSD detector (SURVEY.md section 8f, rows f1/f2).

Mirrors, for inference with the shipped 3DSSD configuration (anchor-free 'Dist-Anchor-free' regression, sigmoid
classification, one class, `HEAD: [[[6], [6], 'conv1d', [128,], True, 'Det', '']]`, configs/kitti/3dssd/3dssd.yaml:68):
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

from . import tf_ops
from .params import TrainableParams, prepare

ANGLE_CLS_NUM = 12          # MODEL.ANGLE_CLS_NUM (3dssd.yaml:38)
REG_CHANNELS = 6            # 'Dist-Anchor-free': distances to the 6 faces (head_builder.py:49-55)
MAX_OUTPUT_NUM = 100        # MODEL.FIRST_STAGE.MAX_OUTPUT_NUM (3dssd.yaml:70)
NMS_THRESH = 0.1            # MODEL.FIRST_STAGE.NMS_THRESH (3dssd.yaml:71)
HEAD_3DSSD = [[6], [6], 'conv1d', [128], True, 'Det', '']


def _scope(scope, name):
    return name if scope == '' else scope + "/" + name


def _conv_chain(pp, hi, lo, scopes_bn_relu):
    y = None
    for i, (sc, bn, relu) in enumerate(scopes_bn_relu):
        last = i == len(scopes_bn_relu) - 1
        y, sp = tf_ops.linear_tc(hi, lo, pp.conv(sc, bn), relu=relu, want_f32=last, want_split=not last)
        if not last:
            hi, lo = sp
    return y


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
        pp = prepare(params, feature_input.device)
        hi, lo = tf_ops.split_rows(feature_input)
        pred_cls = _conv_chain(pp, hi, lo, [(_scope(scope, "pred_cls_base"), bn, True), (_scope(scope, "pred_cls"), False, False)])
        pred_reg = _conv_chain(pp, hi, lo, [(_scope(scope, "pred_reg_base"), bn, True), (_scope(scope, "pred_reg"), False, False)])
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
    """PostProcessor.forward for one class: pred_anchors_3d (bs, n, 1, 7), pred_score (bs, n, 1) ->
    fixed-size block (bs, max_output, 9) + count (bs,)."""
    boxes = pred_anchors_3d[:, :, 0, :].contiguous()
    return tf_ops.bev_nms(boxes, pred_score[:, :, 0].contiguous(), nms_threshold, max_output, cls_id=0)


class DetectionHead:
    """HeadBuilder (head_builder.py) + test_forward + PostProcessor for the 3DSSD head spec."""

    def __init__(self, head_cfg=None, params=None, device="cuda", cls_num=1):
        self.cfg = HEAD_3DSSD if head_cfg is None else head_cfg
        self.xyz_index, self.feature_index, self.op_type, self.mlp_list, self.bn, self.layer_type, self.scope = self.cfg
        if self.op_type != 'conv1d' or self.layer_type != 'Det':
            raise NotImplementedError("only the 'conv1d' / 'Det' head of the 3DSSD configuration is built")
        self.cls_num = cls_num
        self.params = prepare(params, device)

    def forward(self, xyz_list, feature_list, return_raw=False, out=None):
        """out=(block, count): preallocated outputs of the NMS (the send buffer of the multi-GPU gather)."""
        xs = [xyz_list[i] for i in self.xyz_index]                                 # head_builder.py:82-85
        fs = [feature_list[i] for i in self.feature_index]
        xyz = xs[0] if len(xs) == 1 else torch.cat(xs, dim=1)
        feat = (fs[0] if len(fs) == 1 else torch.cat(fs, dim=1)).contiguous()
        hi, lo = tf_ops.split_rows(feat)
        y = feat
        for i, ch in enumerate(self.mlp_list):                                    # :93-95
            y, (hi, lo) = tf_ops.linear_tc(hi, lo, self.params.conv(_scope(self.scope, "conv1d_%d" % i), self.bn),
                                           want_f32=True, want_split=True)
        pp, sc = self.params, self.scope
        cls = _conv_chain(pp, hi, lo, [(_scope(sc, "pred_cls_base"), self.bn, True), (_scope(sc, "pred_cls"), False, False)])
        reg = _conv_chain(pp, hi, lo, [(_scope(sc, "pred_reg_base"), self.bn, True), (_scope(sc, "pred_reg"), False, False)])
        # decode_dist_anchor_free + sigmoid (anchor_decoder.py:86-112, single_stage_detector.py:210-211): one kernel
        boxes, score = tf_ops.decode_dist_anchor_free(xyz, reg, cls, ANGLE_CLS_NUM)
        block, cnt = tf_ops.bev_nms(boxes, score, NMS_THRESH, MAX_OUTPUT_NUM, cls_id=0, out=out)   # postprocessor.py:52-120
        if return_raw:
            bs, n, _ = reg.shape
            r4 = reg.view(bs, n, 1, REG_CHANNELS + 2 * ANGLE_CLS_NUM)
            return block, cnt, {"boxes": boxes.unsqueeze(2), "score": score.unsqueeze(-1), "cls": cls,
                                "offset": r4[..., :REG_CHANNELS], "angle_cls": r4[..., REG_CHANNELS:REG_CHANNELS + ANGLE_CLS_NUM],
                                "angle_res": r4[..., REG_CHANNELS + ANGLE_CLS_NUM:], "feat": y}
        return block, cnt

    __call__ = forward
