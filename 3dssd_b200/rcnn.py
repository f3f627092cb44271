"""PointRCNN's two-stage detector at inference (configs/kitti/pointrcnn/tiny_pointrcnn_stage2_test.yaml), DESIGN.md
section 3.16.

Follows DoubleStageDetector.model_forward (/root/reference/lib/modeling/double_stage_detector.py:166-219) and its
test_forward (:298-337):
  1. the RPN (SABackbone over config.ARCH_POINTRCNN_RPN + the 'rpn_head' DetectionHead) with the test yaml's NMS at 0.8:
     at most 100 bottom-centred proposals per scene, block [B, 100, 9] + count [B];
  2. the region pool (tf_ops.region_pool, one kernel): expand, collect 512 points, canonical transform, info conv;
  3. the stage-2 SA layers (SABackbone over config.ARCH_POINTRCNN_RCNN, no aggregation) on B * 100 pooled scenes, their
     lists starting [proposal centres, pooled xyz] / [None, pooled features];
  4. the 'rcnn_head' convs on the tensor cores, the Bin-Anchor decode against the proposals with the softmax score
     times the pool mask (tf_ops.decode_bin_anchor_rows), and the BEV NMS over each scene's real proposals only
     (tf_ops.bev_nms_counted).
Nothing syncs the host, so the whole forward is captured in one CUDA graph (capture()).
"""
import torch

from . import config as _cfg
from . import tf_ops
from .backbone import SABackbone, capture_graph
from .head import ANGLE_CLS_NUM, DetectionHead, head_convs, reg_channels
from .params import init_head_params, init_params, init_rcnn_params, prepare


def cast_bottom_to_center(boxes):
    """model_util.py:243-253: y_centre = y_bottom - h / 2 (fp32, one rounding each)."""
    out = boxes[..., :7].clone()
    out[..., 1] = boxes[..., 1] - boxes[..., 4] / 2.0
    return out


def init_pointrcnn_params(seed=0):
    """Random weights of the whole two-stage detector under the reference's variable names."""
    st = _cfg.STAGE_POINTRCNN_RPN
    ch = _cfg.layer_channels(_cfg.ARCH_POINTRCNN_RPN, 1, aggregation=False)
    p = init_params(_cfg.ARCH_POINTRCNN_RPN, 1, seed=seed, aggregation=False)
    p.update(init_head_params(ch[-1], mlp=(), reg_channels=reg_channels(st) + 2 * ANGLE_CLS_NUM, seed=seed + 1, scope="rpn_head"))
    p.update(init_rcnn_params(ch[-1], seed=seed + 2))
    return p


class PointRCNN:
    """forward(points [B, N, 4]) -> (block [B, 100, 9], count [B]) of the two-stage detector; return_debug=True also
    returns a dict of every intermediate.  rpn_kw go to the RPN's SABackbone (e.g. fps_cluster, latency_mode)."""

    def __init__(self, params=None, device="cuda", seed=0, **rpn_kw):
        self.device = torch.device(device)
        if params is None:
            params = init_pointrcnn_params(seed)
        self.params = prepare(params, self.device).prepare_all()
        self.rpn_stage = _cfg.STAGE_POINTRCNN_RPN_TEST
        self.stage = _cfg.STAGE_POINTRCNN_RCNN
        self.pooler = _cfg.POINTS_POOLER_POINTRCNN
        self.mask_thresh = _cfg.POOLER_MASK_THRESHOLD
        self.rpn_head = DetectionHead(_cfg.HEAD_POINTRCNN_RPN, self.params, device=self.device, stage=self.rpn_stage)
        self.rpn = SABackbone(_cfg.ARCH_POINTRCNN_RPN, self.params, in_channels=1, device=self.device, head=self.rpn_head,
                              aggregation=False, **rpn_kw)
        self.rcnn = SABackbone(_cfg.ARCH_POINTRCNN_RCNN, self.params, device=self.device, aggregation=False)
        (self.head_xyz, self.head_feat, _, self.head_mlp, self.head_bn, _, self.head_scope) = _cfg.HEAD_POINTRCNN_RCNN
        self.reg_channels = reg_channels(self.stage) + 2 * ANGLE_CLS_NUM

    def forward(self, points, return_debug=False):
        rxyz, rfeat, rfps, rdbg = self.rpn.forward(points, return_debug=True)
        props, pcount, raw = self.rpn_head.forward(rxyz, rfeat, return_raw=True)
        base_xyz, base_feat = rxyz[-1], rfeat[-1]
        score = raw["score"][..., 0]
        pool = self.pooler
        pxyz, pfeat, pidx, pcnt = tf_ops.region_pool(base_xyz, base_feat, score, props, pcount,
                                                     self.params.conv(pool[8] + "/conv0", pool[7]), nsample=pool[3],
                                                     context=pool[4], mask_thresh=self.mask_thresh)
        ctr = cast_bottom_to_center(props)[..., :3].contiguous()
        xyz_l, feat_l, fps_l, sdbg = self.rcnn.forward_lists([ctr, pxyz], [None, pfeat], return_debug=True)
        # head_builder.py:81-113 on the [B * P, 512] features as [B, P, 512]: conv1d_0, then the pred_cls / pred_reg chains
        feat = feat_l[self.head_feat[0]].reshape(*xyz_l[self.head_xyz[0]].shape[:2], -1).contiguous()
        _, (cls, reg) = head_convs(self.params, self.head_scope, self.head_bn, self.head_mlp, *tf_ops.split_rows(feat))
        st = self.stage
        boxes, scores = tf_ops.decode_bin_anchor_rows(props, reg, cls, pcnt, st["HALF_BIN_SEARCH_RANGE"], st["BIN_CLASS_NUM"],
                                                      ANGLE_CLS_NUM)
        block, count = tf_ops.bev_nms_counted(boxes, scores, pcount, st["NMS_THRESH"], st["MAX_OUTPUT_NUM"], cls_id=0)
        if return_debug:
            return block, count, {"rpn_xyz": rxyz, "rpn_feat": rfeat, "rpn_fps": rfps, "rpn_dbg": rdbg, "rpn_raw": raw,
                                  "proposals": props, "proposal_count": pcount, "pool_xyz": pxyz, "pool_feat": pfeat,
                                  "pool_idx": pidx, "pool_cnt": pcnt, "ctr": ctr, "rcnn_xyz": xyz_l, "rcnn_feat": feat_l,
                                  "rcnn_fps": fps_l, "rcnn_dbg": sdbg, "cls": cls, "reg": reg, "boxes": boxes,
                                  "scores": scores}
        return block, count

    __call__ = forward

    def capture(self, example_points, warmup=2):
        """Record forward into one CUDA graph; returns replay(points=None) -> (block, count) on the static buffers."""
        return capture_graph(self.forward, example_points, warmup)
