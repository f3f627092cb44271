"""numpy restatement of the detection head, decoding and post-processing of the single-stage 3DSSD detector.

TEST INFRASTRUCTURE ONLY (see ssd3d_oracle.c).  Follows /root/reference/lib/modeling/head_builder.py:81-114,
lib/utils/head_util.py:26-59 (box_regression_head), lib/utils/anchor_decoder.py:6-14, :86-112
(decode_class2angle, decode_dist_anchor_free), lib/modeling/single_stage_detector.py:193-226 (sigmoid scores),
lib/utils/box_3d_utils.py:25-58 (box_3d_to_anchor), lib/utils/anchors_util.py:11-48 (project_to_bev) and
lib/builder/postprocessor.py:52-120 with TensorFlow's greedy non_max_suppression (descending score, a candidate is
dropped when IoU with a kept box is > threshold; ties broken by lower index, which TF 1.4 leaves unspecified).
"""
import math

import numpy as np

from . import ops

ANGLE_CLS_NUM = 12


def _conv(params, scope, x, bn, relu):
    bnp = tuple(params[scope + "/bn/" + k] for k in ("gamma", "beta", "moving_mean", "moving_variance")) if bn else None
    return ops.linear_bn_relu(x, params[scope + "/weights"], params.get(scope + "/biases"), bnp, relu)


def head_forward(xyz, feat, params, mlp=(128,), bn=True, scope=""):
    pre = "" if scope == "" else scope + "/"
    y = feat
    for i in range(len(mlp)):
        y = _conv(params, "%sconv1d_%d" % (pre, i), y, bn, True)
    cls = _conv(params, pre + "pred_cls", _conv(params, pre + "pred_cls_base", y, bn, True), False, False)
    reg = _conv(params, pre + "pred_reg", _conv(params, pre + "pred_reg_base", y, bn, True), False, False)
    off, acls, ares = reg[..., :6], reg[..., 6:6 + ANGLE_CLS_NUM], reg[..., 6 + ANGLE_CLS_NUM:]
    bins = np.argmax(acls, axis=-1)
    res = np.take_along_axis(ares, bins[..., None], axis=-1)[..., 0]
    angle = ((bins.astype(np.float32) + res) * np.float32(2 * np.pi / ANGLE_CLS_NUM)).astype(np.float32)
    ctr = xyz + off[..., :3]
    ctr[..., 1] += off[..., 4]
    lhw = np.maximum(off[..., 3:6] * np.float32(2.0), np.float32(0.1))
    boxes = np.concatenate([ctr, lhw, angle[..., None]], axis=-1).astype(np.float32)
    score = (1.0 / (1.0 + np.exp(-cls.astype(np.float64)))).astype(np.float32)
    return boxes, score[..., 0], {"feat": y, "cls": cls, "reg": reg}


def bev_rects(boxes):
    """BEV rectangles (x1, z1, x2, z2) of boxes [..., 7] in float32, by the recipe of DESIGN.md §3.5 that the kernel
    (csrc/nms.cu) and the C twin share: |cos ry| and |sin ry| in double, rounded once to float32 (libm through `math`,
    as the C twin calls it: numpy's own float32 and SIMD float64 cos are other functions); every product and sum
    rounded to float32 on its own, no fused multiply-add."""
    bx = np.asarray(boxes, np.float32)
    ry = bx[..., 6].ravel().tolist()
    c = np.abs(np.array([math.cos(a) for a in ry], np.float64).astype(np.float32)).reshape(bx.shape[:-1])
    s = np.abs(np.array([math.sin(a) for a in ry], np.float64).astype(np.float32)).reshape(bx.shape[:-1])
    l, w = bx[..., 3], bx[..., 5]
    dimx = (l * c) + (w * s)                              # float32 arrays: each operation rounded on its own
    dimz = (w * c) + (l * s)
    half = np.float32(0.5)
    return np.stack([bx[..., 0] - dimx * half, bx[..., 2] - dimz * half,
                     bx[..., 0] + dimx * half, bx[..., 2] + dimz * half], -1)


def bev_nms(boxes, scores, iou_threshold=0.1, max_output=100, cls_id=0):
    """Greedy BEV NMS per scene, the oracle of csrc/nms.cu and oracle/ssd3d_oracle.c:oracle_bev_nms (DESIGN.md §3.5):
    descending score, ties (+0 and -0 among them) to the lower index; a candidate is dropped when its float32 IoU with
    a kept box is > float32(iou_threshold); a box of area <= 0 neither suppresses nor is suppressed.  NaN scores are
    outside the contract."""
    b, n, _ = boxes.shape
    thr = np.float32(iou_threshold)
    zero = np.float32(0)
    block = np.zeros((b, max_output, 9), np.float32)
    cnt = np.zeros((b,), np.int32)
    for s in range(b):
        bx, sc = boxes[s], scores[s]
        x1, z1, x2, z2 = bev_rects(bx).T
        area = (x2 - x1) * (z2 - z1)
        order = sorted(range(n), key=lambda i: (-float(sc[i]), i))       # -0.0 == 0.0: the lower index first
        kept = []
        for i in order:
            ok = True
            for j in kept:
                if area[i] <= 0 or area[j] <= 0:
                    continue
                iw = min(x2[i], x2[j]) - max(x1[i], x1[j])
                ih = min(z2[i], z2[j]) - max(z1[i], z1[j])
                inter = max(iw, zero) * max(ih, zero)
                if inter / ((area[i] + area[j]) - inter) > thr:
                    ok = False
                    break
            if ok:
                kept.append(i)
                if len(kept) == max_output:
                    break
        for k, i in enumerate(kept):
            block[s, k, :7] = bx[i]
            block[s, k, 7] = sc[i]
            block[s, k, 8] = cls_id
        cnt[s] = len(kept)
    return block, cnt
