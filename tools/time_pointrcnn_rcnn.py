"""Time PointRCNN's two-stage detector (tiny_pointrcnn_stage2_test.yaml, 3dssd_b200.PointRCNN) at B = 8 on the synthetic
KITTI batch of tools/time_pointrcnn.py: the captured two-stage step, and CUDA-event times of its parts -- the RPN (SA +
FP layers, head, decode, NMS at 0.8), the region pool, the stage-2 SA layers on the B * 100 pooled scenes, and the RCNN
head + decode + counted NMS.  The region pool is also set against the reference's own kernels on the same proposals
(oracle/_ref/libref_ops.so, when it is built): queryBoxes3dPointsLauncher plus the three groupPointLauncher gathers of
points_pooler.py:123-133 (xyz, features, mask), which leave the canonical transform and the info conv still to do.
Prints the card name and its power limit, then one JSON line.

    python tools/time_pointrcnn_rcnn.py [--reps 20] [--warmup 3]
"""
import argparse
import ctypes
import importlib
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("3dssd_b200")
C, T = pkg.config, pkg.tf_ops
synth = importlib.import_module("3dssd_b200.synth")
B = 8
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libref_ops.so")


def timed(fn, reps, warmup):
    """ms per call: CUDA events around `reps` back-to-back calls after `warmup` calls."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seed", type=int, default=21)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_pointrcnn_rcnn.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    card = torch.cuda.get_device_name(dev)
    try:
        power = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                        text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        power = "unknown"
    print("card: %s, power limit: %s" % (card, power))

    net = pkg.PointRCNN(device=dev, seed=0)
    pts = torch.from_numpy(synth.kitti_like(B, 16384, seed=a.seed)).to(dev)
    res = {"card": card, "power_limit": power, "batch": B, "points": 16384}
    replay = net.capture(pts)
    res["two_stage_step_ms"] = timed(lambda: replay(), a.reps, a.warmup)

    block, count, d = net.forward(pts, return_debug=True)
    res["proposals_per_scene"] = d["proposal_count"].cpu().tolist()
    res["rpn_ms"] = timed(lambda: net.rpn_head.forward(*net.rpn.forward(pts)[:2], return_raw=True), a.reps, a.warmup)
    pool = net.pooler
    conv0 = net.params.conv(pool[8] + "/conv0", pool[7])
    score = d["rpn_raw"]["score"][..., 0]
    base_xyz, base_feat, props, pcount = d["rpn_xyz"][-1], d["rpn_feat"][-1], d["proposals"], d["proposal_count"]
    pool_fn = lambda: T.region_pool(base_xyz, base_feat, score, props, pcount, conv0, nsample=pool[3], context=pool[4],
                                    mask_thresh=net.mask_thresh)
    res["region_pool_ms"] = timed(pool_fn, a.reps, a.warmup)
    lists = ([d["ctr"], d["pool_xyz"]], [None, d["pool_feat"]])
    res["rcnn_sa_ms"] = timed(lambda: net.rcnn.forward_lists(*lists), a.reps, a.warmup)
    st = net.stage

    def head_decode_nms():
        feat = d["rcnn_feat"][4].reshape(*d["ctr"].shape[:2], -1).contiguous()
        _, (cls, reg) = pkg.head.head_convs(net.params, net.head_scope, net.head_bn, net.head_mlp, *T.split_rows(feat))
        boxes, scores = T.decode_bin_anchor_rows(props, reg, cls, d["pool_cnt"], st["HALF_BIN_SEARCH_RANGE"], st["BIN_CLASS_NUM"])
        return T.bev_nms_counted(boxes, scores, pcount, st["NMS_THRESH"], st["MAX_OUTPUT_NUM"])
    res["head_decode_nms_ms"] = timed(head_decode_nms, a.reps, a.warmup)

    if os.path.exists(REF_LIB):
        lib = ctypes.CDLL(REF_LIB)
        p = lambda t: ctypes.c_void_p(t.data_ptr())
        exp = props[..., :7].clone()
        exp[..., 3:6] += pool[4]
        exp = exp.contiguous()
        n, m, ns = base_xyz.shape[1], props.shape[1], pool[3]
        idx = torch.zeros((B, m, ns), dtype=torch.int32, device=dev)
        cnt = torch.zeros((B, m), dtype=torch.int32, device=dev)
        mask = (score >= net.mask_thresh).float().unsqueeze(-1).contiguous()
        gx = torch.empty((B, m, ns, 3), device=dev)
        gf = torch.empty((B, m, ns, base_feat.shape[2]), device=dev)
        gm = torch.empty((B, m, ns, 1), device=dev)

        def ref_pool():      # the reference's launchers run on the legacy default stream, which torch's stream is
            lib._Z26queryBoxes3dPointsLauncheriiiiPKfS0_PiS1_(B, n, m, ns, p(base_xyz), p(exp), p(idx), p(cnt))
            for src, out, c in ((base_xyz, gx, 3), (base_feat, gf, base_feat.shape[2]), (mask, gm, 1)):
                lib._Z18groupPointLauncheriiiiiPKfPKiPf(B, n, c, m, ns, p(src), p(idx), p(out))
        res["ref_query_group_ms"] = timed(ref_pool, a.reps, a.warmup)
        ours_idx = pool_fn()[2]
        torch.cuda.synchronize()
        valid = torch.arange(m, device=dev)[None] < pcount[:, None].long()
        res["ref_pool_idx_equal"] = bool(torch.equal(torch.where(valid[..., None], idx, 0), ours_idx))
    else:
        res["ref_query_group_ms"] = "not measured (oracle/_ref/libref_ops.so is not built)"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
