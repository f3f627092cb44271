"""Time PointRCNN's first stage (the RPN of tiny_pointrcnn_stage1.yaml) at B = 8 on synthetic KITTI scenes
(3dssd_b200/synth.py): the captured RPN step, CUDA-event times of its SA layers, FP layers, head + decode and NMS, the
fused FP route against the eager route it replaced (three_nn, eager weights, three_interpolate, concat, fp32 convs) on the
same inputs with the outputs compared, and the BEV NMS at n = 256 (3DSSD) and n = 16384 (the RPN).  Prints the card name
and its power limit, then one JSON line.

    python tools/time_pointrcnn.py [--reps 20] [--warmup 3]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("3dssd_b200")
C, L, T, P = pkg.config, pkg.layers_util, pkg.tf_ops, pkg.params
synth = importlib.import_module("3dssd_b200.synth")
B = 8


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


def eager_fp(pp, xyz1, xyz2, points1, points2, mlp, scope):
    """The inference FP route before the fused operand kernel: three_nn, the weights by torch ops, three_interpolate,
    torch.cat, then every conv on the fp32 CUDA-core GEMM (tf_ops.linear_bn_relu)."""
    dist, idx = T.three_nn(xyz1, xyz2)
    inv = 1.0 / torch.clamp_min(dist, 1e-10)
    x = T.three_interpolate(points2, idx, (inv / inv.sum(dim=2, keepdim=True)).contiguous())
    x = torch.cat([x, points1], dim=2).contiguous()
    for i in range(len(mlp)):
        f = pp.conv("%s/conv_%d" % (scope, i), True)
        x = T.linear_bn_relu(x, f.w, f.scale, f.shift, relu=True, cin=f.cin)
    return x


def nms_inputs(n, dev, seed):
    rng = np.random.default_rng(seed)
    bx = np.zeros((B, n, 7), np.float32)
    bx[..., 0] = rng.uniform(-40, 40, (B, n))
    bx[..., 1] = rng.uniform(-2, 2, (B, n))
    bx[..., 2] = rng.uniform(0, 70, (B, n))
    bx[..., 3] = rng.uniform(3.2, 4.6, (B, n))
    bx[..., 4] = rng.uniform(1.4, 1.8, (B, n))
    bx[..., 5] = rng.uniform(1.4, 1.9, (B, n))
    bx[..., 6] = rng.uniform(-np.pi, np.pi, (B, n))
    return torch.from_numpy(bx).to(dev), torch.from_numpy(rng.uniform(0, 1, (B, n)).astype(np.float32)).to(dev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seed", type=int, default=21)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_pointrcnn.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    card = torch.cuda.get_device_name(dev)
    try:
        power = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                        text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        power = "unknown"
    print("card: %s, power limit: %s" % (card, power))

    arch, st = C.ARCH_POINTRCNN_RPN, C.STAGE_POINTRCNN_RPN
    params = P.init_params(arch, 1, seed=0, aggregation=False)
    ch = C.layer_channels(arch, 1, aggregation=False)
    hp = P.init_head_params(ch[-1], mlp=(), reg_channels=4 * st["BIN_CLASS_NUM"] + 4 + 24, seed=1, scope="rpn_head")
    head = pkg.head.DetectionHead(C.HEAD_POINTRCNN_RPN, hp, device=dev, stage=st)
    net = pkg.SABackbone(arch, params, in_channels=1, device=dev, head=head, aggregation=False)
    pts = torch.from_numpy(synth.kitti_like(B, 16384, seed=a.seed)).to(dev)
    res = {"card": card, "power_limit": power, "batch": B, "points": 16384}

    replay = net.capture(pts)
    res["rpn_step_ms"] = timed(lambda: replay(), a.reps, a.warmup)

    # stages, eager: the SA layers, the FP layers, head + decode (+ NMS), the NMS alone
    sa = pkg.SABackbone(arch[:4], params, in_channels=1, device=dev, aggregation=False)
    xyz_l, feat_l, _ = sa.forward(pts)
    res["sa_ms"] = timed(lambda: sa.forward(pts), a.reps, a.warmup)
    fp_specs = arch[4:]

    def fp_all(route):
        xl, fl = list(xyz_l), list(feat_l)
        for spec in fp_specs:
            xi, fi, mlps, scope = spec[0], spec[1], spec[4], spec[12]
            if route == "fused":
                y = L.pointnet_fp_module(xl[xi[0]], xl[xi[1]], fl[fi[0]], fl[fi[1]], mlps, False, None, scope, True, params=net.params)
            else:
                y = eager_fp(net.params, xl[xi[0]], xl[xi[1]], fl[fi[0]], fl[fi[1]], mlps, scope)
            xl.append(xl[xi[0]]); fl.append(y)
        return xl, fl
    res["fp_ms"] = timed(lambda: fp_all("fused"), a.reps, a.warmup)
    res["fp_eager_ms"] = timed(lambda: fp_all("eager"), a.reps, a.warmup)
    xl, fl = fp_all("fused")
    _, fe = fp_all("eager")
    torch.cuda.synchronize()
    res["fp_fused_vs_eager_max_rel"] = [float((f - e).abs().max() / e.abs().max().clamp_min(1e-30))
                                        for f, e in zip(fl[5:], fe[5:])]
    res["head_decode_nms_ms"] = timed(lambda: head.forward(xl, fl), a.reps, a.warmup)
    _, _, raw = head.forward(xl, fl, return_raw=True)
    boxes, score = raw["boxes"][:, :, 0].contiguous(), raw["score"][..., 0].contiguous()
    res["nms_rpn_ms"] = timed(lambda: T.bev_nms(boxes, score, st["NMS_THRESH"], st["MAX_OUTPUT_NUM"]), a.reps, a.warmup)
    res["head_decode_ms"] = res["head_decode_nms_ms"] - res["nms_rpn_ms"]

    # the NMS at 3DSSD's n = 256 (IoU 0.1) and the RPN's n = 16384 (IoU 0.85)
    for n, thr in ((256, 0.1), (16384, 0.85)):
        bx, sc = nms_inputs(n, dev, n)
        blk = torch.empty((B, 100, 9), device=dev)
        cnt = torch.empty((B,), dtype=torch.int32, device=dev)
        res["nms_n%d_ms" % n] = timed(lambda: T.bev_nms(bx, sc, thr, 100, out=(blk, cnt)), 10 * a.reps, a.warmup)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
