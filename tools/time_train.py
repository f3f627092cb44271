"""Forward + backward of the 3DSSD backbone (ARCH_3DSSD, vote layer, CG layer) plus the detection head in training mode
(params.TrainableParams, is_training=True) on one GPU, timed with CUDA events after warm-up; then every launch of the
backward kernels (linear_wgrad, bn_train_grad, rowgroup_max_grad, group_concat_grad) of one step timed with its own
event pair, and the issued / algorithmic MMA rate of linear_wgrad against the 989 TFLOP/s BF16 data-sheet figure of the
H100 SXM.  The loss is the mean of the squared head outputs and vote offsets, a stand-in; --loss det trains against the
3DSSD detection loss (loss.assign_targets + loss.detection_loss) on synth.kitti_like_with_boxes scenes and also times
each launch of det_assign, det_loss and det_loss_grad.  Prints the card name and its power limit, then one JSON line.

    python tools/time_train.py [--batch 8] [--points 16384] [--steps 5] [--warmup 2] [--loss squares|det]
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
T = pkg.tf_ops
PEAK_BF16 = 989e12            # H100 SXM data sheet, dense BF16


def train_forward(arch, tp, xyz, feat):
    """backbone.train_forward: returns (outputs of the head, raw vote offsets)."""
    o = pkg.backbone.train_forward(arch, tp, xyz, feat)
    return o.head, o.vote_offsets


def trainable(arch, device, seed=0):
    d = pkg.params.init_params(arch, 1, seed=seed, random_bias=True)
    d.update(pkg.params.init_head_params(pkg.config.layer_channels(arch, 1)[-1], seed=seed + 1))
    return pkg.params.TrainableParams(d, device)


def step(arch, tp, xyz, feat):
    outs, offs = train_forward(arch, tp, xyz, feat)
    loss = sum((o.float() ** 2).mean() for o in outs) + sum((o ** 2).mean() for o in offs)
    loss.backward()
    return loss


def det_step(arch, tp, xyz, feat, gt_boxes, gt_labels):
    """One step with the real 3DSSD objective: train_forward -> assign_targets -> detection_loss -> backward."""
    o = pkg.backbone.train_forward(arch, tp, xyz, feat)
    tg = pkg.loss.assign_targets(o.base_xyz, o.vote_base, gt_boxes, gt_labels)
    losses = pkg.loss.detection_loss(o.base_xyz, *o.head, o.vote_offsets[-1], tg)
    losses["total"].backward()
    return losses


class _Timed:
    """Wraps the tf_ops backward entry points: each launch gets its own CUDA event pair."""

    def __init__(self, names):
        self.names, self.rec, self.orig = names, [], {}

    def __enter__(self):
        for n in self.names:
            f = getattr(T, n)
            self.orig[n] = f

            def wrap(*a, _f=f, _n=n, **k):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                r = _f(*a, **k)
                e.record()
                shape = (a[0].numel() // a[0].shape[-1], a[0].shape[-1], a[1].shape[-1]) if _n == "linear_wgrad" else \
                    (tuple(a[0].shape) + ((a[2].shape[1],) if _n == "det_assign" else ()))
                self.rec.append((_n, shape, s, e))
                return r
            setattr(T, n, wrap)
        return self

    def __exit__(self, *a):
        for n, f in self.orig.items():
            setattr(T, n, f)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--points", type=int, default=16384)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--loss", choices=("squares", "det"), default="squares",
                    help="squares: mean of squared head outputs and vote offsets (a stand-in); det: the 3DSSD detection "
                         "loss on synth.kitti_like_with_boxes scenes, with the target and loss launches timed as well")
    ap.add_argument("--max-boxes", type=int, default=40, help="GT rows per scene of --loss det")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_train.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    card = torch.cuda.get_device_name(dev)
    try:
        power = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                                        text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        power = "unknown"
    print("card: %s, power limit / max SM clock: %s" % (card, power))
    arch = pkg.config.ARCH_3DSSD
    synth = importlib.import_module("3dssd_b200.synth")
    timed = ["linear_wgrad", "bn_train_grad", "rowgroup_max_grad", "group_concat_grad"]
    if a.loss == "det":
        p, boxes, labels = synth.kitti_like_with_boxes(a.batch, a.points, a.max_boxes, seed=1)
        pts = torch.from_numpy(p).to(dev)
        gb, gl = torch.from_numpy(boxes).to(dev), torch.from_numpy(labels).to(dev)
        run = lambda: det_step(arch, tp, xyz, feat, gb, gl)
        timed += ["det_assign", "det_loss", "det_loss_grad"]
    else:
        pts = torch.from_numpy(synth.kitti_like(a.batch, a.points, seed=1)).to(dev)
        run = lambda: step(arch, tp, xyz, feat)
    xyz, feat = T.split_points(pts)
    tp = trainable(arch, dev)
    for _ in range(a.warmup):
        run()
        tp_zero(tp)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(a.steps):
        run()
        tp_zero(tp)
    e.record()
    torch.cuda.synchronize()
    step_ms = s.elapsed_time(e) / a.steps
    with _Timed(timed) as tm:
        run()
        tp_zero(tp)
    torch.cuda.synchronize()
    per = {}
    wg_ms = wg_issued = wg_alg = 0.0
    for n, shape, s1, e1 in tm.rec:
        ms = s1.elapsed_time(e1)
        per.setdefault(n, []).append((shape, round(ms, 4)))
        if n == "linear_wgrad":
            rows, cin, cout = shape
            bn = 16 if cout <= 16 else (32 if cout <= 32 else 64)
            wg_ms += ms
            wg_issued += 3 * 2.0 * ((rows + 63) // 64 * 64) * ((cin + 63) // 64 * 64) * ((cout + bn - 1) // bn * bn)
            wg_alg += 2.0 * rows * cin * cout
    for n, lst in per.items():
        print("%-18s %3d launches %8.3f ms" % (n, len(lst), sum(ms for _, ms in lst)))
        for shape, ms in lst:
            print("    %-28s %8.4f ms" % (shape, ms))
    res = {"card": card, "power_limit_max_sm_clock": power, "batch": a.batch, "points": a.points, "loss": a.loss,
           "train_step_ms": round(step_ms, 3),
           "backward_kernels_ms": {n: round(sum(ms for _, ms in lst), 3) for n, lst in per.items() if not n.startswith("det_")},
           "linear_wgrad_issued_bf16_tflops": round(wg_issued / (wg_ms * 1e-3) / 1e12, 2),
           "linear_wgrad_issued_share_of_989": round(wg_issued / (wg_ms * 1e-3) / PEAK_BF16, 4),
           "linear_wgrad_algorithmic_tflops": round(wg_alg / (wg_ms * 1e-3) / 1e12, 2),
           "linear_wgrad_algorithmic_share_of_989": round(wg_alg / (wg_ms * 1e-3) / PEAK_BF16, 4)}
    if a.loss == "det":
        res["det_kernels_ms"] = {n: round(sum(ms for _, ms in lst), 4) for n, lst in per.items() if n.startswith("det_")}
    print(json.dumps(res))


def tp_zero(tp):
    for t in tp.parameters():
        t.grad = None


if __name__ == "__main__":
    main()
