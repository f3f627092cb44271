"""Times SyncBN (csrc/bn.cu ssd3d_bn_train_sync / ssd3d_bn_train_grad_sync, DESIGN.md section 3.18) and prints the card
name and power limit, then one JSON line:
  per_call        at every BatchNorm shape of one ARCH_3DSSD step at 8 x 16384 points (tests/golden/
                  train_backward_shapes.json): bn_train against bn_train_sync and bn_train_grad against bn_train_grad_sync
                  at world 1, alternating, CUDA events around every call (what a caller waits for, host enqueue included).
                  The sync call's extra time is the exchange launch: at world 1 its wait is on itself.
  step_ms         one training step (ARCH_3DSSD + head, detection loss, Adam: solver.Trainer) at world 1 with and without
                  sync_bn, alternating, profiler off.
  multi_gpu       the exchange between GPUs is not measured here: it needs >= 2 GPUs and torchrun (tools/train_dp.py
                  --gpus G --sync-bn against the same command without it).  With fewer GPUs the JSON says "not measured".

    python tools/time_sync_bn.py [--rounds 50] [--steps 10] [--batch 4] [--points 16384]
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
S = importlib.import_module("3dssd_b200.solver")
synth = importlib.import_module("3dssd_b200.synth")


def bn_shapes(batch=8):
    d = json.load(open(os.path.join(ROOT, "tests", "golden", "train_backward_shapes.json")))
    out = []
    for name, s in d["calls"]:
        t = (batch * int(np.prod(s[1:-2])), int(s[-2]))
        if name == "bn_train_grad" and t not in out:
            out.append(t)
    return out


def alternate(fns, rounds, warmup=3):
    """Median ms of each callable, run in turn `rounds` times after `warmup` rounds, CUDA events around every call."""
    for _ in range(warmup):
        for f in fns:
            f()
    torch.cuda.synchronize()
    ev = [[] for _ in fns]
    for _ in range(rounds):
        for i, f in enumerate(fns):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            f()
            e.record()
            ev[i].append((s, e))
    torch.cuda.synchronize()
    return [float(np.median([s.elapsed_time(e) for s, e in x])) for x in ev]


def per_call(dev, rounds):
    T, D = pkg.tf_ops, pkg.dist
    rows_out = []
    for rows, c in bn_shapes():
        area = D.bn_sync_area_bytes(1, c)
        sym = torch.zeros((2 * area,), dtype=torch.uint8, device=dev)
        peers = torch.tensor([sym.data_ptr()], dtype=torch.int64, device=dev)
        st = torch.zeros((2, 4), dtype=torch.int32, device=dev)
        fw, bw = (T.BnSyncSlot(peers, 1, 0, d * area, st[d]) for d in (0, 1))
        x = torch.randn((rows, c), device=dev)
        go = torch.randn((rows, c), device=dev)
        g, b = torch.rand(c, device=dev) + 0.5, torch.randn(c, device=dev)
        mm, mv = torch.zeros(c, device=dev), torch.ones(c, device=dev)
        r = T.bn_train(x, g, b)
        f_plain, f_sync = alternate([lambda: T.bn_train(x, g, b, mm, mv), lambda: T.bn_train_sync(x, g, b, fw, mm, mv)], rounds)
        b_plain, b_sync = alternate([lambda: T.bn_train_grad(x, go, *r[1:], g), lambda: T.bn_train_grad_sync(x, go, *r[1:], g, bw)],
                                    rounds)
        assert int(st[:, 2].sum().item()) == 0
        rows_out.append({"rows": rows, "c": c, "fwd_ms": round(f_plain, 4), "fwd_sync_ms": round(f_sync, 4),
                         "bwd_ms": round(b_plain, 4), "bwd_sync_ms": round(b_sync, 4)})
    return rows_out


def step_ms(dev, steps, batch, points):
    arch = pkg.config.ARCH_3DSSD
    p, bx, lb = synth.kitti_like_with_boxes(batch, points, 40, seed=1)
    pts, boxes, labels = (torch.from_numpy(a).to(dev) for a in (p, bx, lb))
    xyz, feat = pkg.tf_ops.split_points(pts)
    trainers = []
    for sync in (False, True):
        d = pkg.params.init_params(arch, 1, seed=0, random_bias=True)
        d.update(pkg.params.init_head_params(pkg.config.layer_channels(arch, 1)[-1], seed=1))
        trainers.append(S.Trainer(arch, pkg.params.TrainableParams(d, dev), S.Solver(), sync_bn=sync))
    plain, sync = alternate([lambda tr=tr: tr.step(xyz, feat, boxes, labels) for tr in trainers], steps, warmup=2)
    assert trainers[1].dp.timeouts() == 0
    return plain, sync


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=50)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--points", type=int, default=16384)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_sync_bn.py measures on a CUDA device; none is available")
    dev = torch.device("cuda", 0)
    card = torch.cuda.get_device_name(dev)
    try:
        power = subprocess.check_output(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                                        text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        power = "unknown"
    calls = per_call(dev, a.rounds)
    plain, sync = step_ms(dev, a.steps, a.batch, a.points)
    res = {"card": card, "power_limit_max_sm_clock": power, "world": 1, "per_call": calls,
           "per_step_sum_ms": {k: round(sum(c[k] for c in calls), 3) for k in ("fwd_ms", "fwd_sync_ms", "bwd_ms", "bwd_sync_ms")},
           "step_ms": {"batch": a.batch, "points": a.points, "plain": round(plain, 3), "sync_bn": round(sync, 3)},
           "multi_gpu": "not measured" if torch.cuda.device_count() < 2 else
           "not measured here: tools/train_dp.py --gpus %d --sync-bn under torchrun" % torch.cuda.device_count()}
    print("card: %s, power limit / max SM clock: %s" % (card, power))
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
