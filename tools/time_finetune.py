"""Time one full training step of 3DSSD against one fine-tuning step with a frozen backbone (DESIGN.md section 3.19):
solver.Trainer steps (forward, targets, losses, backward, clip / exchange at world size 1, optimizer) at --batch x
--points on synth.kitti_like_with_boxes scenes, once with every variable trained and once with only --train-prefix
trained.  Both trainers are warmed up, then timed with CUDA events in alternating rounds of --round steps until each has
run for about --seconds, so that clock and thermal drift fall on both alike.  Prints the card name and its power limit
beside the times, then one JSON line.

    python tools/time_finetune.py [--batch 4] [--points 16384] [--train-prefix layer4,conv1d_0,pred_] [--seconds 20]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--points", type=int, default=16384)
    ap.add_argument("--max-boxes", type=int, default=40)
    ap.add_argument("--train-prefix", default="layer4,conv1d_0,pred_")
    ap.add_argument("--solver", choices=("adam", "momentum"), default="adam")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--round", type=int, default=5, help="steps per timed round")
    ap.add_argument("--seconds", type=float, default=20.0, help="timed seconds per configuration (about)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_finetune.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    card = torch.cuda.get_device_name(dev)
    try:
        prop = torch.cuda.get_device_properties(dev)                 # query the timed card only, by its PCI address
        bus = "%08X:%02X:%02X.0" % (prop.pci_domain_id, prop.pci_bus_id, prop.pci_device_id)
        power = subprocess.check_output(["nvidia-smi", "-i", bus, "--query-gpu=power.limit,clocks.max.sm",
                                         "--format=csv,noheader"], text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        power = "unknown"
    print("card: %s, power limit / max SM clock: %s" % (card, power))
    arch = pkg.config.ARCH_3DSSD
    d = pkg.params.init_params(arch, 1, seed=0, random_bias=True)
    d.update(pkg.params.init_head_params(pkg.config.layer_channels(arch, 1)[-1], seed=1))
    synth = importlib.import_module("3dssd_b200.synth")
    p, boxes, labels = synth.kitti_like_with_boxes(a.batch, a.points, a.max_boxes, seed=1)
    xyz, feat = pkg.tf_ops.split_points(torch.from_numpy(p).to(dev))
    gb, gl = torch.from_numpy(boxes).to(dev), torch.from_numpy(labels).to(dev)
    prefixes = [s for s in a.train_prefix.split(",") if s]
    solver = S.Solver(type=a.solver)
    runs = {"full": S.Trainer(arch, pkg.params.TrainableParams(d, dev), solver),
            "frozen": S.Trainer(arch, pkg.params.TrainableParams(d, dev, trainable=prefixes), solver)}
    for tr in runs.values():
        for _ in range(a.warmup):
            tr.step(xyz, feat, gb, gl)
    torch.cuda.synchronize()
    times = {k: [] for k in runs}
    while min(sum(v) for v in times.values()) < 1e3 * a.seconds:
        for k, tr in runs.items():                                  # alternate the two configurations round by round
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(a.round):
                tr.step(xyz, feat, gb, gl)
            e.record()
            e.synchronize()
            times[k].append(s.elapsed_time(e))
    res = {"card": card, "power_limit_max_sm_clock": power, "batch": a.batch, "points": a.points, "solver": a.solver,
           "train_prefix": prefixes, "rounds": len(times["full"]), "steps_per_round": a.round,
           "trained_floats": {k: int(tr.optimizer.param.numel()) for k, tr in runs.items()}}
    for k, v in times.items():
        per = np.array(v) / a.round
        res["%s_step_ms" % k] = {"median": round(float(np.median(per)), 3), "min": round(float(per.min()), 3),
                                 "max": round(float(per.max()), 3)}
        print("%-6s step: median %.3f ms (min %.3f, max %.3f) over %d rounds of %d" % (k, np.median(per), per.min(), per.max(),
                                                                                       len(v), a.round))
    res["frozen_over_full"] = round(res["frozen_step_ms"]["median"] / res["full_step_ms"]["median"], 4)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
