"""Time what several classes cost on one GPU, in one process, with the arms alternated round by round:

  nms        the NMS at B = 8, n = 256: C = 1 with ssd3d_bev_nms, C = 3 with the cluster kernel ssd3d_bev_nms_classes,
             C = 3 as three sequential single-class calls (the reference's class loop); each form twice: called from
             Python (host work, wrapper checks and launch included) and replayed from a CUDA graph that holds only its
             kernels (the GPU time of the kernels, back to back)
  inference  the captured 3DSSD inference step (backbone + head + NMS, one CUDA graph) at B = 8 x 16384, C = 1 vs C = 3
  train      one training step (solver.Trainer.step) at --train-batch x 16384, C = 1 vs C = 3

    python tools/time_multiclass.py [--rounds 7] [--reps 50] [--train-batch 4] [--out FILE.json]

Each number is the median over --rounds rounds of the mean over --reps back-to-back runs (CUDA events).  The card's
name and power limit are printed next to the numbers."""
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
synth = importlib.import_module("3dssd_b200.synth")
CLS3 = ("Car", "Pedestrian", "Cyclist")


def card():
    """(name, power limit) of device 0, read with a query only."""
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "unknown"
    return name, out or "unknown"


def time_ms(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def alternate(arms, rounds, reps):
    for fn in arms.values():                    # warm-up: caches, shared-memory attributes, first launches
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    got = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            got[k].append(time_ms(fn, reps))
    return {k: float(np.median(v)) for k, v in got.items()}


def weights(c, seed=0):
    arch = pkg.config.ARCH_3DSSD
    d = pkg.params.init_params(arch, 1, seed=seed, random_bias=True)
    d.update(pkg.params.init_head_params(pkg.config.layer_channels(arch, 1)[-1], cls_channels=c, seed=seed + 1))
    return d


def nms_arms(dev):
    rng = np.random.default_rng(0)
    ctr = rng.uniform(-15, 15, (8, 256, 3)).astype(np.float32)
    boxes = torch.from_numpy(np.concatenate([ctr, rng.uniform(0.5, 4.5, (8, 256, 3)), rng.uniform(-3, 3, (8, 256, 1))], -1)
                             .astype(np.float32)).to(dev)
    scores = torch.from_numpy(rng.uniform(0, 1, (8, 256, 3)).astype(np.float32)).to(dev)
    cols = [scores[..., k].contiguous() for k in range(3)]
    T = pkg.tf_ops
    forms = {"nms_c1": lambda: T.bev_nms(boxes, cols[0], 0.1, 100),
             "nms_c3_cluster": lambda: T.bev_nms(boxes, scores, 0.1, 100, cls_num=3),
             "nms_c3_loop": lambda: [T.bev_nms(boxes, cols[k], 0.1, 100, cls_id=k) for k in range(3)]}
    arms = dict(forms)
    for name, fn in forms.items():
        arms[name + "_graph"] = graph_of(fn)
    return arms


def graph_of(fn):
    """fn captured into a CUDA graph (after a warm-up call on a side stream) -> its replay."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g.replay


def inference_arms(dev):
    arms = {}
    for c in (1, 3):
        w = weights(c)
        net = pkg.SABackbone(params=w, in_channels=1, device=dev, head=pkg.DetectionHead(params=w, device=dev))
        pts = torch.from_numpy(synth.kitti_like_multiclass(8, 16384, 20, CLS3[:c], seed=1)[0]).to(dev)
        replay = net.capture(pts)
        # the graph reads the network's weights in place: the closure keeps the network alive with it
        arms["inference_c%d" % c] = (lambda replay=replay, net=net: replay())
    return arms


def train_arms(dev, batch):
    arms = {}
    for c in (1, 3):
        tr = pkg.solver.Trainer(pkg.config.ARCH_3DSSD, pkg.params.TrainableParams(weights(c), dev), pkg.solver.Solver())
        p, b, l = synth.kitti_like_multiclass(batch, 16384, 20, CLS3[:c], seed=2)
        xyz, feat = pkg.tf_ops.split_points(torch.from_numpy(p).to(dev))
        scene = (xyz, feat, torch.from_numpy(b).to(dev), torch.from_numpy(l).to(dev))
        arms["train_c%d" % c] = (lambda tr=tr, scene=scene: tr.step(*scene))
    return arms


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--train-batch", type=int, default=4)
    ap.add_argument("--out", default=None, help="also write the numbers as JSON")
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("time_multiclass.py times CUDA kernels; no device is available")
    dev = torch.device("cuda", 0)
    name, power = card()
    res = {"card": name, "power_limit": power}
    res.update(alternate(nms_arms(dev), a.rounds, a.reps))
    res.update(alternate(inference_arms(dev), a.rounds, max(1, a.reps // 5)))
    res.update(alternate(train_arms(dev, a.train_batch), a.rounds, max(1, a.reps // 10)))
    print("%s, power limit %s" % (name, power))
    for k, v in res.items():
        if isinstance(v, float):
            print("%-22s %9.4f ms" % (k, v))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
