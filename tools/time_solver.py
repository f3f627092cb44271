"""Times the solver (csrc/solver.cu, DESIGN.md section 3.11) on one GPU and prints the card name and power limit, then one
JSON line:
  adam_step           ssd3d_adam_step over the n = 2 513 858 parameters of ARCH_3DSSD + head against
                      torch.optim.Adam.step() over the same tensors, alternating, CUDA events around every call: that is
                      what a caller waits for, host enqueue included.  The kernel alone is timed as a CUDA graph of 20
                      launches replayed back to back; achieved bytes/s = 28 n / kernel time (4 reads + 3 writes of 4 bytes
                      per element) and its share of the 3.35 TB/s of the H100 SXM data sheet -- the kernel is bound by
                      memory, so that is its share of peak.
  weight_operands     ssd3d_weight_operands for every conv weight against the torch sequence it replaces (FoldedConv of W
                      and of W^T per weight, as _ConvTrain builds them); the kernel alone as above.
  launches_per_step   kernels of one training step (batch 4, detection loss) with and without the operand cache, counted
                      with torch.profiler in runs of their own.
  step_ms             the training step both ways, alternating, profiler off.

    python tools/time_solver.py [--launches 200] [--steps 10] [--batch 4] [--points 16384]
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
PEAK_HBM = 3.35e12            # H100 SXM data sheet, bytes/s


def model(dev, seed=0):
    arch = pkg.config.ARCH_3DSSD
    d = pkg.params.init_params(arch, 1, seed=seed, random_bias=True)
    d.update(pkg.params.init_head_params(pkg.config.layer_channels(arch, 1)[-1], seed=seed + 1))
    return pkg.params.TrainableParams(d, dev)


def timed(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    return s, e


def alternate(fns, rounds, warmup):
    """Run the callables in turn `rounds` times after `warmup` rounds -> median and mean ms of each."""
    for _ in range(warmup):
        for f in fns:
            f()
    torch.cuda.synchronize()
    ev = [[] for _ in fns]
    for _ in range(rounds):
        for i, f in enumerate(fns):
            ev[i].append(timed(f))
    torch.cuda.synchronize()
    ms = [np.array([s.elapsed_time(e) for s, e in lst]) for lst in ev]
    return [{"median_ms": round(float(np.median(m)), 5), "mean_ms": round(float(m.mean()), 5)} for m in ms]


def kernel_ms(fn, launches, per_graph=20):
    """ms per launch of `fn` (one kernel launch) with no host in the way: a graph of per_graph launches, replayed."""
    stream = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        with torch.cuda.graph(graph, stream=stream):
            for _ in range(per_graph):
                fn()
    graph.replay()
    torch.cuda.synchronize()
    reps = max(1, launches // per_graph)
    s, e = timed(lambda: [graph.replay() for _ in range(reps)])
    torch.cuda.synchronize()
    return round(s.elapsed_time(e) / (reps * per_graph), 5)


def torch_operands(tp):
    """What a step's forwards and backwards build without the cache: both folds of every weight."""
    dev = tp.device
    for s in tp.weight_scopes():
        w = tp.tensors[s + "/weights"].detach()
        cin, cout = w.shape
        pkg.params.FoldedConv(w, torch.ones((cout,), dtype=torch.float32, device=dev), torch.zeros((cout,), device=dev))
        pkg.params.FoldedConv(w.t().contiguous(), torch.ones((cin,), dtype=torch.float32, device=dev),
                              torch.zeros((cin,), dtype=torch.float32, device=dev))


def count_kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA and "mem" not in ev.name.lower()[:6])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--points", type=int, default=16384)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_solver.py measures on a CUDA device; none is available")
    dev = torch.device("cuda:0")
    card = torch.cuda.get_device_name(dev)
    try:
        power = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                                        text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        power = "unknown"
    print("card: %s, power limit / max SM clock: %s" % (card, power))
    solver = S.Solver()

    # ---- the two kernels against what they replace -------------------------------------------------------------------
    tp = model(dev)
    adam = S.Adam(tp, solver)
    n = adam.param.numel()
    g = torch.randn((n,), generator=torch.Generator(device=dev).manual_seed(0), device=dev) * 0.01
    adam.grad.copy_(g)
    tq = model(dev)
    opt = torch.optim.Adam(tq.parameters(), lr=1e-3)
    off = 0
    for t in tq.parameters():
        t.grad = g[off:off + t.numel()].view(t.shape).clone()
        off += t.numel()
    T = pkg.tf_ops
    ours = lambda: T.adam_step(adam.param, adam.grad, adam.m, adam.v, adam.state, solver.steps, solver.lr_values(),
                               solver.beta1, solver.beta2, solver.epsilon)
    r_adam = alternate([ours, opt.step], a.launches, 10)
    r_ops = alternate([tp.refresh_operands, lambda: torch_operands(tq)], a.launches, 5)
    k_adam, k_ops = kernel_ms(ours, a.launches), kernel_ms(tp.refresh_operands, a.launches)
    sec = k_adam * 1e-3
    res = {"card": card, "power_limit_max_sm_clock": power, "n_params": n, "tensors": len(tq.parameters()),
           "conv_weights": len(tp.weight_scopes()), "launches_timed": a.launches,
           "adam_step_call": r_adam[0], "torch_adam_step_call": r_adam[1], "adam_step_kernel_ms": k_adam,
           "adam_step_bytes": 28 * n, "adam_step_tb_per_s": round(28 * n / sec / 1e12, 3),
           "adam_step_share_of_3.35_tb_per_s_memory_bound": round(28 * n / sec / PEAK_HBM, 4),
           "weight_operands_call": r_ops[0], "torch_operand_sequence_call": r_ops[1], "weight_operands_kernel_ms": k_ops}
    del tq, opt, adam, tp

    # ---- the training step with and without the operand cache ---------------------------------------------------------
    p, b, l = synth.kitti_like_with_boxes(a.batch, a.points, 40, seed=1)
    xyz, feat = T.split_points(torch.from_numpy(p).to(dev))
    boxes, labels = torch.from_numpy(b).to(dev), torch.from_numpy(l).to(dev)
    cached = S.Trainer(pkg.config.ARCH_3DSSD, model(dev), solver)
    plain = S.Trainer(pkg.config.ARCH_3DSSD, model(dev), solver)
    plain.tp.operand_cache = None                 # measurement only: the same step on the uncached path
    run = [lambda: cached.step(xyz, feat, boxes, labels), lambda: plain.step(xyz, feat, boxes, labels)]
    r_step = alternate(run, a.steps, 2)
    res["step_ms"] = {"operand_cache": r_step[0], "no_cache": r_step[1], "batch": a.batch, "points": a.points, "steps": a.steps}
    res["launches_per_step"] = {"operand_cache": count_kernels(run[0]), "no_cache": count_kernels(run[1])}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
