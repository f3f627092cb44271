"""Per-launch time of the tensor-core GEMMs of one throughput step, every call replayed alone.

    python tools/time_tc_shapes.py [--reps R] [--out DIR]

Runs one eager step of the `bench.py --gpus 1` network (built as tools/profile_step.py builds it) with bench.MlpTimer
wrapped around tf_ops.linear_tc / linear_tc_hoisted / linear_tc_gather, then replays each recorded call alone: once under
torch.profiler to read which kernel and tile width the launch plan picked, then R times back to back between CUDA events.
Per launch it prints the route, rows (8 x the live unit count on unit lists), K, N, the in-step ms MlpTimer saw, the
replayed ms, issued bf16 TFLOP/s (three MMAs per product, padded K and N, as MlpTimer counts them) and the operand bytes
per issued FLOP that the tile implies:
    TMA-fed A (linear_tc):            4 (128 + BN) bytes of A_hi/A_lo/B_hi/B_lo per 6 * 128 * BN FLOP and K element
    A built in shared memory (gather / hoisted routes): 4 BN bytes of B_hi/B_lo per 6 * 128 * BN FLOP.
The replays run with a warm L2 when an operand fits it; the in-step column is what the step itself saw. The card's name,
power limit and clocks are read in the same run. Writes DIR/time_tc_shapes.json (default DIR: <tmp>/time_tc_shapes).
"""
import argparse
import importlib
import json
import os
import re
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

ROUTES = ("linear_tc", "linear_tc_hoisted", "linear_tc_gather")


def shape_of(name, a, kw):
    """(rows, K padded, N) of one recorded call; rows = 8 x units[0] on unit lists."""
    if kw.get("units") is not None:
        rows = int(kw["units"][0].item()) * 8
    elif name == "linear_tc":
        rows = a[0].numel() // a[0].shape[-1]
    else:
        rows = a[5].numel() if name == "linear_tc_hoisted" else a[3].numel()
    f = a[2] if name == "linear_tc" else (a[6] if name == "linear_tc_hoisted" else a[4])
    return rows, f.kp, f.cout


def kernel_of(torch, fn, a, kw):
    """Name of the linear_tc kernel one call launches, from a profiled replay."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn(*a, **kw)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if "linear_tc" in e.name and "kernel" in e.name]
    if not names:
        raise SystemExit("the profiler recorded no linear_tc kernel for a replayed call")
    return names[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20, help="timed back-to-back replays per launch")
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "time_tc_shapes"))
    args = ap.parse_args()

    import torch
    bench = importlib.import_module("bench")
    profile_step = importlib.import_module("profile_step")
    pkg = importlib.import_module("3dssd_b200")
    synth = importlib.import_module("3dssd_b200.synth")
    if not torch.cuda.is_available():
        raise SystemExit("time_tc_shapes.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    arch = pkg.config.ARCH_3DSSD
    params = pkg.params.init_params(arch, 1, seed=0)
    head_params = pkg.params.init_head_params(pkg.config.layer_channels(arch, 1)[-1], seed=1)
    pts = torch.from_numpy(synth.kitti_like(bench.SCENES_PER_GPU, bench.NPOINTS, seed=1000)).to(dev)
    head = pkg.DetectionHead(params=head_params, device=dev)
    net = pkg.SABackbone(arch, params, in_channels=1, device=dev, ffps_mode="direct", mlp_mode="tc", head=head,
                         gather_in_kernel=True, hoist_first=2, fps_cluster=-4, latency_mode=False,
                         fps_packet=False, fps_bucket=None)
    gather = pkg.dist.DetectionGather(bench.SCENES_PER_GPU, dev)

    def step():
        out = net.forward(pts)
        net.detections(out[0], out[1], out=gather.out())

    for _ in range(2):
        step()
    torch.cuda.synchronize()
    torch.cuda._sleep(int(0.08 * 1.9e9))        # as bench.py: keep the GPU busy so each event pair brackets kernel time
    mt = bench.MlpTimer(torch, pkg.tf_ops)
    with mt:
        step()
    torch.cuda.synchronize()
    fns = {n: mt.saved[n] for n in ROUTES}

    rows_out = []
    for name, e0, e1, a, kw in mt.rec:
        if name not in ROUTES:
            continue
        fn = fns[name]
        rows, kp, n = shape_of(name, a, kw)
        flop = 3.0 * mt._flops(name, a, kw)
        kname = kernel_of(torch, fn, a, kw)
        m = re.search(r"<(\d+)", kname)
        bn = int(m.group(1)) if m else 0
        tma_a = name == "linear_tc"
        op_bytes = 4 * ((128 if tma_a else 0) + bn)
        for _ in range(3):
            fn(*a, **kw)
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda._sleep(int(0.01 * 1.9e9))     # the host enqueues every replay before the first one runs
        t0.record()
        for _ in range(args.reps):
            fn(*a, **kw)
        t1.record()
        torch.cuda.synchronize()
        ms = t0.elapsed_time(t1) / args.reps
        rows_out.append({"route": name, "units": kw.get("units") is not None, "unit_pool": bool(kw.get("unit_pool", False)),
                         "rows": rows, "kp": kp, "n": n, "kernel": kname.split("(")[0].replace("void ", "").strip(),
                         "bn": bn, "gflop_issued": flop / 1e9, "ms_in_step": e0.elapsed_time(e1), "ms": ms,
                         "tflops_issued": flop / (ms * 1e-3) / 1e12,
                         "operand_bytes_per_flop": op_bytes / (6.0 * 128 * bn) if bn else None})
    card = profile_step.card_info(torch)
    tot_fl = sum(r["gflop_issued"] for r in rows_out)
    tot_ms = sum(r["ms"] for r in rows_out)
    print("card: %(name)s, power limit %(power_limit_w).0f W, max SM clock %(sm_max_mhz)d MHz, SM clock now %(sm_mhz_now)d MHz"
          % card)
    print("%-18s %6s %7s %5s %5s %-26s %8s %8s %8s %8s %7s" % ("route", "pool", "rows", "K", "N", "kernel", "GFLOP", "ms step",
                                                          "ms", "TFLOP/s", "B/FLOP"))
    for r in sorted(rows_out, key=lambda r: -r["gflop_issued"]):
        print("%-18s %6s %7d %5d %5d %-26s %8.2f %8.4f %8.4f %8.1f %7.4f" % (
            r["route"] + ("+units" if r["units"] else ""), "unit" if r["unit_pool"] else "", r["rows"], r["kp"], r["n"],
            r["kernel"][-26:], r["gflop_issued"], r["ms_in_step"], r["ms"], r["tflops_issued"],
            r["operand_bytes_per_flop"] or 0.0))
    print("%d launches, %.1f GFLOP issued, %.3f ms replayed alone: %.1f TFLOP/s" % (len(rows_out), tot_fl, tot_ms,
                                                                                    tot_fl / tot_ms))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "time_tc_shapes.json"), "w") as f:
        json.dump({"card": card, "reps": args.reps, "launches": rows_out}, f, indent=1)
    print("wrote", os.path.join(args.out, "time_tc_shapes.json"))


if __name__ == "__main__":
    main()
