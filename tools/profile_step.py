"""Where the SM-time of one throughput step goes, per kernel, under torch.profiler (CUDA activities).

    python tools/profile_step.py [--steps S] [--out DIR]

Builds the step exactly as `bench.py --gpus 1` does (same arch, seeds, head and options: D-FPS cluster cap -4 as in the
pipelined step, bucket layer-1 FPS, gather-in-kernel, hoist_first=2) and runs S eager steps after two warm-up steps.
Steps of the throughput benchmark overlap 24 deep, so what bounds them is SM-time, not latency: per kernel name this
prints launches, total duration, grid size and SM-ms = duration x min(CTAs of the grid, 132), and each kernel's share
of the step's SM-ms.  Writes DIR/profile_step.json (default DIR: <tmp>/profile_step) with the card's name, power
limit and max SM clock read in the same run.
"""
import argparse
import importlib
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

NUM_SMS = 132


def card_info(torch):
    """NVML's view of the card torch runs on (matched by UUID: NVML ignores CUDA_VISIBLE_DEVICES)."""
    import pynvml
    pynvml.nvmlInit()
    h = pynvml.nvmlDeviceGetHandleByUUID("GPU-" + str(torch.cuda.get_device_properties(0).uuid))
    name = pynvml.nvmlDeviceGetName(h)
    return {"name": name.decode() if isinstance(name, bytes) else name,
            "power_limit_w": pynvml.nvmlDeviceGetPowerManagementLimit(h) / 1000.0,
            "sm_max_mhz": pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM),
            "sm_mhz_now": pynvml.nvmlDeviceGetClockInfo(h, pynvml.NVML_CLOCK_SM)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3, help="profiled eager steps (totals are divided by this)")
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "profile_step"))
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    bench = importlib.import_module("bench")
    pkg = importlib.import_module("3dssd_b200")
    synth = importlib.import_module("3dssd_b200.synth")
    if not torch.cuda.is_available():
        raise SystemExit("profile_step.py needs a CUDA device")
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
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        trace = json.load(open(path))

    rows = {}
    for ev in trace.get("traceEvents", []):
        if ev.get("cat") != "kernel":
            continue
        grid = ev.get("args", {}).get("grid", [1, 1, 1])
        ctas = grid[0] * grid[1] * grid[2]
        dur_ms = float(ev.get("dur", 0.0)) * 1e-3
        name = ev["name"].split("(")[0].split("<")[0].replace("void ", "").strip()
        r = rows.setdefault(name, {"launches": 0, "ms": 0.0, "sm_ms": 0.0, "grids": set()})
        r["launches"] += 1
        r["ms"] += dur_ms
        r["sm_ms"] += dur_ms * min(ctas, NUM_SMS)
        r["grids"].add(ctas)
    if not rows:
        raise SystemExit("the profiler recorded no kernels")
    total = sum(r["sm_ms"] for r in rows.values())
    table = []
    for name, r in sorted(rows.items(), key=lambda kv: -kv[1]["sm_ms"]):
        table.append({"kernel": name, "launches_per_step": r["launches"] / args.steps, "ms_per_step": r["ms"] / args.steps,
                      "grid_ctas": sorted(r["grids"]), "sm_ms_per_step": r["sm_ms"] / args.steps,
                      "share": r["sm_ms"] / total})
    res = {"card": card_info(torch), "steps": args.steps, "sm_ms_per_step": total / args.steps,
           "note": "eager steps of the bench.py --gpus 1 throughput network; SM-ms = kernel duration x min(grid CTAs, %d)"
                   % NUM_SMS, "kernels": table}
    print("card: %(name)s, power limit %(power_limit_w).0f W, max SM clock %(sm_max_mhz)d MHz" % res["card"])
    print("%-34s %8s %10s %14s %10s %7s" % ("kernel", "launches", "ms", "grid CTAs", "SM-ms", "share"))
    for t in table:
        g = t["grid_ctas"]
        gs = str(g[0]) if len(g) == 1 else "%d-%d" % (g[0], g[-1])
        print("%-34s %8.1f %10.3f %14s %10.2f %6.1f%%" % (t["kernel"][:34], t["launches_per_step"], t["ms_per_step"], gs,
                                                         t["sm_ms_per_step"], 100 * t["share"]))
    print("total SM-ms per step: %.2f" % res["sm_ms_per_step"])
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "profile_step.json"), "w") as f:
        json.dump(res, f, indent=1)
    print("wrote", os.path.join(args.out, "profile_step.json"))


if __name__ == "__main__":
    main()
