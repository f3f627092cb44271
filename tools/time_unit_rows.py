"""Every unit-list launch of one eager bench step at 8 and at 4 rows per unit, launch by launch.

    python tools/time_unit_rows.py [--reps R] [--out DIR]

Builds the `bench.py --gpus 1` backbone (8 scenes x 16384 points, kitti_like seed 1000, init_params seed 0) twice, with
layers_util.UNIT_ROWS = 8 and = 4, runs one eager step of each to warm up, then runs the step R more times with every
unit-list call of tf_ops (sa_mlp_fused[_hoisted], linear_tc[_hoisted] on a list, hoist_expand_split on a list) between
CUDA events.  Per launch it prints the route, the convolved rows (units[0] x W, read after the step), the median
event ms and the issued bf16 TFLOP/s from those rows (three MMAs per product, K and N padded to 16).  Both widths'
outputs are compared bit for bit.  The card's name and power limit are read in the same run.
Writes DIR/time_unit_rows.json (default DIR: <tmp>/time_unit_rows).
"""
import argparse
import functools
import importlib
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

pkg = importlib.import_module("3dssd_b200")
T, lu = pkg.tf_ops, importlib.import_module("3dssd_b200.layers_util")
synth = importlib.import_module("3dssd_b200.synth")

ROUTES = ("sa_mlp_fused", "sa_mlp_fused_hoisted", "linear_tc", "linear_tc_hoisted", "hoist_expand_split")


def _r16(x):
    return (int(x) + 15) // 16 * 16


def _flop_per_row(name, a, kw):
    """Issued MMA FLOP per convolved row: 3 split products x 2 x padded K x padded N, over the convs of the call"""
    if name.startswith("sa_mlp_fused"):
        st = a[7] if name == "sa_mlp_fused_hoisted" else a[5]
        dims = [st.cin] + list(st.nout)
        return sum(6 * _r16(k) * _r16(n) for k, n in zip(dims[:-1], dims[1:]))
    if name == "hoist_expand_split":
        return 0
    f = a[2] if name == "linear_tc" else a[6]
    return 6 * f.kp * _r16(f.cout)


def run(width, pts, arch, params, reps):
    lu.UNIT_ROWS = width
    net = pkg.SABackbone(arch, params, in_channels=1, device=pts.device)
    out = net.forward(pts)
    torch.cuda.synchronize()
    log = []
    orig = {n: getattr(T, n) for n in ROUTES}

    def timed(name, fn):
        @functools.wraps(fn)
        def call(*a, **kw):
            units = kw.get("units")
            if units is None:
                return fn(*a, **kw)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            r = fn(*a, **kw)
            e1.record()
            log.append((name, a, kw, units, e0, e1))
            return r
        return call
    for n in ROUTES:
        setattr(T, n, timed(n, orig[n]))
    per = {}
    try:
        for _ in range(reps):
            log.clear()
            out = net.forward(pts)
            torch.cuda.synchronize()
            for i, (name, a, kw, units, e0, e1) in enumerate(log):
                rows = int(units[0].item()) * getattr(units, "unit_rows", 8)
                d = per.setdefault(i, dict(route=name, rows=rows, flop=rows * _flop_per_row(name, a, kw), ms=[]))
                d["ms"].append(e0.elapsed_time(e1))
    finally:
        for n in ROUTES:
            setattr(T, n, orig[n])
        lu.UNIT_ROWS = 4
    res = []
    for i in sorted(per):
        d = per[i]
        ms = float(np.median(d["ms"]))
        res.append(dict(route=d["route"], rows=d["rows"], ms=ms, tflops=d["flop"] / ms / 1e9 if d["flop"] else None))
    return res, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=os.path.join(tempfile.gettempdir(), "time_unit_rows"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_unit_rows: needs a CUDA device")
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    arch = pkg.config.ARCH_3DSSD
    params = pkg.params.init_params(arch, 1, seed=0)
    pts = torch.from_numpy(synth.kitti_like(8, 16384, seed=1000)).cuda()
    r8, o8 = run(8, pts, arch, params, args.reps)
    r4, o4 = run(4, pts, arch, params, args.reps)

    def flat(o):
        if isinstance(o, torch.Tensor):
            return [o]
        return [t for x in (o if isinstance(o, (list, tuple)) else []) for t in flat(x)]
    same = all(torch.equal(x, y) for x, y in zip(flat(o8), flat(o4))) and len(flat(o8)) == len(flat(o4))
    print("card: %s | outputs bit-identical: %s" % (card, same))
    print("%3s %-22s %9s %9s %8s %8s %7s %7s %6s" % ("#", "route", "rows W=8", "rows W=4", "ms W=8", "ms W=4", "TF/s 8", "TF/s 4",
                                                    "t4/t8"))
    for i, (a, b) in enumerate(zip(r8, r4)):
        tf = lambda d: "%7.1f" % d["tflops"] if d["tflops"] else "      -"
        print("%3d %-22s %9d %9d %8.4f %8.4f %s %s %6.2f" % (i, a["route"], a["rows"], b["rows"], a["ms"], b["ms"], tf(a), tf(b),
                                                           b["ms"] / a["ms"]))
    t8, t4 = sum(d["ms"] for d in r8), sum(d["ms"] for d in r4)
    print("sum of unit-list launches: %.3f ms at W=8, %.3f ms at W=4 (%.2fx)" % (t8, t4, t4 / t8))
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "time_unit_rows.json"), "w") as fh:
        json.dump(dict(card=card, identical=same, w8=r8, w4=r4), fh, indent=1)


if __name__ == "__main__":
    main()
