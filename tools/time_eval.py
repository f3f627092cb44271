"""Time the GPU KITTI evaluator (tf_ops.evaluate_labels) against its single-threaded C twin (oracle/kitti_eval_twin.c)
on a synthetic 3,769-frame validation set (the size of KITTI val).  The GPU figure is the whole call -- uploads, the three
launches, the host getThresholds step between them and the precision curves -- timed with CUDA events after a warm-up;
the host threshold step is also timed on its own.  Prints the card name and its power limit, then one JSON line.

    python tools/time_eval.py [--frames 3769] [--reps 5]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("3dssd_b200")
from oracle import kitti_eval as K  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=3769)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=11)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_eval.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    card = torch.cuda.get_device_name(dev)
    try:
        power = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                        text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        power = "unknown"
    print("card: %s, power limit: %s" % (card, power))
    rows, labels, nl = K.synthetic_frames(a.frames, seed=a.seed, max_labels=12)
    pairs = int(sum(int(n) * len(l) for n, l in zip(nl, labels)))
    d_rows, d_nl = torch.from_numpy(rows).to(dev), torch.from_numpy(nl).to(dev)

    ev = lambda: pkg.tf_ops.evaluate_labels(d_rows, labels, d_nl)
    ref = ev()                                             # warm-up (and the result to check)
    torch.cuda.synchronize()
    gpu_ms = []
    for _ in range(a.reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        ev()
        e1.record()
        e1.synchronize()
        gpu_ms.append(e0.elapsed_time(e1))

    # the host step alone: getThresholds for every evaluated case, on as many scores as 60% of the label rows (about
    # the true positives of this set's first pass)
    flags = pkg.evaluation.eval_flags(rows)
    rng = np.random.default_rng(0)
    tp_scores = [rng.uniform(0.3, 1, int(0.6 * sum(len(l) for l in labels))) for _ in range(27)]
    t0 = time.perf_counter()
    for cs in range(27):
        if flags[cs // 9][(cs // 3) % 3]:
            pkg.evaluation.get_thresholds(tp_scores[cs], len(tp_scores[cs]) + 100)
    host_ms = (time.perf_counter() - t0) * 1e3

    K.build()
    t0 = time.perf_counter()
    exp = K.twin_evaluate(rows, labels, nl)
    twin_ms = (time.perf_counter() - t0) * 1e3
    same = all(np.array_equal(x.cpu().numpy(), y, equal_nan=True) for x, y in zip(ref, exp))
    gpu = float(np.median(gpu_ms))
    res = {"card": card, "power_limit": power, "frames": a.frames, "detections": int(rows.shape[0]),
           "label_rows": int(sum(len(l) for l in labels)), "pairs": pairs, "gpu_evaluate_ms": round(gpu, 2),
           "gpu_evaluate_ms_all": [round(x, 2) for x in gpu_ms], "host_thresholds_ms": round(host_ms, 2),
           "twin_cpu_ms": round(twin_ms, 1), "twin_over_gpu": round(twin_ms / gpu, 2), "bit_identical": same}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
