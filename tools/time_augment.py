"""Time the GPU augmentation plus point choice (augment.Augmentor) for a batch of KITTI-sized scenes: the four kernels
from device-resident scenes and draws to the [B, 16384, 4] block, timed with CUDA events after a warm-up.  Scenes are
synth.kitti_like_with_boxes draws of 18k..24k points with up to 40 boxes (a KITTI frame in the camera's field of view
holds about 20k points), half of them noised, rotated and scaled.  Prints the card name and its power limit, then one
JSON line.

    python tools/time_augment.py [--scenes 8] [--reps 50]
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
synth = importlib.import_module("3dssd_b200.synth")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=8)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--seed", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_augment.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    card = torch.cuda.get_device_name(dev)
    try:
        power = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                        text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        power = "unknown"
    print("card: %s, power limit: %s" % (card, power))
    rng = np.random.default_rng(a.seed)
    sizes = rng.integers(18000, 24001, a.scenes)
    clouds, boxes, labels = [], np.zeros((a.scenes, 40, 7), np.float32), np.zeros((a.scenes, 40), np.int32)
    for s, n in enumerate(sizes):
        p, b, l = synth.kitti_like_with_boxes(1, int(n), 40, seed=a.seed + 101 * s)
        clouds.append(p[0])
        boxes[s], labels[s] = b[0], l[0]
    offsets = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    pts = torch.from_numpy(np.concatenate(clouds)).to(dev)
    gb, gl = torch.from_numpy(boxes).to(dev), torch.from_numpy(labels).to(dev)
    aug = pkg.augment.Augmentor(16384, dev)
    gen = torch.Generator(device=dev).manual_seed(a.seed)
    draws = pkg.augment.draw(a.scenes, 40, int(offsets[-1]), 16384, gen, dev)
    draws = draws._replace(scene_u=torch.full((a.scenes, 6), 0.25, dtype=torch.float64, device=dev))   # every stage on
    for _ in range(3):
        aug(pts, offsets, None, gb, gl, draws)
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(a.reps):
        aug(pts, offsets, None, gb, gl, draws)
    t1.record()
    torch.cuda.synchronize()
    ms = t0.elapsed_time(t1) / a.reps
    print(json.dumps({"card": card, "power_limit": power, "scenes": a.scenes, "points": int(offsets[-1]), "boxes": 40,
                      "augment_ms": round(ms, 4)}))


if __name__ == "__main__":
    main()
