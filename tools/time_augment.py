"""Time the GPU augmentation plus point choice (augment.Augmentor) for a batch of KITTI-sized scenes: the four kernels
from device-resident scenes and draws to the [B, 16384, 4] block, timed with CUDA events after a warm-up.  Scenes are
synth.kitti_like_with_boxes draws of 18k..24k points with up to 40 boxes (a KITTI frame in the camera's field of view
holds about 20k points), half of them noised, rotated and scaled.  Prints the card name and its power limit, then one
JSON line.  With --mixup the same call with the mixup paste in front (15 objects drawn per scene from a database
built from other synthetic scenes, flat ground planes) is timed in the same run, the two alternating rep by rep.

    python tools/time_augment.py [--scenes 8] [--reps 50] [--mixup]
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
    ap.add_argument("--mixup", action="store_true", help="also time the call with the mixup paste, alternating")
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
    calls = {"augment_ms": lambda: aug(pts, offsets, None, gb, gl, draws)}
    extra = {}
    if a.mixup:
        MX = pkg.mixup
        p, b, l = synth.kitti_like_with_boxes(16, 20000, 40, seed=a.seed + 7777)
        db = MX.ObjectDatabase.build(p.reshape(-1, 4), np.arange(0, 17 * 20000, 20000), b, l, device=dev)
        ids = MX.Sampler(db, seed=a.seed).ids(0, a.scenes)
        planes = np.tile(np.asarray(MX.FLAT_PLANE, np.float64), (a.scenes, 1))
        lay = MX.layout(offsets, ids, db.host_offsets, 40)
        mdraws = pkg.augment.draw(a.scenes, lay.rows, lay.total, 16384, gen, dev)
        mdraws = mdraws._replace(scene_u=torch.full((a.scenes, 6), 0.25, dtype=torch.float64, device=dev))
        mix = MX.Mixup(db, ids, planes)
        calls["augment_mixup_ms"] = lambda: aug(pts, offsets, None, gb, gl, mdraws, mixup=mix)
        extra = {"db_objects": len(db), "drawn": int((ids >= 0).sum()), "pasted_points": lay.total - int(offsets[-1])}
    for f in calls.values():
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    total = {k: 0.0 for k in calls}
    for _ in range(a.reps):                                # alternate the variants rep by rep
        for k, f in calls.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            f()
            t1.record()
            torch.cuda.synchronize()
            total[k] += t0.elapsed_time(t1)
    res = {"card": card, "power_limit": power, "scenes": a.scenes, "points": int(offsets[-1]), "boxes": 40}
    res.update({k: round(v / a.reps, 4) for k, v in total.items()})
    res.update(extra)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
