"""Build the mixup object database (mixup.ObjectDatabase, DESIGN.md section 3.13) on the GPU and save it as one .npz.

    python tools/build_mixup_db.py --data DIR --out DB.npz [--batch 8]
    python tools/build_mixup_db.py --synthetic N --out DB.npz

--data reads the reference's per-frame sample dicts (*.npy, kitti_io.read_sample) in name order, --batch frames at a
time through kitti_io.make_ragged_batch; --synthetic builds from N synth.kitti_like_with_boxes scenes.  Every Car row
holding at least 5 points of its frame inside the row grown by 0.1 becomes an object with those points, as the
reference's preprocessing does (generate_mixup_sample).  Prints the object and point totals."""
import argparse
import glob
import importlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("3dssd_b200")
synth = importlib.import_module("3dssd_b200.synth")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--data", default=None, help="directory of the reference's per-frame sample dicts (*.npy)")
    ap.add_argument("--synthetic", type=int, default=0, help="build from this many synthetic scenes instead")
    ap.add_argument("--out", required=True)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--seed", type=int, default=500, help="seed of the synthetic scenes")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("build_mixup_db.py builds on a CUDA device; none is available")
    if bool(a.data) == bool(a.synthetic):
        raise SystemExit("give exactly one of --data DIR and --synthetic N")
    dev = torch.device("cuda", 0)
    MX = pkg.mixup
    parts = []
    if a.data:
        files = sorted(glob.glob(os.path.join(a.data, "*.npy")))
        if not files:
            raise SystemExit("--data %s holds no *.npy sample" % a.data)
        for first in range(0, len(files), a.batch):
            samples = [pkg.kitti_io.read_sample(f) for f in files[first:first + a.batch]]
            pts, off, _, boxes, labels = pkg.kitti_io.make_ragged_batch(samples)
            parts.append(MX.ObjectDatabase.build(pts, off.numpy(), boxes, labels, frame_base=first, device=dev))
    else:
        for first in range(0, a.synthetic, a.batch):
            n = min(a.batch, a.synthetic - first)
            p, b, l = synth.kitti_like_with_boxes(n, 20000, 40, seed=a.seed + first)
            off = np.arange(0, (n + 1) * 20000, 20000)
            parts.append(MX.ObjectDatabase.build(p.reshape(-1, 4), off, b, l, frame_base=first, device=dev))
    db = MX.ObjectDatabase.concat(parts)
    db.save(a.out)
    print("%d objects, %d points -> %s" % (len(db), int(db.host_offsets[-1]), a.out))


if __name__ == "__main__":
    main()
