"""Builds tests/golden/realscan_16384.npz from the reference's sample KITTI scan (SURVEY.md section 8d, distribution B).

mayavi/kitti_sample_scan.txt of the reference holds 123 398 velodyne points (x forward, y left, z up).  They are mapped
to the rect camera frame of configs/kitti/3dssd/3dssd.yaml:3 (x_r = -y_v, y_r = -z_v, z_r = x_v), cropped to the
detection range x in (-40, 40), y in (-5, 3), z in (0, 70) and |x| < z (about 90 degrees of field of view), and a seeded
choice of 16 384 of them is stored with a U(0,1) intensity: one real LiDAR scene in the loader's [16384, 4] layout.
Needs a reference checkout (path in $REFERENCE):   REFERENCE=<checkout> python tests/golden/make_realscan.py
"""
import os

import numpy as np

SRC = os.path.join(os.environ.get("REFERENCE", "."), "mayavi", "kitti_sample_scan.txt")
HERE = os.path.dirname(os.path.abspath(__file__))


def main():
    v = np.loadtxt(SRC, dtype=np.float32)
    r = np.stack([-v[:, 1], -v[:, 2], v[:, 0]], axis=1)
    keep = (np.abs(r[:, 0]) < 40) & (r[:, 1] > -5) & (r[:, 1] < 3) & (r[:, 2] > 0) & (r[:, 2] < 70) & (np.abs(r[:, 0]) < r[:, 2])
    r = r[keep]
    rng = np.random.default_rng(1000)
    sel = rng.choice(r.shape[0], 16384, replace=False)
    pts = np.concatenate([r[sel], rng.uniform(0, 1, (16384, 1)).astype(np.float32)], axis=1).astype(np.float32)
    np.savez_compressed(os.path.join(HERE, "realscan_16384.npz"), points=pts, source="mayavi/kitti_sample_scan.txt",
                        kept=int(keep.sum()))
    print("kept", int(keep.sum()), "of", v.shape[0], "-> wrote realscan_16384.npz", pts.shape, pts.min(0), pts.max(0))


if __name__ == "__main__":
    main()
