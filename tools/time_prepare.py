"""Time the KITTI preprocessing pass (prepare.py, DESIGN.md section 3.14) on seeded synthetic raw frames.

    python tools/time_prepare.py --out DIR [--frames 64] [--points 120000] [--batch 32] [--repeats 20]

Writes a raw KITTI-layout tree of --frames seeded velodyne sweeps (360 degrees, about --points points each, a KITTI
calibration, 1242 x 375 images, four Car rows per frame) under DIR/raw, then reports
  kernel   tf_ops.prepare_points on one batch of --batch frames already on the device: CUDA events, warmed, the median
           of --repeats launches
  tool     tools/prepare_kitti.py's pass over the whole tree into DIR/out: frames/s, with the time waited for reading,
           spent in the batch's GPU work (kernel, semantic labels, the one synchronisation and copy back) and writing
  twin     the numpy twin (oracle/prepare.py) on the same frames: CPU seconds per frame.  This is the twin, not the
           reference's own pass (which needs TensorFlow)
Prints the card name and its power limit first.  Needs a CUDA device."""
import argparse
import importlib
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("3dssd_b200")
PR = importlib.import_module("3dssd_b200.prepare")
sys.path.insert(0, os.path.join(ROOT, "tools"))
import prepare_kitti  # noqa: E402
from oracle import prepare as OP  # noqa: E402

KITTI = {"P2": "7.215377e+02 0 6.095593e+02 4.485728e+01 0 7.215377e+02 1.728540e+02 2.163791e-01 0 0 1 2.745884e-03",
         "R0_rect": "9.999239e-01 9.837760e-03 -7.445048e-03 -9.869795e-03 9.999421e-01 -4.278459e-03 7.402527e-03 "
                    "4.351614e-03 9.999631e-01",
         "Tr_velo_to_cam": "7.533745e-03 -9.999714e-01 -6.166020e-04 -4.069766e-03 1.480249e-02 7.280733e-04 -9.998902e-01 "
                           "-7.631618e-02 9.998621e-01 7.523790e-03 1.480755e-02 -2.717806e-01"}


def png(w, h):
    import zlib

    def chunk(t, data):
        return len(data).to_bytes(4, "big") + t + data + (zlib.crc32(t + data) & 0xFFFFFFFF).to_bytes(4, "big")
    return b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", w.to_bytes(4, "big") + h.to_bytes(4, "big") + bytes([8, 2, 0, 0, 0])) + chunk(b"IEND", b"")


def sweep(rng, n):
    az = rng.uniform(-np.pi, np.pi, n)
    r = 2 + rng.exponential(18, n)
    el = rng.uniform(-0.43, 0.03, n)
    return np.stack([r * np.cos(az) * np.cos(el), r * np.sin(az) * np.cos(el), 1.73 + r * np.sin(el), rng.uniform(0, 1, n)],
                    1).astype(np.float32)


def write_tree(root, frames, points, seed=0):
    rng = np.random.default_rng(seed)
    d = os.path.join(root, "training")
    for sub in ("velodyne", "calib", "image_2", "label_2"):
        os.makedirs(os.path.join(d, sub), exist_ok=True)
    calib = "".join("%s: %s\n" % kv for kv in KITTI.items())
    for i in range(frames):
        f = "%06d" % i
        sweep(rng, int(points * rng.uniform(0.95, 1.05))).tofile(os.path.join(d, "velodyne", f + ".bin"))
        open(os.path.join(d, "calib", f + ".txt"), "w").write(calib)
        open(os.path.join(d, "image_2", f + ".png"), "wb").write(png(1242, 375))
        lines = ["Car 0.00 0 -1.57 100 150 300 250 1.56 1.70 3.90 %.2f 1.65 %.2f %.2f" % (rng.uniform(-12, 12), rng.uniform(8, 40),
                                                                                        rng.uniform(-3, 3)) for _ in range(4)]
        open(os.path.join(d, "label_2", f + ".txt"), "w").write("\n".join(lines) + "\n")
    lst = os.path.join(root, "train.txt")
    open(lst, "w").write("\n".join("%06d" % i for i in range(frames)) + "\n")
    return d, lst


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--points", type=int, default=120000)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--repeats", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_prepare.py times the GPU pass; no CUDA device is available")
    dev = torch.device("cuda", 0)
    try:
        power = subprocess.check_output(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                                        text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        power = "unknown"
    print("card: %s, power limit: %s" % (torch.cuda.get_device_name(dev), power))
    raw = os.path.join(a.out, "raw")
    split_dir, lst = write_tree(raw, a.frames, a.points)
    frames = [PR.read_frame(split_dir, i, i, ("Car",)) for i in range(min(a.batch, a.frames))]
    off = np.concatenate([[0], np.cumsum([len(f.points) for f in frames])])
    pts = torch.from_numpy(np.concatenate([f.points for f in frames])).to(dev)
    calib = torch.from_numpy(np.stack([f.calib for f in frames])).to(dev)
    hw = np.array([f.hw for f in frames])
    for _ in range(3):
        pkg.tf_ops.prepare_points(pts, off, calib, hw)
    times = []
    for _ in range(a.repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        pkg.tf_ops.prepare_points(pts, off, calib, hw)
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1))
    kernel_ms = float(np.median(times))
    print("kernel: %.3f ms per batch of %d frames (%d points), median of %d" % (kernel_ms, len(frames), int(off[-1]), a.repeats))
    t0 = time.perf_counter()
    st = prepare_kitti.run(raw, "training", lst, os.path.join(a.out, "out"), batch=a.batch, device=dev, log=lambda *s: None)
    wall = time.perf_counter() - t0
    print("tool: %d frames in %.3f s = %.1f frames/s; read (waited) %.3f s, gpu %.3f s, write %.3f s; %d of %d points kept"
          % (st["read"], wall, st["read"] / wall, st["t_read"], st["t_gpu"], st["t_write"], st["points_kept"], st["points_read"]))
    k = min(8, len(frames))
    t0 = time.perf_counter()
    OP.prepare([(f.name, f.points, f.calib, f.hw, f.boxes, f.classes) for f in frames[:k]])
    twin = (time.perf_counter() - t0) / k
    print("numpy twin (oracle/prepare.py, not the reference): %.1f ms per frame on the CPU" % (1e3 * twin))


if __name__ == "__main__":
    main()
