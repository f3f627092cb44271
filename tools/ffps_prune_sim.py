"""CPU simulation of the skip rule of ffps_bucket_kernel (csrc/fps.cu) on the benchmark's layer-2 F-FPS operands: the
layer-1 xyz / features of synth.kitti_like(8, 16384, seed=1000) with init_params(ARCH_3DSSD, 1, seed=0), computed by the
CPU oracle.  Buckets are the kernel's: 32 consecutive points of the 3-D Morton order of xyz (cubic cells sized by the
widest axis), centre = mean row, radius and largest squared norm per bucket; a bucket is skipped when
    (|w - c| * 0.9999 - rho * 1.0001)^2 * 0.9999 - 8.4e-6 (sq_w + sqmax)  >=  max running distance in the bucket.
Prints phi, the fraction of the 128 buckets a round touches, per range of rounds and on average over the 511 rounds and
8 scenes, and checks that no skipped point would have lowered its running distance.
Usage: python tools/ffps_prune_sim.py"""
import importlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("3dssd_b200")
synth = importlib.import_module("3dssd_b200.synth")
from oracle import layers as olayers  # noqa: E402


def spread10(v):
    v = v.astype(np.uint64) & 0x3ff
    v = (v | (v << 16)) & 0x30000ff
    v = (v | (v << 8)) & 0x300f00f
    v = (v | (v << 4)) & 0x30c30c3
    return (v | (v << 2)) & 0x9249249


def morton_order(p):
    lo = p.min(0)
    ext = (p.max(0) - lo).max()
    q = np.clip(((p - lo) * np.float32(1023.999 / ext if ext > 0 else 0)).astype(np.int64), 0, 1023)
    return np.argsort(spread10(q[:, 0]) | (spread10(q[:, 1]) << 1) | (spread10(q[:, 2]) << 2), kind="stable")


def simulate(F, xyz, m, bs=32):
    n = len(F)
    order = morton_order(xyz)
    nb = n // bs
    bid = np.empty(n, np.int64)
    bid[order] = np.arange(n) // bs
    F64 = F.astype(np.float64)
    Fo = F64[order].reshape(nb, bs, -1)
    c = Fo.mean(1)
    rho = np.sqrt(((Fo - c[:, None]) ** 2).sum(2).max(1)) * 1.0001
    sq = (F64 ** 2).sum(1)
    sqmax = sq[order].reshape(nb, bs).max(1)
    td = np.full(n, 1e38, np.float32)
    old, phi = 0, []
    for _ in range(1, m):
        val = ((sq[old] + sq) - 2.0 * (F64 @ F64[old])).astype(np.float32)
        g = np.maximum(np.sqrt(((c - F64[old]) ** 2).sum(1)) * 0.9999 - rho, 0.0)
        lb = g * g * 0.9999 - 8.4e-6 * (sq[old] + sqmax)
        skip = lb >= td[order].reshape(nb, bs).max(1)
        phi.append(1.0 - skip.mean())
        assert np.all(val[skip[bid]] >= td[skip[bid]])
        td = np.minimum(td, val)
        old = int(np.argmax(td))
    return np.array(phi)


def main():
    arch = pkg.config.ARCH_3DSSD
    params = pkg.params.init_params(arch, 1, seed=0)
    xyz_l, feat_l, _ = olayers.backbone_forward(arch[:1], synth.kitti_like(8, 16384, seed=1000), params)
    xyz, feat = xyz_l[1], feat_l[1]
    phis = np.array([simulate(np.concatenate([xyz[s], feat[s]], 1), xyz[s], 512) for s in range(len(xyz))])
    for a, b in ((1, 16), (16, 64), (64, 128), (128, 256), (256, 384), (384, 512)):
        print("rounds %3d-%3d: phi %.3f" % (a, b - 1, phis[:, a - 1:b - 1].mean()))
    print("per scene:", " ".join("%.3f" % v for v in phis.mean(1)))
    print("mean phi over %d rounds x %d scenes: %.3f" % (phis.shape[1], phis.shape[0], phis.mean()))


if __name__ == "__main__":
    main()
