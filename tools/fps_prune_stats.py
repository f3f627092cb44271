"""Touched-bucket fraction of the two pruned FPS kernels (csrc/fps_bucket.cu) on the benchmark's operands, counted on the
CPU by their lane-by-lane C models in oracle/ (fps_pruned_model.c, ffps_prune_model.c):
  * layer 1, fps3_bucket_kernel: D-FPS of 4096 from the 16384-point xyz of synth.kitti_like(8, 16384, seed=1000),
    512 buckets of 32 points;
  * layer 2, ffps_bucket_kernel: F-FPS of 512 from the layer-1 xyz / features of those scenes with
    init_params(ARCH_3DSSD, 1, seed=0) (computed by the CPU oracle), 128 buckets of 32 points.
Prints, per kernel and scene, the fraction of the buckets a round touches (bucket updates over rounds x buckets) and
its mean over the scenes, and checks that the sampled indices are the oracle's.  Usage: python tools/fps_prune_stats.py"""
import importlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("3dssd_b200")
synth = importlib.import_module("3dssd_b200.synth")
from oracle import layers as olayers  # noqa: E402
from oracle import ops  # noqa: E402


def layer1(xyz, m=4096):
    phi = []
    for s in range(len(xyz)):
        x = np.ascontiguousarray(xyz[s:s + 1], np.float32)
        idx, (updates, rounds, _) = ops.fps_pruned_model(m, x)
        assert np.array_equal(idx, ops.farthest_point_sample(m, x)), s
        phi.append(updates / (rounds * 512))
    return phi


def layer2(xyz, feat, m=512):
    phi = []
    for s in range(len(xyz)):
        idx, (bad, touched) = ops.ffps_prune_model(m, np.concatenate([xyz[s], feat[s]], 1))
        assert bad == 0, s
        assert np.array_equal(idx, ops.farthest_point_sample_features(m, xyz[s:s + 1], feat[s:s + 1])[0]), s
        phi.append(touched / ((m - 1) * 128))
    return phi


def _report(name, phi):
    print("%s: per scene %s; mean %.4f" % (name, " ".join("%.4f" % v for v in phi), np.mean(phi)))


def main():
    pts = synth.kitti_like(8, 16384, seed=1000)
    _report("layer 1 D-FPS (fps3_bucket_kernel, 4095 rounds, 512 buckets)", layer1(pts[..., :3]))
    arch = pkg.config.ARCH_3DSSD
    xyz_l, feat_l, _ = olayers.backbone_forward(arch[:1], pts, pkg.params.init_params(arch, 1, seed=0))
    _report("layer 2 F-FPS (ffps_bucket_kernel, 511 rounds, 128 buckets)", layer2(xyz_l[1], feat_l[1]))


if __name__ == "__main__":
    main()
