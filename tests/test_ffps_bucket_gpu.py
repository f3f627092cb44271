"""The 4-CTA F-FPS with bucket pruning (ffps_bucket_kernel, csrc/fps.cu), which a capped cluster request selects for
full-range calls of 2048 < n <= 4096 points with <= 68 channels: its indices must equal the 8-CTA kernel's and the CPU
oracle's bit for bit -- on the benchmark's own layer-2 operands and on scenes where the skip bound is tight (duplicated
points, quantised, all-zero or 1e4-offset features, exact ties), at b = 1 and 8, on strided inputs with placed output."""
import importlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _oracle(oracle_ops, m, xyz, feat):
    return oracle_ops.farthest_point_sample_features(m, np.ascontiguousarray(xyz), np.ascontiguousarray(feat))


def _scene(kind, b, n, seed):
    rng = np.random.default_rng(seed)
    xyz = np.stack([rng.uniform(-40, 40, (b, n)), rng.uniform(-3, 1, (b, n)), 70 * rng.uniform(0, 1, (b, n)) ** 2],
                   -1).astype(np.float32)
    feat = np.maximum(rng.normal(0.0, 0.5, (b, n, 64)), 0.0).astype(np.float32)
    if kind == "dups":            # a third of the points repeat others exactly (coordinates and features)
        src = rng.integers(0, n, (b, n // 3))
        for s in range(b):
            xyz[s, n - n // 3:] = xyz[s, src[s]]
            feat[s, n - n // 3:] = feat[s, src[s]]
    elif kind == "quantised":     # few distinct feature values: many equal distances
        feat = np.round(feat * 2) / 2
    elif kind == "zero":
        feat[:] = 0.0
    elif kind == "offset":        # large norms: the rounding margin of the skip bound dominates small distances
        feat = feat + np.float32(1e4)
    elif kind == "ties":          # integer lattice in xyz, integer features: exact, massively tied distances
        xyz = rng.integers(0, 8, (b, n, 3)).astype(np.float32)
        feat = rng.integers(0, 2, (b, n, 64)).astype(np.float32)
    return xyz, feat


@pytest.mark.parametrize("kind,b,n,m", [("plain", 8, 4096, 512), ("plain", 1, 3000, 700), ("dups", 2, 4096, 512),
                                        ("quantised", 2, 4096, 512), ("zero", 1, 4096, 300), ("offset", 2, 4096, 512),
                                        ("ties", 2, 4096, 512), ("plain", 1, 2049, 2049)])
def test_ffps_bucket_matches_cluster_kernel_and_oracle(pkg, oracle_ops, cuda, kind, b, n, m):
    xyz, feat = _scene(kind, b, n, 7 + n)
    tx, tf = torch.from_numpy(xyz).to(cuda), torch.from_numpy(feat).to(cuda)
    got = pkg.tf_ops.farthest_point_sample_features(m, tx, tf, cluster=-4).cpu().numpy()
    eight = pkg.tf_ops.farthest_point_sample_features(m, tx, tf).cpu().numpy()
    assert np.array_equal(got, eight)
    assert np.array_equal(got, _oracle(oracle_ops, m, xyz, feat))


def test_ffps_bucket_on_bench_operands(pkg, oracle_ops, cuda):
    """The benchmark's layer-2 F-FPS operands: layer 1 of the 3DSSD table on its eight scenes (oracle-computed)."""
    synth = importlib.import_module("3dssd_b200.synth")
    from oracle import layers as olayers
    arch = pkg.config.ARCH_3DSSD
    params = pkg.params.init_params(arch, 1, seed=0)
    xyz_l, feat_l, _ = olayers.backbone_forward(arch[:1], synth.kitti_like(8, 16384, seed=1000), params)
    xyz, feat = xyz_l[1], feat_l[1]
    tx, tf = torch.from_numpy(xyz).to(cuda), torch.from_numpy(feat).to(cuda)
    for cl in (-4, -2, -1):
        got = pkg.tf_ops.farthest_point_sample_features(512, tx, tf, cluster=cl).cpu().numpy()
        assert np.array_equal(got, pkg.tf_ops.farthest_point_sample_features(512, tx, tf).cpu().numpy()), cl
    assert np.array_equal(got, _oracle(oracle_ops, 512, xyz, feat))


def test_ffps_bucket_strided_and_placed(pkg, oracle_ops, cuda):
    """[:, a:a+n] slices of wider xyz / feature tensors (own scene strides), output into columns of a wider buffer with
    an index offset."""
    xyz, feat = _scene("plain", 3, 4096, 11)
    big = torch.zeros((3, 4200, 3), device=cuda)
    wide = torch.zeros((3, 4300, 64), device=cuda)
    big[:, 50:50 + 4096] = torch.from_numpy(xyz).to(cuda)
    wide[:, 100:100 + 4096] = torch.from_numpy(feat).to(cuda)
    buf = torch.full((3, 1100), -7, dtype=torch.int32, device=cuda)
    pkg.tf_ops.farthest_point_sample_features(512, big[:, 50:50 + 4096], wide[:, 100:100 + 4096], out=(buf, 300),
                                              idx_offset=1000, cluster=-4)
    got = buf.cpu().numpy()
    assert np.array_equal(got[:, 300:812], _oracle(oracle_ops, 512, xyz, feat) + 1000)
    assert (got[:, :300] == -7).all() and (got[:, 812:] == -7).all()


def test_ffps_cluster_request_keeps_other_routes(pkg, oracle_ops, cuda):
    """Partial ranges and scenes the 8-CTA kernel does not need are unchanged by a cluster request."""
    xyz, feat = _scene("plain", 2, 4096, 3)
    tx, tf = torch.from_numpy(xyz).to(cuda), torch.from_numpy(feat).to(cuda)
    buf = torch.zeros((2, 512), dtype=torch.int32, device=cuda)
    temp = torch.empty((2, 4096), device=cuda)
    for j0, j1 in ((0, 200), (200, 512)):
        pkg.tf_ops.farthest_point_sample_features(512, tx, tf, out=(buf, 0), rounds=(j0, j1), temp=temp, cluster=-4)
    assert np.array_equal(buf.cpu().numpy(), _oracle(oracle_ops, 512, xyz, feat))
    small = pkg.tf_ops.farthest_point_sample_features(256, tx[:, :2048], tf[:, :2048], cluster=-4).cpu().numpy()
    assert np.array_equal(small, _oracle(oracle_ops, 256, xyz[:, :2048], feat[:, :2048]))
