"""The skip rule of the 4-CTA F-FPS with bucket pruning (ffps_bucket_kernel, csrc/fps_bucket.cu), without a GPU.
oracle/ffps_prune_model.c runs the F-FPS with the kernel's fp32 arithmetic and bucket bounds and counts, every round, the
points of skipped buckets whose value would have been below their running distance: there must be none, on the
benchmark's layer-2 operands and on scenes where the bound is tight, and the sampled indices must be the oracle's.
With the rounding margin dropped the same model must find such points.  The plan that picks the kernel is pinned in
tests/test_fps_plan_cpu.py."""
import importlib

import numpy as np
import pytest


def _model(oracle_ops, x, m, with_margin=True):
    """(bad points, indices, fraction of the buckets a round touches)"""
    idx, (bad, touched) = oracle_ops.ffps_prune_model(m, x, with_margin)
    return bad, idx, touched / ((m - 1) * ((x.shape[0] + 31) // 32))


def _scene(kind, n, seed):
    rng = np.random.default_rng(seed)
    xyz = np.stack([rng.uniform(-40, 40, n), rng.uniform(-3, 1, n), 70 * rng.uniform(0, 1, n) ** 2], -1)
    feat = np.maximum(rng.normal(0.0, 0.5, (n, 64)), 0.0)
    if kind == "dups":
        src = rng.integers(0, n, n // 3)
        xyz[n - n // 3:], feat[n - n // 3:] = xyz[src], feat[src]
    elif kind == "quantised":
        feat = np.round(feat * 2) / 2
    elif kind == "zero":
        feat[:] = 0.0
    elif kind == "offset":
        feat = feat + 1e4
    elif kind == "ties":
        xyz = rng.integers(0, 8, (n, 3)).astype(np.float64)
        feat = rng.integers(0, 2, (n, 64)).astype(np.float64)
    return np.concatenate([xyz, feat], 1).astype(np.float32)


@pytest.mark.parametrize("kind", ["plain", "dups", "quantised", "zero", "offset", "ties"])
def test_skip_rule_never_changes_a_distance(oracle_ops, kind):
    x = _scene(kind, 4096, 5)
    bad, idx, _ = _model(oracle_ops, x, 512)
    assert bad == 0
    assert np.array_equal(idx, oracle_ops.farthest_point_sample_features(512, x[None, :, :3], x[None, :, 3:])[0])


def test_skip_rule_on_bench_operands(oracle_ops):
    """Layer-1 output of the benchmark's first two scenes (the layer-2 F-FPS operands): exact, and a round touches
    about a tenth of the buckets (tools/fps_prune_stats.py gives the mean over the eight scenes)."""
    pkg = importlib.import_module("3dssd_b200")
    synth = importlib.import_module("3dssd_b200.synth")
    from oracle import layers as olayers
    arch = pkg.config.ARCH_3DSSD
    xyz_l, feat_l, _ = olayers.backbone_forward(arch[:1], synth.kitti_like(2, 16384, seed=1000),
                                                pkg.params.init_params(arch, 1, seed=0))
    for s in range(2):
        x = np.concatenate([xyz_l[1][s], feat_l[1][s]], 1)
        bad, idx, phi = _model(oracle_ops, x, 512)
        assert bad == 0
        assert phi < 0.2, phi
        assert np.array_equal(idx, oracle_ops.farthest_point_sample_features(512, xyz_l[1][s:s + 1], feat_l[1][s:s + 1])[0])


def test_skip_rule_needs_its_margin(oracle_ops):
    """Features offset by 1e4: the values' rounding error (~ 8e-6 * |x|^2, hundreds) dwarfs the true distances, so
    without E the bound skips points whose computed value is below their running distance."""
    bad, _, _ = _model(oracle_ops, _scene("offset", 4096, 5), 512, with_margin=False)
    assert bad > 0
