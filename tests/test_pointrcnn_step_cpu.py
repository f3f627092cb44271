"""The float64 restatement of PointRCNN's FP layers that tests/test_pointrcnn_step_gpu.py holds the RPN to, checked on
the CPU first: against the CPU oracle's pointnet_fp_module (oracle/layers.py) at small shapes where unknown points sit on
known ones (d = 0) and known points are duplicated (zero-distance ties), plus the latency schedule's cut of the RPN's
D-FPS layers."""
import importlib

import numpy as np
import pytest
import torch

from test_bench_step_gpu import FEATURE_TOL, conv64, gather_rows, rel_err

C = importlib.import_module("3dssd_b200.config")
P = importlib.import_module("3dssd_b200.params")
L = importlib.import_module("3dssd_b200.layers_util")

AMBIGUOUS_REL = 1e-6


# ---- float64 restatements (also used by tests/test_pointrcnn_step_gpu.py) --------------------------------------------

def sqdist64(xyz1, xyz2, idx):
    """float64 squared distances (b, n, k) from the unknown points xyz1 (b, n, 3) to their known points xyz2[idx]."""
    return ((gather_rows(xyz2.double(), idx) - xyz1.double().unsqueeze(2)) ** 2).sum(-1)


def three_nn64(xyz1, xyz2, chunk=1024):
    """three_nn (tf_interpolate_g.cu:24-84) in float64 on the float32 points, one rank further: (d, idx) (b, n, 4) of
    the four nearest known points by squared distance, equal distances in index order (the kernels replace a neighbour
    only on a strictly smaller distance).  Missing neighbours (m < 4) are d = inf, idx = 0, as the kernels leave them."""
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    x1, x2 = xyz1.double(), xyz2.double()
    ds, ids = [], []
    for q0 in range(0, n, chunk):
        d = sum((x1[:, q0:q0 + chunk, k:k + 1] - x2[..., k].unsqueeze(1)) ** 2 for k in range(3))    # (b, q, m)
        v, i = torch.sort(d, dim=-1, stable=True)
        ds.append(v[..., :4])
        ids.append(i[..., :4])
        del d, v, i
    d, idx = torch.cat(ds, 1), torch.cat(ids, 1)
    if m < 4:
        d = torch.cat([d, torch.full((b, n, 4 - m), float("inf"), dtype=d.dtype, device=d.device)], -1)
        idx = torch.cat([idx, torch.zeros((b, n, 4 - m), dtype=idx.dtype, device=idx.device)], -1)
    return d, idx


def nn_ambiguous(xyz2, d, idx):
    """(b, n) bool: unknown points whose three nearest neighbours float32 rounding may order differently than float64
    does -- two consecutive ones of the four nearest at distances within AMBIGUOUS_REL that are distinct known points.
    Copies of one known point are at equal distances in any precision and keep index order, so they are not ambiguous."""
    near = ((d[..., 1:] - d[..., :-1]) <= AMBIGUOUS_REL * d[..., 1:]) & torch.isfinite(d[..., 1:])
    p = gather_rows(xyz2, idx)
    same = (p[..., 1:, :] == p[..., :-1, :]).all(-1)
    return (near & ~same).any(-1)


def fp_layer64(params, scope, nconv, bn, xyz1, xyz2, points1, points2, idx=None):
    """pointnet_fp_module (layers_util.py:192-225) in float64: the three nearest known points (idx (b, n, 3), or
    three_nn64's), weights inv_k / sum(inv), inv_k = 1 / max(d_k, 1e-10) on the float64 squared distances, the
    interpolation, [interpolated | points1] and the convs (conv + BN with the moving statistics + ReLU).  Returns the
    features (b, n, c) float64 and the neighbours used."""
    if idx is None:
        idx = three_nn64(xyz1, xyz2)[1][..., :3]
    dist = torch.clamp_min(sqdist64(xyz1, xyz2, idx), 1e-10)
    if xyz2.shape[1] < 3:                                  # neighbours the kernels never found weigh nothing
        dist = torch.where(torch.arange(3, device=dist.device) < xyz2.shape[1], dist, torch.full_like(dist, float("inf")))
    inv = 1.0 / dist
    w = inv / inv.sum(-1, keepdim=True)
    x = (gather_rows(points2.double(), idx) * w.unsqueeze(-1)).sum(2)
    if points1 is not None:
        x = torch.cat([x, points1.double()], -1)
    for i in range(nconv):
        x = conv64(params, "%s/conv_%d" % (scope, i), x, bn, True)
    return x, idx


# ---- checks against the CPU oracle ----------------------------------------------------------------------------------

def fp_scene(b, n, m, c2, c1, seed):
    """Known points with exact copies (each third one repeats the first, so three copies tie at every distance), unknown
    points on known points (d = 0, also on the copies) and repeated unknown points, on a 1/64 m grid like a scan."""
    rng = np.random.default_rng(seed)
    xyz2 = (np.round(rng.uniform(-8, 8, (b, m, 3)) * 64) / 64).astype(np.float32)
    xyz2[:, 2::3] = xyz2[:, 0:1]
    xyz1 = (np.round(rng.uniform(-8, 8, (b, n, 3)) * 64) / 64).astype(np.float32)
    k = min(n // 2, m)
    xyz1[:, :k] = xyz2[:, :k]
    xyz1[:, k:k + 8] = xyz1[:, k + 8:k + 16]
    p2 = rng.standard_normal((b, m, c2)).astype(np.float32)
    p1 = rng.standard_normal((b, n, c1)).astype(np.float32)
    return xyz1, xyz2, p1, p2


# (scope, n unknown, m known): rpn_fp_layer1 (c2 = 256, c1 = 1) and rpn_fp_layer3 (512, 256) at small sizes
FP_CASES = [("rpn_fp_layer1", 200, 37), ("rpn_fp_layer3", 96, 24), ("rpn_fp_layer1", 50, 3), ("rpn_fp_layer1", 40, 2)]


@pytest.fixture(scope="module")
def rpn_params():
    return P.init_params(C.ARCH_POINTRCNN_RPN, 1, seed=0, aggregation=False)


@pytest.mark.parametrize("case", FP_CASES, ids=lambda c: "%s-n%d-m%d" % c)
def test_three_nn64_matches_the_oracle(oracle_ops, case):
    """Same neighbours as the C oracle's three_nn wherever the order is unambiguous, including the d = 0 neighbours and
    the three-way ties of copies; the oracle's float32 distances within float32 rounding of the float64 ones."""
    _, n, m = case
    xyz1, xyz2, _, _ = fp_scene(2, n, m, 4, 1, seed=n + m)
    edist, eidx = oracle_ops.three_nn(xyz1, xyz2)
    d, idx = three_nn64(torch.from_numpy(xyz1), torch.from_numpy(xyz2))
    amb = nn_ambiguous(torch.from_numpy(xyz2), d, idx).numpy()
    assert amb.mean() <= 0.05
    np.testing.assert_array_equal(idx[..., :3].numpy()[~amb], eidx[~amb])
    k = min(m, 3)
    d3 = d[..., :k].numpy()
    assert np.all(np.abs(edist[..., :k] - d3) <= 1e-6 * d3)
    if m > 3:                                              # the premise: zero distances and ties of copies occur
        assert (d3[..., 0] == 0).sum() >= 2 * min(n // 2, m) and (d3[..., 0] == d3[..., 2]).any()


@pytest.mark.parametrize("case", FP_CASES, ids=lambda c: "%s-n%d-m%d" % c)
def test_fp_layer64_vs_oracle(oracle_ops, rpn_params, case):
    """fp_layer64 on its own float64 neighbours against oracle/layers.py:pointnet_fp_module in float32."""
    from oracle import layers as olayers
    scope, n, m = case
    spec = next(s for s in C.ARCH_POINTRCNN_RPN if s[12] == scope)
    c2 = rpn_params[scope + "/conv_0/weights"].shape[0] - {"rpn_fp_layer1": 1, "rpn_fp_layer3": 256}[scope]
    c1 = rpn_params[scope + "/conv_0/weights"].shape[0] - c2
    xyz1, xyz2, p1, p2 = fp_scene(2, n, m, c2, c1, seed=3 * n + m)
    exp = olayers.pointnet_fp_module(xyz1, xyz2, p1, p2, spec[4], False, None, scope, True, params=rpn_params)
    t = torch.from_numpy
    got, idx = fp_layer64(rpn_params, scope, len(spec[4]), True, t(xyz1), t(xyz2), t(p1), t(p2))
    e = rel_err(exp, got.numpy(), rtol=FEATURE_TOL)
    assert e < FEATURE_TOL, "%s: rel err %g" % (scope, e)
    # and on the oracle's own neighbours, to float32 rounding
    _, eidx = oracle_ops.three_nn(xyz1, xyz2)
    got2, _ = fp_layer64(rpn_params, scope, len(spec[4]), True, t(xyz1), t(xyz2), t(p1), t(p2), idx=t(eidx).long())
    assert rel_err(exp, got2.numpy(), rtol=1e-5, atol_frac=1e-6) < 1e-5


def test_fp_layer64_sees_a_wrong_weight(rpn_params):
    """The restatement is not blind to the neighbours: taking the fourth nearest point instead of the third moves the
    features far past FEATURE_TOL."""
    scope, n, m = FP_CASES[0]
    spec = next(s for s in C.ARCH_POINTRCNN_RPN if s[12] == scope)
    xyz1, xyz2, p1, p2 = (torch.from_numpy(a) for a in fp_scene(1, n, m, 256, 1, seed=1))
    d, idx = three_nn64(xyz1, xyz2)
    y, _ = fp_layer64(rpn_params, scope, len(spec[4]), True, xyz1, xyz2, p1, p2, idx=idx[..., :3])
    y2, _ = fp_layer64(rpn_params, scope, len(spec[4]), True, xyz1, xyz2, p1, p2, idx=idx[..., [0, 1, 3]])
    assert (y - y2).abs().max() > 1e2 * FEATURE_TOL * y.abs().max()


# ---- the latency schedule of the RPN's D-FPS layers -----------------------------------------------------------------

def test_latency_parts_of_the_rpn_layers():
    """latency_mode cuts every RPN SA layer's D-FPS into resumable parts of whole 128-row tiles: four parts in layers 1
    and 2, two in layer 3; layer 4's 64 samples stay one launch.  So resumed D-FPS launches run at all three sizes."""
    parts = [L._part_bounds(spec[8][0], (0.34, 0.28, 0.22, 0.16)) for spec in C.ARCH_POINTRCNN_RPN[:4]]
    assert parts == [[(0, 1408), (1408, 2560), (2560, 3456), (3456, 4096)],
                     [(0, 384), (384, 640), (640, 896), (896, 1024)],
                     [(0, 128), (128, 256)],
                     [(0, 64)]]
