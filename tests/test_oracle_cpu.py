"""CPU-side tests (-m "not gpu"): the oracle against the committed golden vectors of the reference's own
kernels (tests/golden/*.npz, see make_golden.py), against independent numpy restatements, and the
reference's documented quirks (FPS tie-break, ball-query back-fill)."""
import glob
import os

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


# ---- independent (slow, obviously-correct) numpy restatements -------------------------------------------
def np_sqdist_bq(q, p):
    """t = dy*dy ; t = fma(dx,dx,t) ; t = fma(dz,dz,t) evaluated exactly: float64 products of float32 values
    are exact, and one rounding to float32 per step reproduces fma's single rounding."""
    d = q[None, :].astype(np.float32) - p.astype(np.float32)   # [n,3] float32 differences (rounded, as on GPU)
    dx, dy, dz = (d[:, i].astype(np.float64) for i in range(3))
    t = (dy * dy).astype(np.float32)
    t = (dx * dx + t.astype(np.float64)).astype(np.float32)
    t = (dz * dz + t.astype(np.float64)).astype(np.float32)
    return t


def np_ball_query(radius, nsample, xyz1, xyz2, min_radius=None):
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    idx = np.zeros((b, m, nsample), np.int32)
    cnt = np.zeros((b, m), np.int32)
    for bi in range(b):
        for j in range(m):
            t = np_sqdist_bq(xyz2[bi, j], xyz1[bi])
            d = np.sqrt(t).astype(np.float32)
            if min_radius is None:
                hit = np.maximum(d, np.float32(1e-20)) < np.float32(radius)
            else:
                hit = (d == 0) | ((d >= np.float32(min_radius)) & (d < np.float32(radius)))
            ks = np.nonzero(hit)[0][:nsample]
            cnt[bi, j] = len(ks)
            if len(ks):
                idx[bi, j, :] = ks[0]
                idx[bi, j, :len(ks)] = ks
    return idx, cnt


def np_fps(npoint, pts):
    """Reference order: value desc, k mod 1024 asc, k asc."""
    b, n, c = pts.shape
    out = np.zeros((b, npoint), np.int32)
    k = np.arange(n)
    order_key = (k % 1024).astype(np.int64) * (1 << 32) + k
    for bi in range(b):
        td = np.full(n, np.float32(1e38))
        old = 0
        for j in range(1, npoint):
            diff = pts[bi] - pts[bi, old][None]
            d = np.zeros(n, np.float32)
            for l in range(c):
                d = (diff[:, l].astype(np.float64) ** 2 + d.astype(np.float64)).astype(np.float32)
            td = np.minimum(d, td)
            mx = td.max()
            cand = np.nonzero(td == mx)[0]
            old = int(cand[np.argmin(order_key[cand])])
            out[bi, j] = old
    return out


# ---- tests -------------------------------------------------------------------------------------------------
def test_fps_matches_numpy_restatement(oracle_ops):
    rng = np.random.default_rng(0)
    pts = rng.uniform(-1, 1, (2, 300, 3)).astype(np.float32)
    np.testing.assert_array_equal(oracle_ops.farthest_point_sample(64, pts), np_fps(64, pts))
    pts = rng.uniform(-1, 1, (1, 2500, 3)).astype(np.float32)     # n > 1024: several points per thread class
    np.testing.assert_array_equal(oracle_ops.farthest_point_sample(40, pts), np_fps(40, pts))
    feats = rng.standard_normal((2, 200, 7)).astype(np.float32)   # generic c
    np.testing.assert_array_equal(oracle_ops.farthest_point_sample(50, feats), np_fps(50, feats))


def test_fps_tie_break_is_thread_class_then_index(oracle_ops):
    """SURVEY.md appendix worked example: among equal maxima the winner has the lowest k mod 1024, then the
    lowest k -- k=1025 beats k=2."""
    n = 4096
    pts = np.zeros((1, n, 3), np.float32)
    pts[0, 2] = [3.0, 0, 0]
    pts[0, 1025] = [-3.0, 0, 0]                                   # same distance from point 0 as k=2
    out = oracle_ops.farthest_point_sample(3, pts)
    assert out[0].tolist() == [0, 1025, 2]
    # exact duplicates everywhere: after every point is at distance 0 the reference keeps returning index 0
    pts = np.tile(np.array([[1.0, 2.0, 3.0]], np.float32), (1, 100, 1))
    assert oracle_ops.farthest_point_sample(5, pts)[0].tolist() == [0, 0, 0, 0, 0]


def test_fps_with_distance_equals_fps_on_same_matrix(oracle_ops):
    rng = np.random.default_rng(1)
    f = rng.standard_normal((2, 180, 5)).astype(np.float32)
    dist = oracle_ops.calc_square_dist(f)
    idx = oracle_ops.farthest_point_sample_with_distance(30, dist)
    # numpy restatement of the with-distance loop
    for bi in range(2):
        td = np.full(180, np.float32(1e38)); old = 0; exp = [0]
        for _ in range(29):
            td = np.minimum(dist[bi, old], td)
            mx = td.max(); cand = np.nonzero(td == mx)[0]
            old = int(cand[np.argmin((cand % 1024) * (1 << 20) + cand)]); exp.append(old)
        assert idx[bi].tolist() == exp


def test_calc_square_dist_close_to_float64(oracle_ops):
    rng = np.random.default_rng(2)
    f = rng.standard_normal((1, 96, 67)).astype(np.float32)
    got = oracle_ops.calc_square_dist(f)
    f64 = f.astype(np.float64)
    exp = ((f64[0, :, None, :] - f64[0, None, :, :]) ** 2).sum(-1)
    np.testing.assert_allclose(got[0], exp, rtol=0, atol=2e-4)
    assert np.array_equal(got[0], got[0].T)                        # the pinned order is symmetric


@pytest.mark.parametrize("dilated", [False, True])
def test_ball_query_matches_numpy_restatement(oracle_ops, dilated):
    rng = np.random.default_rng(3)
    xyz1 = rng.uniform(0, 1, (2, 400, 3)).astype(np.float32)
    xyz2 = np.ascontiguousarray(xyz1[:, :50])
    if dilated:
        idx, cnt = oracle_ops.query_ball_point_dilated(0.15, 0.3, 16, xyz1, xyz2)
        eidx, ecnt = np_ball_query(0.3, 16, xyz1, xyz2, min_radius=0.15)
    else:
        idx, cnt = oracle_ops.query_ball_point(0.2, 16, xyz1, xyz2)
        eidx, ecnt = np_ball_query(0.2, 16, xyz1, xyz2)
    np.testing.assert_array_equal(cnt, ecnt)
    np.testing.assert_array_equal(idx, eidx)
    assert (cnt >= 1).all()                                        # queries are a subset of xyz1: self hit


def test_ball_query_backfill_and_empty_rows(oracle_ops):
    xyz1 = np.array([[[0, 0, 0], [0.05, 0, 0], [5, 5, 5], [0.08, 0, 0]]], np.float32)
    xyz2 = np.array([[[0, 0, 0], [100, 100, 100]]], np.float32)
    idx, cnt = oracle_ops.query_ball_point(0.1, 5, xyz1, xyz2)
    assert cnt.tolist() == [[3, 0]]
    assert idx[0, 0].tolist() == [0, 1, 3, 0, 0]                   # first hit back-fills (tf_grouping_g.cu:245-248)
    assert idx[0, 1].tolist() == [0, 0, 0, 0, 0]                   # empty ball: zeros (reference: uninitialised)
    # dilated: the d == 0 self-hit is always taken, even when min_radius > 0
    idx, cnt = oracle_ops.query_ball_point_dilated(0.06, 0.1, 4, xyz1, xyz2)
    assert cnt.tolist() == [[2, 0]] and idx[0, 0].tolist() == [0, 3, 0, 0]


def test_gather_group_interpolate(oracle_ops):
    rng = np.random.default_rng(4)
    pts = rng.standard_normal((2, 50, 6)).astype(np.float32)
    idx = rng.integers(0, 50, (2, 20)).astype(np.int32)
    np.testing.assert_array_equal(oracle_ops.gather_point(pts, idx), np.take_along_axis(pts, idx[..., None].astype(np.int64), 1))
    gidx = rng.integers(-1, 50, (2, 7, 4)).astype(np.int32)
    g = oracle_ops.group_point(pts, gidx)
    for bi in range(2):
        for j in range(7):
            for s in range(4):
                exp = np.zeros(6, np.float32) if gidx[bi, j, s] == -1 else pts[bi, gidx[bi, j, s]]
                np.testing.assert_array_equal(g[bi, j, s], exp)
    # three_nn / three_interpolate
    xyz1 = rng.uniform(0, 1, (2, 30, 3)).astype(np.float32)
    xyz2 = rng.uniform(0, 1, (2, 11, 3)).astype(np.float32)
    dist, nidx = oracle_ops.three_nn(xyz1, xyz2)
    for bi in range(2):
        for i in range(30):
            t = np_sqdist_bq(xyz1[bi, i], xyz2[bi])
            order = np.argsort(t, kind="stable")[:3]
            assert nidx[bi, i].tolist() == order.tolist()
            np.testing.assert_array_equal(dist[bi, i], t[order])
    w = rng.uniform(0, 1, (2, 30, 3)).astype(np.float32)
    out = oracle_ops.three_interpolate(pts[:, :11].copy(), nidx, w)
    exp = np.einsum("bnk,bnkc->bnc", w.astype(np.float64), pts[:, :11][np.arange(2)[:, None, None], nidx].astype(np.float64))
    np.testing.assert_allclose(out, exp, rtol=1e-5, atol=1e-6)
    # fewer than three known points: the reference's 1e40 sentinel becomes +inf, index 0
    d2, i2 = oracle_ops.three_nn(xyz1[:, :2].copy(), xyz2[:, :2].copy())
    assert np.isinf(d2[..., 2]).all() and (i2[..., 2] == 0).all()


def test_linear_bn_relu_oracle(oracle_ops):
    rng = np.random.default_rng(5)
    x = rng.standard_normal((3, 5, 9)).astype(np.float32)
    w = rng.standard_normal((9, 4)).astype(np.float32)
    b = rng.standard_normal(4).astype(np.float32)
    bn = tuple(rng.uniform(0.5, 1.5, 4).astype(np.float32) for _ in range(4))
    y = oracle_ops.linear_bn_relu(x, w, b, bn, relu=True)
    g, be, mu, var = (t.astype(np.float64) for t in bn)
    exp = np.maximum(((x.astype(np.float64) @ w + b) - mu) * g / np.sqrt(var + 1e-3) + be, 0)
    np.testing.assert_allclose(y, exp, rtol=1e-6, atol=1e-6)


def _golden_files():
    return sorted(p for p in glob.glob(os.path.join(GOLDEN, "*.npz")) if "op" in np.load(p).files)


@pytest.mark.parametrize("path", _golden_files() or [None])
def test_oracle_against_reference_golden_vectors(oracle_ops, path):
    """Pins the oracle: outputs of the REFERENCE's own CUDA kernels (oracle/_ref, compiled unmodified from
    the reference sources by tests/golden/make_golden.py and run on a GPU) must be reproduced bit-for-bit."""
    if path is None:
        pytest.skip("no golden vectors committed yet (parity unpinned)")
    z = np.load(path)
    op = str(z["op"])
    if op == "farthest_point_sample":
        np.testing.assert_array_equal(oracle_ops.farthest_point_sample(int(z["npoint"]), z["inp"]), z["out"])
    elif op == "farthest_point_sample_with_distance":
        np.testing.assert_array_equal(oracle_ops.farthest_point_sample_with_distance(int(z["npoint"]), z["dist"]), z["out"])
    elif op == "query_ball_point":
        idx, cnt = oracle_ops.query_ball_point(float(z["radius"]), int(z["nsample"]), z["xyz1"], z["xyz2"])
        np.testing.assert_array_equal(cnt, z["cnt"])
        np.testing.assert_array_equal(idx, z["idx"] * (z["cnt"] > 0)[..., None])
    elif op == "query_ball_point_dilated":
        idx, cnt = oracle_ops.query_ball_point_dilated(float(z["min_radius"]), float(z["max_radius"]), int(z["nsample"]),
                                                       z["xyz1"], z["xyz2"])
        np.testing.assert_array_equal(cnt, z["cnt"])
        np.testing.assert_array_equal(idx, z["idx"] * (z["cnt"] > 0)[..., None])
    elif op == "gather_point":
        np.testing.assert_array_equal(oracle_ops.gather_point(z["inp"], z["idx"]), z["out"])
    elif op == "group_point":
        np.testing.assert_array_equal(oracle_ops.group_point(z["points"], z["idx"]), z["out"])
    elif op == "three_nn":
        dist, idx = oracle_ops.three_nn(z["xyz1"], z["xyz2"])
        np.testing.assert_array_equal(idx, z["idx"])
        np.testing.assert_array_equal(dist, z["dist"])
    elif op == "three_interpolate":
        np.testing.assert_array_equal(oracle_ops.three_interpolate(z["points"], z["idx"], z["weight"]), z["out"])
    else:
        raise AssertionError("unknown golden op " + op)


def test_oracle_bev_nms_hand_case():
    """Greedy NMS restatement: ties go to the lower index, identical boxes suppress each other, far boxes survive."""
    from oracle import head
    b = np.array([[[0, 0, 0, 2, 1, 2, 0], [0.1, 0, 0.1, 2, 1, 2, 0], [10, 0, 10, 2, 1, 2, 0.3], [0, 0, 0, 2, 1, 2, 0]]], np.float32)
    s = np.array([[0.9, 0.8, 0.7, 0.9]], np.float32)
    blk, cnt = head.bev_nms(b, s, 0.1, 100)
    assert cnt.tolist() == [2]
    np.testing.assert_array_equal(blk[0, 0, :7], b[0, 0])
    np.testing.assert_array_equal(blk[0, 1, :7], b[0, 2])
    assert (blk[0, 2:] == 0).all()


def test_matrix_free_ffps_restatement_equals_matrix_route(oracle_ops):
    """The on-the-fly evaluation the CUDA kernel performs (oracle.ops.farthest_point_sample_features, numpy) picks the same
    indices as the reference's two-op route on the CPU oracle: calc_square_dist + farthest_point_sample_with_distance."""
    rng = np.random.default_rng(8)
    xyz = rng.uniform(-3, 3, (2, 90, 3)).astype(np.float32)
    feats = np.maximum(rng.standard_normal((2, 90, 13)), 0).astype(np.float32)
    feats[:, 40] = feats[:, 7]; xyz[:, 40] = xyz[:, 7]                     # an exact duplicate: ties
    cat = np.concatenate([xyz, feats], -1)
    exp = oracle_ops.farthest_point_sample_with_distance(30, oracle_ops.calc_square_dist(cat))
    got = oracle_ops.farthest_point_sample_features(30, xyz, feats)
    np.testing.assert_array_equal(got, exp)
    q = (rng.integers(0, 3, (1, 70, 5)) * 0.5).astype(np.float32)        # quantised: many equal distances
    np.testing.assert_array_equal(oracle_ops.farthest_point_sample_features(25, q),
                                  oracle_ops.farthest_point_sample_with_distance(25, oracle_ops.calc_square_dist(q)))


def test_oracle_on_real_lidar_scene(oracle_ops):
    """Domain invariants of the CPU oracle on the committed real scan (tests/golden/realscan_16384.npz): D-FPS picks
    4096 distinct points starting at index 0 with non-increasing pick distances; every dilated-shell neighbour list is
    ascending up to its count, back-filled with the first hit, and its members lie inside the shell."""
    pts = np.load(os.path.join(GOLDEN, "realscan_16384.npz"))["points"][None, :, :3].astype(np.float32)
    idx = oracle_ops.farthest_point_sample(4096, pts)[0]
    assert idx[0] == 0 and len(set(idx.tolist())) == 4096
    sel = pts[0, idx].astype(np.float64)
    # distance of pick j to the picks before it is non-increasing in j (the defining property of FPS), checked on a prefix
    mind = [np.min(((sel[:j] - sel[j]) ** 2).sum(-1)) for j in range(1, 400)]
    assert all(mind[j] <= mind[j - 1] * (1 + 1e-5) for j in range(1, len(mind)))
    q = np.ascontiguousarray(pts[:, idx[:512]])
    nbr, cnt = oracle_ops.query_ball_point_dilated(0.4, 0.8, 64, pts, q)
    assert cnt.min() >= 1 and cnt.max() <= 64
    d = np.sqrt(((pts[0, nbr[0]].astype(np.float64) - q[0][:, None, :]) ** 2).sum(-1))
    for i in range(512):
        c = cnt[0, i]
        row = nbr[0, i]
        assert (np.diff(row[:c]) > 0).all() and (row[c:] == row[0]).all()
        ok = (d[i, :c] == 0) | ((d[i, :c] >= 0.4 - 1e-5) & (d[i, :c] < 0.8 + 1e-5))
        assert ok.all()


def test_oracle_training_mode_batchnorm_properties(oracle_ops):
    """The float64 restatement of training-mode BatchNorm (tf_util.py:424-444): with gamma = 1, beta = 0 every conv
    output before the ReLU has zero batch mean / unit batch variance, decay = 0 makes the moving statistics equal the
    batch statistics, and inference on the updated parameters reproduces the training output (same statistics)."""
    from oracle import layers as olayers
    rng = np.random.default_rng(0)
    x = rng.standard_normal((2, 50, 8, 6)).astype(np.float32)
    prm = {"s/weights": rng.standard_normal((6, 5)).astype(np.float32), "s/biases": rng.standard_normal(5).astype(np.float32),
           "s/bn/gamma": np.ones(5, np.float32), "s/bn/beta": np.zeros(5, np.float32),
           "s/bn/moving_mean": rng.standard_normal(5).astype(np.float32), "s/bn/moving_variance": np.ones(5, np.float32)}
    upd = {}
    y = olayers._conv(prm, "s", x, bn=True, relu=False, train=(0.0, upd))
    flat = y.reshape(-1, 5).astype(np.float64)
    assert np.abs(flat.mean(0)).max() < 1e-5 and np.abs(flat.var(0) - upd["s"]["batch_variance"] / (upd["s"]["batch_variance"] + 1e-3)).max() < 1e-4
    np.testing.assert_array_equal(upd["s"]["moving_mean"], upd["s"]["batch_mean"])
    prm2 = dict(prm, **{"s/bn/moving_mean": upd["s"]["moving_mean"], "s/bn/moving_variance": upd["s"]["moving_variance"]})
    y_inf = olayers._conv(prm2, "s", x, bn=True, relu=False)
    assert np.abs(y_inf - y).max() < 1e-4
    upd9 = {}
    olayers._conv(prm, "s", x, bn=True, relu=True, train=(0.9, upd9))
    np.testing.assert_allclose(upd9["s"]["moving_mean"], prm["s/bn/moving_mean"] * 0.9 + upd["s"]["batch_mean"] * 0.1, rtol=1e-5, atol=1e-6)
