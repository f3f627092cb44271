"""The pruned D-FPS, pruned F-FPS and culled ball query under changes of a scene's magnitude, without a GPU.

The kernels that skip work (csrc/fps_bucket.cu, csrc/ball_query_grid.cu) argue their exactness with relative error
bounds plus absolute floors, and their Morton buckets and grid cells come from the scene's bounding box.  KITTI-sized
scenes do not show whether those bounds hold far from the origin, at tiny scales or when one stray point stretches the
box.  The maps below move a scene there:

  * scale2(x, k): multiply by 2^k.  While every nonzero squared term stays a normal float and no squared distance nears
    the 1e38 start value of FPS, every operation of the reference (differences, fma chains, sqrt, comparisons with
    radii scaled the same way, F-FPS's sq + sq - 2 dot) is exact-scaled, so every index, list, count and unit must stay
    the same.  The range check fails loudly instead of letting an out-of-range k pass vacuously.
  * dyadic(x) + translate(x, t): on the 2^-4 grid with extents <= 128 and |coordinate| < 2^19 every coordinate, difference
    and squared distance is exact, so a translation by a multiple of 2^-4 changes no distance and no index.
  * shift (float translation by 1e2..1e5 m), stretch (one stray return 1e3..1e6 m away), flat, collinear and tied
    (equal widest extents): no exact relation; the results must equal the restatement of the reference.

Here the CPU models of the kernels (oracle/fps_pruned_model.c, bq_grid_model.c, ffps_prune_model.c) are compared with
the restatement (oracle/ops.py) under every map; tests/test_scene_transforms_gpu.py runs the CUDA kernels on the same
scenes."""
import importlib

import numpy as np
import pytest

from oracle import ops as oracle_ops
from test_bq_grid_model_cpu import _check as bq_model_check
from test_ffps_bucket_cpu import _scene as ffps_scene

synth = importlib.import_module("3dssd_b200.synth")

EXACT_MIN_SQ = 2.0 ** -120     # smallest nonzero squared term after scaling: a normal float (2^-126) with room for sums
EXACT_MAX_ABS = 2.0 ** 60      # largest |coordinate| after scaling: squared distances stay far below FPS's 1e38 start
GRID = 2.0 ** -4               # the dyadic grid
GRID_MAX_ABS = 2.0 ** 19       # |coordinate| < 2^19 on a 2^-4 grid: 23 significant bits, exact in float32
GRID_MAX_EXT = 128.0           # extents <= 2^7: differences < 2^8, squared distances < 2^17 on a 2^-8 grid, exact

LAYER1_SHELLS = ([0.0, 0.2, 0.4], [0.2, 0.4, 0.8], [32, 32, 64])      # 3dssd.yaml layer 1, dilated
PLAIN_SHELLS = ([0.0, 0.0], [1.6, 3.2], [16, 32])                     # plain query, two radii


# ---------------------------------------------------------------------------------------------------------------------
# scene maps
# ---------------------------------------------------------------------------------------------------------------------
def _min_gap(x, values):
    """smallest nonzero |a - b| of two coordinates on one axis of one scene; values: also the smallest nonzero |a|"""
    x = np.asarray(x, np.float64)
    x = x.reshape((-1,) + x.shape[-2:])
    best = np.inf
    for s in range(x.shape[0]):
        for a in range(x.shape[2]):
            v = np.unique(x[s, :, a])
            if v.size > 1:
                best = min(best, np.diff(v).min())
            if values and (v != 0).any():
                best = min(best, np.abs(v[v != 0]).min())
    return best


def scale2_in_range(x, k, also=(), values=False, radii=()):
    """(ok, why): is scaling x (and the clouds `also` that enter the same distances, e.g. queries) by 2^k exact for every
    operation of the kernels and the reference?  values=True for F-FPS rows: products of the values themselves enter
    the norms, and the squared norms of a pair must stay below the 1e38 start value."""
    x = np.asarray(x, np.float32)
    clouds = np.concatenate([x] + [np.asarray(a, np.float32) for a in also], axis=-2)
    gap = _min_gap(clouds, values)
    big = float(np.abs(clouds).max()) if clouds.size else 0.0
    if np.isfinite(gap) and gap * gap * 4.0 ** k < EXACT_MIN_SQ:
        return False, "2^%d: smallest nonzero squared gap %g scales below 2^-120" % (k, gap * gap)
    if big * 2.0 ** k > EXACT_MAX_ABS:
        return False, "2^%d: largest |coordinate| %g scales above 2^60" % (k, big)
    if values:
        sq = float((np.asarray(clouds, np.float64) ** 2).sum(-1).max())
        if 2 * sq * 4.0 ** k > EXACT_MAX_ABS ** 2:
            return False, "2^%d: largest squared row norm %g scales above 2^119" % (k, sq)
    for r in radii:
        if r != 0 and (r * 2.0 ** k) ** 2 < EXACT_MIN_SQ:
            return False, "2^%d: radius %g scales below 2^-60" % (k, r)
    return True, ""


def scale2(x, k, also=(), values=False, radii=()):
    """x * 2^k, exact; fails unless the scaled scene stays in the range where the reference's arithmetic is exact-scaled"""
    ok, why = scale2_in_range(x, k, also, values, radii)
    assert ok, why
    return np.ldexp(np.asarray(x, np.float32), k).astype(np.float32)


def on_grid(x):
    x = np.asarray(x, np.float64)
    return bool((np.round(x / GRID) * GRID == x).all())


def dyadic(x):
    """x rounded to the 2^-4 grid (a KITTI-like scene: extents <= 128)"""
    y = (np.round(np.asarray(x, np.float64) / GRID) * GRID).astype(np.float32)
    ext = np.ptp(y.reshape((-1,) + y.shape[-2:]), axis=-2)
    assert (ext <= GRID_MAX_EXT).all(), ext.max()
    return y


def translate(x, t):
    """x + t exactly: x on the 2^-4 grid with extents <= 128, t a multiple of 2^-4, the result within |.| < 2^19 -- so
    every coordinate, difference and squared distance of the translated scene is exact and equals the original's"""
    t = np.asarray(t, np.float64)
    assert on_grid(x) and on_grid(t), "translate needs x and t on the 2^-4 grid"
    ext = np.ptp(np.asarray(x).reshape((-1,) + x.shape[-2:]), axis=-2)
    assert (ext <= GRID_MAX_EXT).all(), ext.max()
    y = np.asarray(x, np.float64) + t
    assert np.abs(y).max() < GRID_MAX_ABS, np.abs(y).max()
    out = y.astype(np.float32)
    assert (out.astype(np.float64) == y).all()
    return out


def shift(x, t):
    """x + t in float32: coordinates round, no exact relation to the original"""
    return (np.asarray(x, np.float32) + np.asarray(t, np.float32)).astype(np.float32)


STRAY = np.array([0.6, 0.0, 0.8])       # horizontal direction (camera frame: y is down): stretches both widest axes


def stretch(x, far, j=None):
    """one point (index n // 3 of every scene) replaced by a stray return `far` metres out: the bounding box grows by
    `far`, so the Morton grid and the ball-query grid put nearly the whole scene into one or two cells"""
    y = np.array(x, np.float32, copy=True)
    j = y.shape[-2] // 3 if j is None else j
    y[..., j, :3] = (y[..., j, :3].astype(np.float64) + far * STRAY).astype(np.float32)
    return y


def flat(x):
    y = np.array(x, np.float32, copy=True)
    y[..., 1] = np.float32(1.65)        # every point on the ground plane
    return y


def collinear(x):
    """every point on one line through the scene (the scan's x coordinate as the parameter)"""
    t = np.asarray(x, np.float64)[..., :1]
    return (np.array([2.0, 1.65, 35.0]) + t * np.array([1.0, 0.02, 0.7])).astype(np.float32)


def tied(x):
    """x and z extents exactly equal (80 m): the two widest axes a0 / a1 of the grid set-up tie"""
    y = dyadic(x).astype(np.float64)
    y[..., 2] = np.clip(np.round(y[..., 2] * (80.0 / 70.0) / GRID) * GRID, 0.0, 80.0)
    y[..., 0] = np.clip(y[..., 0], -40.0, 40.0)
    y[..., 0, 0], y[..., 0, 2] = -40.0, 0.0
    y[..., 1, 0], y[..., 1, 2] = 40.0, 80.0
    return y.astype(np.float32)


# (id, base scene, map, radius factor).  Exact maps: the outputs must equal the base scene's.  The scale range is what
# the checks allow: the float KITTI scene's smallest gap is 2^-23 (k >= -37), the dyadic scene's 2^-4 (k >= -56); at
# k = -48 .. -56 the squared distances of late FPS rounds fall below the 1e-30 floor of the D-FPS skip rule.
EXACT_MAPS = [("scale-16", "kitti", lambda x: scale2(x, -16), 2.0 ** -16),
              ("scale-7", "kitti", lambda x: scale2(x, -7), 2.0 ** -7),
              ("scale-1", "kitti", lambda x: scale2(x, -1), 0.5),
              ("scale+3", "kitti", lambda x: scale2(x, 3), 8.0),
              ("scale+16", "kitti", lambda x: scale2(x, 16), 2.0 ** 16),
              ("scale-48", "dyadic", lambda x: scale2(x, -48), 2.0 ** -48),
              ("scale-56", "dyadic", lambda x: scale2(x, -56), 2.0 ** -56),
              ("translate-x5e5", "dyadic", lambda x: translate(x, [499968.0, 0.0, 0.0]), 1.0),
              ("translate-diag", "dyadic", lambda x: translate(x, [300000.5, -200000.0625, 400000.3125]), 1.0),
              ("translate-neg", "dyadic", lambda x: translate(x, [-262144.0, 131072.4375, -65536.0]), 1.0)]
FLOAT_MAPS = [("shift-1e2", lambda x: shift(x, [123.456, 0.0, 0.0])),
              ("shift-1e4", lambda x: shift(x, [7071.07, -7071.07, 7071.07])),
              ("shift-1e5", lambda x: shift(x, [1.0e5 + 0.3, 0.0, -7.3e4])),
              ("stretch-1e3", lambda x: stretch(x, 1e3)),
              ("stretch-1e4", lambda x: stretch(x, 1e4)),
              ("stretch-1e6", lambda x: stretch(x, 1e6)),
              ("flat", flat), ("collinear", collinear), ("tied", tied)]
EXACT_IDS = [m[0] for m in EXACT_MAPS]
FLOAT_IDS = [m[0] for m in FLOAT_MAPS]


def exact_map(name):
    return next(m for m in EXACT_MAPS if m[0] == name)


def float_map(name):
    return next(m for m in FLOAT_MAPS if m[0] == name)


def base_scene(kind, b, n, seed):
    """the KITTI-like scene (xyz) and its dyadic rounding"""
    pts = synth.kitti_like(b, n, seed=seed)[..., :3].copy()
    return pts if kind == "kitti" else dyadic(pts)


def apply_map(fn, *clouds):
    """one map applied to several clouds of the same scenes at once (candidates, then queries), so a translation or a
    range check sees every coordinate that enters a distance"""
    sizes = [c.shape[1] for c in clouds]
    out = fn(np.concatenate(clouds, axis=1))
    return np.split(out, np.cumsum(sizes)[:-1], axis=1)


# ---------------------------------------------------------------------------------------------------------------------
# the maps themselves
# ---------------------------------------------------------------------------------------------------------------------
def test_maps_are_what_they_claim():
    pts = base_scene("kitti", 2, 4096, 3)
    d = dyadic(pts)
    assert on_grid(d) and not on_grid(pts)
    for name, base, fn, f in EXACT_MAPS:
        x = d if base == "dyadic" else pts
        y = fn(x)
        assert y.dtype == np.float32 and y.shape == x.shape
        if name.startswith("scale"):
            np.testing.assert_array_equal(np.ldexp(y, -int(np.log2(f))), x)           # invertible: nothing rounded
        else:
            t = (y.astype(np.float64) - x)[:, :1]
            assert (y.astype(np.float64) - x == t).all()                              # one exact offset for every point
            sq = lambda v: ((v[:, :64, None].astype(np.float64) - v[:, None, :64]) ** 2).sum(-1)
            np.testing.assert_array_equal(sq(y), sq(x))
    for name, fn in FLOAT_MAPS:
        y = fn(pts)
        assert y.dtype == np.float32 and y.shape == pts.shape and np.isfinite(y).all()
    e = np.ptp(tied(pts), axis=1)
    assert (e[:, 0] == e[:, 2]).all() and (e[:, 1] < e[:, 0]).all()
    assert np.ptp(stretch(pts, 1e6), axis=1).min(axis=0)[0] > 5e5


@pytest.mark.parametrize("k", [-40, 64])
def test_scale2_refuses_an_inexact_range(k):
    """Out of range the check fails instead of scaling: at 2^-40 the float scene's 2^-23 gaps square to 2^-126, at 2^64
    its coordinates exceed 2^60."""
    pts = base_scene("kitti", 1, 4096, 3)
    assert not scale2_in_range(pts, k)[0]
    with pytest.raises(AssertionError):
        scale2(pts, k)
    feat = ffps_scene("plain", 512, 1)
    assert not scale2_in_range(feat, -70 if k < 0 else 56, values=True)[0]       # 2 |row|^2 ~ 2^14 exceeds 2^120 at 2^56
    with pytest.raises(AssertionError):
        translate(pts, [0.0, 0.0, 0.0])                  # not on the grid
    with pytest.raises(AssertionError):
        translate(dyadic(pts), [2.0 ** 19, 0.0, 0.0])    # leaves |x| < 2^19


# ---------------------------------------------------------------------------------------------------------------------
# pruned D-FPS model
# ---------------------------------------------------------------------------------------------------------------------
FPS_N, FPS_M = 16384, 1024


@pytest.fixture(scope="module")
def fps_base():
    """untransformed scene -> restatement indices, per base kind"""
    out = {}
    for kind in ("kitti", "dyadic"):
        pts = base_scene(kind, 1, FPS_N, 1000)
        out[kind] = (pts, oracle_ops.farthest_point_sample(FPS_M, pts))
    return out


@pytest.mark.parametrize("name", EXACT_IDS)
def test_pruned_fps_model_invariant_under_exact_maps(fps_base, name):
    _, base, fn, _ = exact_map(name)
    pts, exp = fps_base[base]
    np.testing.assert_array_equal(oracle_ops.fps_pruned_model(FPS_M, pts)[0], exp)
    x = fn(pts)
    np.testing.assert_array_equal(oracle_ops.farthest_point_sample(FPS_M, x), exp, err_msg="restatement, " + name)
    for contract in (True, False):
        got, _ = oracle_ops.fps_pruned_model(FPS_M, x, contract=contract)
        np.testing.assert_array_equal(got, exp, err_msg="model, %s, contract %s" % (name, contract))


@pytest.mark.parametrize("name", FLOAT_IDS)
def test_pruned_fps_model_equals_restatement_under_float_maps(fps_base, name):
    x = float_map(name)[1](fps_base["kitti"][0])
    exp = oracle_ops.farthest_point_sample(FPS_M, x)
    for contract in (True, False):
        np.testing.assert_array_equal(oracle_ops.fps_pruned_model(FPS_M, x, contract=contract)[0], exp,
                                      err_msg="%s, contract %s" % (name, contract))


def test_pruned_fps_model_resumes_on_a_translated_scene(fps_base):
    """The resume state (distances + bucket permutation) of a far-off scene, cut where the latency schedule cuts."""
    pts, exp = fps_base["dyadic"]
    x = exact_map("translate-diag")[2](pts)
    out = np.full((1, FPS_M), -7, np.int32)
    temp = np.zeros((1, 2 * FPS_N), np.float32)
    cuts = (0, 1, 348, 635, 860, FPS_M)
    for j0, j1 in zip(cuts[:-1], cuts[1:]):
        oracle_ops.fps_pruned_model(FPS_M, x, rounds=(j0, j1), temp=temp, out=out)
        np.testing.assert_array_equal(out[:, :j1], exp[:, :j1])


# ---------------------------------------------------------------------------------------------------------------------
# culled ball query model
# ---------------------------------------------------------------------------------------------------------------------
BQ_N, BQ_M = 16384, 1024


def _bq_model(shells, dilated, pts, q, f=1.0):
    lows, highs, ks = shells
    idx, cnt, units, _ = oracle_ops.query_ball_point_grid_model([r * f for r in lows], [r * f for r in highs], ks, pts, q,
                                                               dilated)
    return idx, cnt, [sorted(u[1:1 + int(u[0])].tolist()) for u in units]


@pytest.fixture(scope="module")
def bq_base():
    """per base kind: candidates, queries (D-FPS centres plus off-cloud vote-like centres), and the model's outputs"""
    out = {}
    rng = np.random.default_rng(4)
    for kind in ("kitti", "dyadic"):
        pts = base_scene(kind, 1, BQ_N, 1000)
        q = oracle_ops.gather_point(pts, oracle_ops.farthest_point_sample(BQ_M, pts))
        q[:, -128:] += rng.normal(0, 0.5, (1, 128, 3)).astype(np.float32)
        q = dyadic(q) if kind == "dyadic" else q
        out[kind] = (pts, q, {d: _bq_model(LAYER1_SHELLS if d else PLAIN_SHELLS, d, pts, q) for d in (True, False)})
    return out


@pytest.mark.parametrize("name", EXACT_IDS)
def test_grid_model_invariant_under_exact_maps(bq_base, name):
    _, base, fn, f = exact_map(name)
    pts, q, exp = bq_base[base]
    x, y = apply_map(fn, pts, q)
    for dilated in (True, False):
        shells = LAYER1_SHELLS if dilated else PLAIN_SHELLS
        if name.startswith("scale"):
            assert scale2_in_range(pts, int(np.log2(f)), also=(q,), radii=shells[1])[0]
        bq_model_check(x, y, [r * f for r in shells[0]], [r * f for r in shells[1]], shells[2], dilated)
        idx, cnt, units = _bq_model(shells, dilated, x, y, f)
        for s in range(len(shells[2])):
            np.testing.assert_array_equal(cnt[s], exp[dilated][1][s], err_msg="%s shell %d counts" % (name, s))
            np.testing.assert_array_equal(idx[s], exp[dilated][0][s], err_msg="%s shell %d lists" % (name, s))
            assert units[s] == exp[dilated][2][s], "%s shell %d unit list" % (name, s)


@pytest.mark.parametrize("name", FLOAT_IDS)
def test_grid_model_equals_restatement_under_float_maps(bq_base, name):
    pts, q, _ = bq_base["kitti"]
    x, y = apply_map(float_map(name)[1], pts, q)
    for dilated in (True, False):
        bq_model_check(x, y, *(LAYER1_SHELLS if dilated else PLAIN_SHELLS), dilated)


# ---------------------------------------------------------------------------------------------------------------------
# pruned F-FPS model
# ---------------------------------------------------------------------------------------------------------------------
FFPS_N, FFPS_M = 4096, 512


def _ffps_restatement(m, x):
    return oracle_ops.farthest_point_sample_with_distance(m, oracle_ops.calc_square_dist(x[None]))[0]


@pytest.fixture(scope="module")
def ffps_base():
    x = ffps_scene("plain", FFPS_N, 5)
    idx, (bad, _) = oracle_ops.ffps_prune_model(FFPS_M, x)
    assert bad == 0
    np.testing.assert_array_equal(idx, _ffps_restatement(FFPS_M, x))
    return x, idx


@pytest.mark.parametrize("k", [-24, -9, -1, 5, 20])
def test_ffps_model_invariant_under_scale2(ffps_base, k):
    x, exp = ffps_base
    y = scale2(x, k, values=True)
    idx, (bad, _) = oracle_ops.ffps_prune_model(FFPS_M, y)
    assert bad == 0
    np.testing.assert_array_equal(idx, exp)
    np.testing.assert_array_equal(_ffps_restatement(FFPS_M, y), exp)


def test_ffps_model_on_translated_xyz():
    """xyz 1e4 m out (features unchanged): the squared norms reach 3e8, their rounding error dwarfs the feature
    distances.  With its margin the skip rule stays exact; without it, it skips points it must not -- the scene reaches
    the margin.  The count of those points is itself invariant under 2^k scaling."""
    x = ffps_scene("plain", FFPS_N, 5)
    x[:, :3] = shift(x[:, :3], [7071.07, 0.0, 7071.07])
    idx, (bad, _) = oracle_ops.ffps_prune_model(FFPS_M, x)
    assert bad == 0
    np.testing.assert_array_equal(idx, _ffps_restatement(FFPS_M, x))
    idx0, (bad0, _) = oracle_ops.ffps_prune_model(FFPS_M, x, with_margin=False)
    assert bad0 > 0
    for k in (-12, 12):
        y = scale2(x, k, values=True)
        np.testing.assert_array_equal(oracle_ops.ffps_prune_model(FFPS_M, y)[0], idx)
        i1, (b1, _) = oracle_ops.ffps_prune_model(FFPS_M, y, with_margin=False)
        assert b1 == bad0
        np.testing.assert_array_equal(i1, idx0)
