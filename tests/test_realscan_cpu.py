"""Eight scenes of the reference's real LiDAR scan in the loader's [16384, 4] layout, and the CPU models of the pruned
D-FPS, the culled ball query and the pruned F-FPS on them, without a GPU.

tests/golden/realscan_full.npz holds all 123 398 points of the reference's mayavi/kitti_sample_scan.txt (velodyne frame,
made by tests/golden/make_realscan.py as delta-coded millimetres with a seeded intensity code; its decode_full() restores
the float32 points bit for bit).  realscan_scenes() maps them to the rect camera
frame (x_r = -y_v, y_r = -z_v, z_r = x_v), takes eight regions of the scan and fills each to 16 384 points the way the
reference's loader does (kitti_dataloader.py:137-147): without replacement when a region has at least 16 384 points,
otherwise every point once followed by a with-replacement draw of the rest.  So a short region enters the network with
exact duplicates, and where it has fewer distinct points than a layer samples the later FPS rounds all run at
min-distance 0: only the tie rule and the pruned kernels' skip rules decide which point is picked.

  S0  the detection-range crop (|x| < 40, -5 < y < 3, 0 < z < 70, |x| < z)        31 975 points
  S1  the crop within 10 m (z < 10): dense, 616 pads                               15 768
  S2  the crop at 20-70 m                                                           7 203
  S3  the crop at 30-70 m: fewer distinct points than layer 1's 4096 samples       1 505
  S4  the crop's narrow wedge |x| < 0.25 z                                          9 559
  S5  S0 rotated about the vertical axis by 0.3 rad
  S6  the rear half mirrored into the field of view (z -> -z), then cropped       28 104
  S7  the crop at z >= 50 m: fewer distinct points than layer 2's 512 samples        343

tests/test_realscan_step_gpu.py runs the benchmarked step and its routes on the same eight scenes."""
import functools
import importlib
import importlib.util
import os

import numpy as np
import pytest

from oracle import ops as oracle_ops
from test_bq_grid_model_cpu import _check as bq_model_check
from test_scene_transforms_cpu import LAYER1_SHELLS, PLAIN_SHELLS

HERE = os.path.dirname(os.path.abspath(__file__))
FULL = os.path.join(HERE, "golden", "realscan_full.npz")
SUBSAMPLE = os.path.join(HERE, "golden", "realscan_16384.npz")

NPOINTS = 16384                 # cfg.MODEL.POINTS_NUM_FOR_TRAINING: the loader's scene size
L1_SAMPLES = 4096               # layer 1's D-FPS
L2_SAMPLES = 512                # layer 2's F-FPS and D-FPS
ROTATION = 0.3                  # S5's angle about the vertical axis, radians (not a dyadic fraction of pi)
SCENE_SEED = 2024

# (region points, distinct xyz rows) of every scene before the choice; S5 is S0's choice rotated
SOURCE_COUNTS = {"S0": (31975, 31974), "S1": (15768, 15767), "S2": (7203, 7203), "S3": (1505, 1505),
                 "S4": (9559, 9558), "S6": (28104, 28104), "S7": (343, 343)}
NAMES = ["S0", "S1", "S2", "S3", "S4", "S5", "S6", "S7"]


@functools.lru_cache(maxsize=None)
def _make_realscan():
    spec = importlib.util.spec_from_file_location("make_realscan", os.path.join(HERE, "golden", "make_realscan.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def full_scan():
    """[123398, 4] float32: the scan in the velodyne frame with its intensity"""
    z = np.load(FULL)
    return _make_realscan().decode_full(z["mm_delta"], z["neg_zero"], z["intensity_code"])


def camera_frame(v):
    """velodyne (x forward, y left, z up) -> rect camera (x right, y down, z forward), intensity kept"""
    return np.ascontiguousarray(np.stack([-v[:, 1], -v[:, 2], v[:, 0], v[:, 3]], axis=1), dtype=np.float32)


def in_range(r):
    """the detection range of make_realscan.py and its 90-degree field of view"""
    return ((np.abs(r[:, 0]) < 40) & (r[:, 1] > -5) & (r[:, 1] < 3) & (r[:, 2] > 0) & (r[:, 2] < 70)
            & (np.abs(r[:, 0]) < r[:, 2]))


@functools.lru_cache(maxsize=None)
def scene_sources():
    """name -> [n, 4] camera-frame points of each region, in the scan's order (S5 has none: it is S0's choice rotated)"""
    r = camera_frame(full_scan())
    crop = r[in_range(r)]
    z = crop[:, 2]
    rear = r.copy()
    rear[:, 2] = -rear[:, 2]
    return {"S0": crop, "S1": crop[z < 10], "S2": crop[z >= 20], "S3": crop[z >= 30],
            "S4": crop[np.abs(crop[:, 0]) < 0.25 * z], "S6": rear[in_range(rear)], "S7": crop[z >= 50]}


def loader_choice(n, rng, npoints=NPOINTS):
    """kitti_dataloader.py:137-147: npoints indices without replacement when n >= npoints, otherwise a permutation of
    all n followed by npoints - n drawn with replacement"""
    if n >= npoints:
        return rng.choice(n, npoints, replace=False)
    return np.concatenate([rng.choice(n, n, replace=False), rng.choice(n, npoints - n, replace=True)])


def rotate_vertical(p, angle):
    """rotation about the camera y axis (vertical), in float64, rounded once to float32"""
    c, s = np.cos(angle), np.sin(angle)
    q = np.asarray(p, np.float64).copy()
    x, z = q[:, 0].copy(), q[:, 2].copy()
    q[:, 0], q[:, 2] = c * x + s * z, -s * x + c * z
    return q.astype(np.float32)


@functools.lru_cache(maxsize=None)
def _scenes_cached():
    src = scene_sources()
    out, choice = [], {}
    for i, name in enumerate(NAMES):
        if name == "S5":
            out.append(rotate_vertical(out[0], ROTATION))
            choice[name] = choice["S0"]
            continue
        rng = np.random.default_rng(SCENE_SEED + i)
        choice[name] = loader_choice(src[name].shape[0], rng)
        out.append(src[name][choice[name]])
    return np.ascontiguousarray(np.stack(out), dtype=np.float32), choice


def realscan_scenes():
    """[8, 16384, 4] float32 (S0..S7) and name -> the loader's choice of source rows"""
    pts, choice = _scenes_cached()
    return pts.copy(), dict(choice)


def distinct_rows(x):
    return np.unique(np.ascontiguousarray(x).view(np.dtype((np.void, x.dtype.itemsize * x.shape[-1])))).size


# ---------------------------------------------------------------------------------------------------------------------
# the fixture and the scenes
# ---------------------------------------------------------------------------------------------------------------------
def test_full_scan_fixture():
    """All 123 398 points of the scan, one pair of them exact duplicates; the 16 384-point fixture is a choice from its
    detection-range crop."""
    v = full_scan()
    assert v.shape == (123398, 4) and v.dtype == np.float32 and np.isfinite(v).all()
    assert (v[:, 3] > 0).all() and (v[:, 3] < 1).all() and 0.45 < v[:, 3].mean() < 0.55
    assert np.unique(v[:, 3]).size == 256                             # every intensity code occurs
    assert distinct_rows(v[:, :3]) == 123397
    assert ((v[:, :3] == 0) & np.signbit(v[:, :3])).sum() == 12      # the text's "-0.000" entries stay -0
    r = camera_frame(v)
    crop = r[in_range(r)]
    sub = np.load(SUBSAMPLE)
    assert int(sub["kept"]) == crop.shape[0] == 31975
    rows = lambda a: set(map(bytes, np.ascontiguousarray(a[:, :3])))
    assert rows(sub["points"]) <= rows(crop)


def test_scene_sources_have_the_stated_counts():
    src = scene_sources()
    assert sorted(src) == sorted(SOURCE_COUNTS)
    for name, (n, distinct) in SOURCE_COUNTS.items():
        assert src[name].shape == (n, 4), name
        assert distinct_rows(src[name][:, :3]) == distinct, name
        assert in_range(src[name]).all(), name
    assert np.abs(scene_sources()["S4"][:, 0]).max() < 0.25 * 70


@pytest.mark.parametrize("name", NAMES)
def test_scenes_follow_the_loader_choice(name):
    """Every row of a scene is a row of its region, bit for bit; a region with at least 16 384 points is drawn without
    replacement, a shorter one holds each of its points and pads with exact copies."""
    pts, choice = realscan_scenes()
    i = NAMES.index(name)
    x = pts[i]
    assert x.shape == (NPOINTS, 4) and x.dtype == np.float32
    c = choice[name]
    if name == "S5":
        np.testing.assert_array_equal(x, rotate_vertical(pts[0], ROTATION))
        assert not np.array_equal(x[:, [0, 2]], pts[0][:, [0, 2]])
        np.testing.assert_array_equal(x[:, [1, 3]], pts[0][:, [1, 3]])          # height and intensity stay
        assert distinct_rows(x[:, :3]) == distinct_rows(pts[0][:, :3])
        return
    n, distinct = SOURCE_COUNTS[name]
    np.testing.assert_array_equal(x, scene_sources()[name][c])
    if n >= NPOINTS:
        assert np.unique(c).size == NPOINTS
    else:
        assert np.unique(c).size == n and np.array_equal(np.sort(c[:n]), np.arange(n))
        assert NPOINTS - n == {"S1": 616, "S2": 9181, "S3": 14879, "S4": 6825, "S7": 16041}[name]
    assert distinct_rows(x[:, :3]) == min(distinct, distinct_rows(scene_sources()[name][np.unique(c)][:, :3]))
    assert distinct_rows(x) == np.unique(c).size                # a pad is an exact copy, intensity included


def test_exhaustion_claims():
    """S3 has fewer distinct points than layer 1 samples; S7 fewer than layer 2 samples.  Layer 2 samples the layer-1
    centres, which are rows of the scene, and a centre's features are a function of its coordinates (the ball query
    lists the same neighbours for equal centres), so both layer-2 samplers of S7 run out of distinct points too.
    The other scenes have more distinct points than layer 1 samples."""
    pts, _ = realscan_scenes()
    d = {name: distinct_rows(pts[i][:, :3]) for i, name in enumerate(NAMES)}
    assert d["S3"] == 1505 < L1_SAMPLES
    assert d["S7"] == 343 < L2_SAMPLES
    assert all(d[k] > L1_SAMPLES for k in ("S0", "S1", "S2", "S4", "S5", "S6")), d
    for name in ("S3", "S7"):
        i = NAMES.index(name)
        idx = oracle_ops.farthest_point_sample(L1_SAMPLES, pts[i:i + 1, :, :3])[0]
        picked = pts[i][idx, :3]
        assert distinct_rows(picked) == d[name]             # every distinct point once, then repeats
        assert distinct_rows(picked[:d[name]]) == d[name]


# ---------------------------------------------------------------------------------------------------------------------
# the CPU models of the pruned kernels against the oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def layer1_fps():
    """[8, 4096] oracle D-FPS indices of the eight scenes"""
    pts, _ = realscan_scenes()
    return oracle_ops.farthest_point_sample(L1_SAMPLES, pts[..., :3])


@pytest.mark.parametrize("name", NAMES)
def test_pruned_dfps_model_layer1(layer1_fps, name):
    i = NAMES.index(name)
    pts, _ = realscan_scenes()
    x = pts[i:i + 1, :, :3]
    for contract in (True, False):
        got, _ = oracle_ops.fps_pruned_model(L1_SAMPLES, x, contract=contract)
        np.testing.assert_array_equal(got[0], layer1_fps[i], err_msg="%s, contract %s" % (name, contract))


@pytest.mark.parametrize("name", ["S3", "S7"])
def test_pruned_dfps_model_resumed_past_exhaustion(layer1_fps, name):
    """Resumed at the latency schedule's cuts, the later ones past the last distinct point."""
    i = NAMES.index(name)
    pts, _ = realscan_scenes()
    x = pts[i:i + 1, :, :3]
    out = np.full((1, L1_SAMPLES), -7, np.int32)
    temp = np.zeros((1, 2 * NPOINTS), np.float32)
    cuts = (0, 1, 343, 1392, 2539, 3440, L1_SAMPLES)
    for j0, j1 in zip(cuts[:-1], cuts[1:]):
        oracle_ops.fps_pruned_model(L1_SAMPLES, x, rounds=(j0, j1), temp=temp, out=out)
        np.testing.assert_array_equal(out[0, :j1], layer1_fps[i, :j1])


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("dilated", [True, False])
def test_grid_model_layer1(layer1_fps, name, dilated):
    """Layer 1's shells (dilated) and a plain two-radius query, centred on the layer-1 samples."""
    i = NAMES.index(name)
    pts, _ = realscan_scenes()
    x = np.ascontiguousarray(pts[i:i + 1, :, :3])
    q = oracle_ops.gather_point(x, layer1_fps[i:i + 1])
    bq_model_check(x, q, *(LAYER1_SHELLS if dilated else PLAIN_SHELLS), dilated)


@pytest.mark.parametrize("name", ["S0", "S3"])
def test_pruned_ffps_model_on_layer1_features(name):
    """The layer-2 F-FPS operands: the oracle's layer-1 centres and features of the scene."""
    pkg = importlib.import_module("3dssd_b200")
    from oracle import layers as olayers
    arch = pkg.config.ARCH_3DSSD
    i = NAMES.index(name)
    pts, _ = realscan_scenes()
    xyz_l, feat_l, _ = olayers.backbone_forward(arch[:1], pts[i:i + 1], pkg.params.init_params(arch, 1, seed=0))
    x = np.concatenate([xyz_l[1][0], feat_l[1][0]], 1)
    idx, (bad, _) = oracle_ops.ffps_prune_model(L2_SAMPLES, x)
    assert bad == 0
    np.testing.assert_array_equal(idx, oracle_ops.farthest_point_sample_features(L2_SAMPLES, xyz_l[1], feat_l[1])[0])
    if name == "S3":
        assert distinct_rows(x) <= 1505 < x.shape[0]
