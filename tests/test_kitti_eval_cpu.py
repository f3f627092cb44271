"""KITTI evaluator on the CPU (DESIGN.md section 3.10): the overlaps of the float64 restatement (oracle/kitti_eval.py)
against an independent halfspace-intersection computation and closed forms; the C twin (the GPU kernels' recipe)
against the restatement; the evaluator's rules on hand-written frames; getThresholds; the label parser, the detection
rows, R40 AP, and the operand checks of the tf_ops wrappers."""
import math

import numpy as np
import pytest
import torch

from oracle import kitti_eval as K

CAR, PED, CYC, VAN, SIT, DC, OTHER = range(7)


@pytest.fixture(scope="module")
def twin():
    K.build()
    return K.twin()


# ---- overlaps ------------------------------------------------------------------------------------------------------
def _halfspaces(b):
    """A rotated (t1, t3, l, w, ry) rectangle as 4 halfspaces A x + c <= 0 in the (x, z) plane, built from its axes."""
    t1, t3, l, w, ry = b
    ax = np.array([math.cos(ry), -math.sin(ry)])      # the box's l axis in (x, z)
    az = np.array([math.sin(ry), math.cos(ry)])       # its w axis
    ctr = np.array([t1, t3])
    hs = []
    for n, half in ((ax, abs(l) / 2), (-ax, abs(l) / 2), (az, abs(w) / 2), (-az, abs(w) / 2)):
        hs.append([n[0], n[1], -(n @ ctr) - half])
    return np.array(hs)


def _area_independent(a, b):
    from scipy.optimize import linprog
    from scipy.spatial import ConvexHull, HalfspaceIntersection
    hs = np.vstack([_halfspaces(a), _halfspaces(b)])
    norm = np.linalg.norm(hs[:, :2], axis=1)
    # Chebyshev centre: the deepest point of the intersection (negative depth when the rectangles are disjoint)
    res = linprog([0, 0, -1], A_ub=np.hstack([hs[:, :2], norm[:, None]]), b_ub=-hs[:, 2], bounds=[(None, None)] * 3,
                  method="highs")
    assert res.status == 0, res.message
    if res.x[2] < 1e-7:
        return 0.0
    return ConvexHull(HalfspaceIntersection(hs, res.x[:2]).intersections).volume


def _random_pairs(n, seed):
    rng = np.random.default_rng(seed)
    edges = np.array([-np.pi + k * 2 * np.pi / 12 for k in range(13)] + [np.pi, -np.pi])
    out = []
    for i in range(n):
        d = [rng.uniform(-3, 3), rng.uniform(0.5, 2), rng.uniform(10, 30), rng.uniform(0.3, 5), rng.uniform(0.5, 2),
             rng.uniform(0.3, 3), 0.0]
        g = list(d)
        g[0] += rng.normal(0, 1.0)
        g[1] += rng.normal(0, 0.5)
        g[2] += rng.normal(0, 1.0)
        g[3:6] = [x * rng.uniform(0.6, 1.4) for x in d[3:6]]
        kind = i % 4
        d[6] = float(rng.choice(edges)) if kind == 0 else rng.uniform(-4, 4)
        g[6] = d[6] + rng.normal(0, 1e-7) if kind == 1 else (float(rng.choice(edges)) if kind == 2 else rng.uniform(-4, 4))
        out.append((np.float32(d).astype(np.float64), np.float32(g).astype(np.float64)))
    return out


def test_python_overlaps_match_an_independent_halfspace_intersection():
    for d, g in _random_pairs(10000, 0):
        inter = _area_independent((d[0], d[2], d[3], d[5], d[6]), (g[0], g[2], g[3], g[5], g[6]))
        ad, ag = d[3] * d[5], g[3] * g[5]
        bev, v3 = K.box_overlaps(d, g)
        assert abs(bev - inter / (ad + ag - inter)) < 1e-9, (d, g)
        yov = max(0.0, min(d[1], g[1]) - max(d[1] - d[4], g[1] - g[4]))
        vd, vg = d[4] * d[3] * d[5], g[4] * g[3] * g[5]
        assert abs(v3 - inter * yov / (vd + vg - inter * yov)) < 1e-9, (d, g)


def _closed_form_cases():
    car = [0.0, 1.5, 20.0, 4.0, 1.5, 2.0, 0.3]
    sq = [1.0, 1.0, 10.0, 2.0, 1.0, 2.0, 0.0]
    yield car, car, 1.0, 1.0                                                # identical
    yield sq, sq[:6] + [np.pi / 2], 1.0, 1.0                               # a square turned by 90 degrees
    inner = [0.0, 1.5, 20.0, 2.0, 0.75, 1.0, 0.0]
    outer = [0.0, 1.5, 20.0, 4.0, 1.5, 2.0, 0.0]
    yield inner, outer, 2.0 / 8.0, (2.0 * 0.75) / (8.0 * 1.5)              # contained: area and volume ratios
    yield [0.0, 1.5, 20.0, 4.0, 1.5, 2.0, 0.0], [4.0, 1.5, 20.0, 4.0, 1.5, 2.0, 0.0], 0.0, 0.0      # edge-touching
    yield [0.0, 1.5, 20.0, 4.0, 1.5, 2.0, 0.0], [4.0, 1.5, 22.0, 4.0, 1.5, 2.0, 0.0], 0.0, 0.0      # corner-touching
    yield [0.0, 1.5, 20.0, 4.0, 1.5, 2.0, 0.0], [9.0, 1.5, 29.0, 4.0, 1.5, 2.0, 0.7], 0.0, 0.0      # disjoint
    yield [0.0, 1.5, 20.0, 4.0, 1.5, 2.0, 0.0], [0.0, -0.5, 20.0, 4.0, 1.5, 2.0, 0.0], 1.0, 0.0     # no y-overlap


@pytest.mark.parametrize("case", list(range(7)))
def test_overlap_closed_forms(twin, case):
    d, g, bev, v3 = list(_closed_form_cases())[case]
    got = K.box_overlaps(d, g)
    assert abs(got[0] - bev) < 1e-12 and abs(got[1] - v3) < 1e-12, got
    tb, t3 = K.twin_box_iou(np.float32([[d]]), np.float32([[g]]))
    assert abs(tb[0, 0, 0] - bev) < 1e-6 and abs(t3[0, 0, 0] - v3) < 1e-6


def test_twin_overlaps_match_the_restatement(twin):
    rng = np.random.default_rng(3)
    pairs = _random_pairs(3000, 1)
    dets = np.zeros((len(pairs), 14), np.float32)
    labs = np.zeros((len(pairs), 15))
    for k, (d, g) in enumerate(pairs):
        x1, y1 = rng.uniform(0, 500, 2)
        dets[k] = [0, x1, y1, x1 + rng.uniform(1, 90), y1 + rng.uniform(1, 90), 0, d[0], d[1], d[2], d[4], d[5], d[3], d[6], 0.5]
        labs[k] = [CAR, 0, 0, 0, x1 + rng.normal(0, 20), y1 + rng.normal(0, 20), x1 + rng.uniform(1, 90), y1 + rng.uniform(1, 90),
                   g[4], g[5], g[3], g[0], g[1], g[2], g[6]]
    got = K.twin_pair_overlaps(dets, labs)
    exp = np.array([K.pair_overlaps(dets[k], labs[k]) for k in range(len(pairs))])
    np.testing.assert_allclose(got, exp, rtol=0, atol=1e-12)


def test_shared_sincos_is_within_two_ulp_of_libm(twin):
    rng = np.random.default_rng(4)
    x = np.concatenate([rng.uniform(-4 * np.pi, 4 * np.pi, 1000000),
                        np.float32([np.pi, -np.pi, np.pi / 2, np.pi / 4]).astype(np.float64),
                        np.array([-np.pi + k * np.pi / 6 for k in range(13)])])
    s, c = K.twin_sincos(x)
    ms = np.array([math.sin(v) for v in x])
    mc = np.array([math.cos(v) for v in x])
    assert np.all(np.abs(s - ms) <= 2 * np.spacing(np.abs(ms)))
    assert np.all(np.abs(c - mc) <= 2 * np.spacing(np.abs(mc)))


# ---- rules on hand-written frames ----------------------------------------------------------------------------------
def lab(t, box=(100, 100, 200, 200), trunc=0.0, occ=0, loc=(0.0, 1.5, 20.0), dims=(1.5, 1.6, 3.9), ry=0.0):
    """A label row: type, 2-D box (x1, y1, x2, y2), truncation, occlusion, location, (h, w, l), ry."""
    return [t, trunc, occ, 0.0] + list(box) + list(dims) + list(loc) + [ry]


def det(c, box=(100, 100, 200, 200), score=0.9, loc=(0.0, 1.5, 20.0), dims=(1.5, 1.6, 3.9), ry=0.0):
    return [c] + list(box) + [0.0] + list(loc) + list(dims) + [ry, score]


FAR = dict(box=(600, 100, 700, 200), loc=(10.0, 1.5, 40.0))
# frame -> {(metric, class, difficulty): (thresholds, tp, fp, fn)}; metrics 0 image, 1 ground, 2 3-D
RULES = {
    "van_under_car": ([lab(CAR), lab(VAN, box=(300, 100, 400, 200), loc=(5.0, 1.5, 20.0))],
                      [det(0), det(0, box=(300, 100, 400, 200), loc=(5.0, 1.5, 20.0), score=0.95)],
                      {(0, 0, 0): ([0.9], [1], [0], [0]), (1, 0, 0): ([0.9], [1], [0], [0])}),
    "person_sitting": ([lab(PED, dims=(1.7, 0.6, 0.8)), lab(SIT, box=(300, 100, 400, 200), loc=(5.0, 1.5, 20.0), dims=(1.7, 0.6, 0.8))],
                       [det(1, dims=(1.7, 0.6, 0.8)), det(1, box=(300, 100, 400, 200), loc=(5.0, 1.5, 20.0), dims=(1.7, 0.6, 0.8), score=0.95)],
                       {(0, 1, 0): ([0.9], [1], [0], [0])}),
    "occlusion_1": ([lab(CAR, occ=1)], [det(0)],
                    {(0, 0, 0): ([], [], [], []), (0, 0, 1): ([0.9], [1], [0], [0])}),
    "truncation_0.15": ([lab(CAR, trunc=0.15)], [det(0)], {(0, 0, 0): ([0.9], [1], [0], [0])}),
    "truncation_0.16": ([lab(CAR, trunc=0.16)], [det(0)],
                        {(0, 0, 0): ([], [], [], []), (0, 0, 1): ([0.9], [1], [0], [0])}),
    "gt_height_40": ([lab(CAR, box=(100, 100, 200, 140))], [det(0, box=(100, 100, 200, 140))],
                     {(0, 0, 0): ([], [], [], []), (0, 0, 1): ([0.9], [1], [0], [0])}),
    "det_height_24.9": ([lab(CAR, box=(100, 100, 200, 130))], [det(0, box=(100, 100, 200, 124.9))],
                        {(0, 0, 1): ([], [], [], [])}),
    "det_height_25": ([lab(CAR, box=(100, 100, 200, 130))], [det(0, box=(100, 100, 200, 125))],
                      {(0, 0, 1): ([0.9], [1], [0], [0])}),
    "dontcare_absorbs": ([lab(CAR), lab(DC, box=(400, 100, 600, 300), loc=(-1000, -1000, -1000), dims=(-1, -1, -1), ry=-10)],
                         [det(0), det(0, box=(420, 120, 520, 220), loc=(-8.0, 1.5, 30.0), score=0.95)],
                         {(0, 0, 0): ([0.9], [1], [0], [0]), (1, 0, 0): ([0.9], [1], [1], [0])}),
    "duplicates": ([lab(CAR), lab(CAR, box=(300, 100, 400, 200), loc=(5.0, 1.5, 20.0))],
                   [det(0), det(0, box=(102, 100, 202, 200), score=0.8), det(0, box=(300, 100, 400, 200), loc=(5.0, 1.5, 20.0), score=0.7)],
                   {(0, 0, 0): ([0.9, 0.7], [1, 2], [0, 1], [1, 0])}),
    "det_on_ignored_gt": ([lab(CAR, occ=3)], [det(0)], {(0, 0, 2): ([], [], [], [])}),
    "score_tie": ([lab(CAR)], [det(0, box=(104, 100, 204, 200), score=0.8), det(0, score=0.8)],
                  {(0, 0, 0): ([0.8], [1], [1], [0])}),
    "no_labels": ([], [det(0, **FAR)], {(0, 0, 0): ([], [], [], [])}),
    "no_detections": ([lab(CAR), lab(PED, box=(300, 100, 400, 200))], [], {}),
}


def _frame(name):
    labels, dets, exp = RULES[name]
    return (np.asarray(dets, np.float32).reshape(-1, 14), [np.asarray(labels, np.float64).reshape(-1, 15)],
            np.array([len(dets)], np.int32), exp)


@pytest.mark.parametrize("name", sorted(RULES))
def test_rules_on_hand_written_frames(twin, name):
    rows, labels, nl, exp = _frame(name)
    out, counts = K.evaluate(rows, labels, nl, return_counts=True)
    for key, (thr, tp, fp, fn) in exp.items():
        got = counts[key]
        assert [round(t, 6) for t in got[0]] == thr and got[1] == tp and got[2] == fp and got[3] == fn, (key, got)
        prec = np.zeros(41, np.float32)
        p = [a / (a + b) for a, b in zip(tp, fp)]
        prec[:len(p)] = [max(p[i:]) for i in range(len(p))]
        np.testing.assert_array_equal(out[2 * key[0]][key[1], key[2]], prec)
    tw = K.twin_evaluate(rows, labels, nl)
    for a, b in zip(out, tw):
        np.testing.assert_array_equal(a, b)
    for k in (1, 3, 5):
        assert np.all(out[k] == -1)                    # AOS is never computed


def test_class_without_detections_gives_minus_one_rows(twin):
    rows = np.concatenate([_frame("van_under_car")[0], _frame("person_sitting")[0]])
    labels = _frame("van_under_car")[1] + _frame("person_sitting")[1]
    out = K.twin_evaluate(rows, labels, np.array([2, 2], np.int32))
    for m in (0, 2, 4):
        assert np.all(out[m][2] == -1)                 # no Cyclist detection: not evaluated
        assert np.all(out[m][0] >= 0) and np.all(out[m][1] >= 0)
    empty = K.twin_evaluate(np.zeros((0, 14), np.float32), labels, np.array([0, 0], np.int32))
    assert all(np.all(a == -1) for a in empty)


def test_get_thresholds_hand_computed_and_bounded(twin):
    from importlib import import_module
    ev = import_module("3dssd_b200.evaluation")
    for scores, n_gt, exp in (([0.7, 0.9, 0.8], 3, [0.9, 0.8, 0.7]), ([0.9, 0.8, 0.7, 0.6], 80, [0.9, 0.8, 0.6]),
                              ([], 5, []), ([0.5, 0.5], 2, [0.5, 0.5])):
        assert K.get_thresholds(scores, n_gt) == exp
        assert ev.get_thresholds(scores, n_gt) == exp
        assert K.twin_get_thresholds(scores, n_gt)[0] == exp
    rng = np.random.default_rng(5)
    for n_gt in range(1, 501):
        v = rng.uniform(0, 1, n_gt)
        t = ev.get_thresholds(v, n_gt)
        assert len(t) <= 41 and (len(t) == 41 or n_gt < 41), (n_gt, len(t))
        assert K.twin_get_thresholds(v, n_gt) == (t, len(t))


def test_twin_equals_restatement_on_synthetic_frames(twin):
    for seed in range(50):
        rows, labels, nl = K.synthetic_frames(200, seed=100 + seed, max_labels=4)
        if K.margin_ok(rows, labels, nl):
            break
    else:
        pytest.fail("no synthetic set with every overlap 1e-9 away from the decisions")
    a, b = K.evaluate(rows, labels, nl), K.twin_evaluate(rows, labels, nl)
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y)
    assert np.any(a[0] > 0) and np.any(a[4] > 0)


# ---- host-side helpers ---------------------------------------------------------------------------------------------
def test_label_parser(pkg, tmp_path):
    ev = pkg.evaluation
    p = tmp_path / "000001.txt"
    p.write_text("Car 0.00 0 -1.58 587.01 173.33 614.12 200.12 1.65 1.67 3.64 -0.65 1.71 46.70 -1.59\n"
                 "DontCare -1 -1 -10 503.89 169.71 590.61 190.13 -1 -1 -1 -1000 -1000 -1000 -10\n"
                 "\n"
                 "VAN 0.3 2 1.0 1 2 3 4 2.0 1.9 5.0 1 2 3 0.5\n"
                 "person_sitting 0 1 0 1 2 3 4 1 1 1 1 2 3 0\n"
                 "Tram 0 0 0 1 2 3 4 1 1 1 1 2 3 0\n")
    r = ev.read_label_file(str(p))
    assert r.shape == (5, 15) and r.dtype == np.float64
    assert list(r[:, 0]) == [0, 5, 3, 4, 6]
    assert r[0, 4] == 587.01 and r[0, 13] == 46.70 and r[0, 14] == -1.59 and r[2, 2] == 2 and r[1, 11] == -1000
    e = tmp_path / "e.txt"
    e.write_text("")
    assert ev.read_label_file(str(e)).shape == (0, 15)
    bad = tmp_path / "bad.txt"
    bad.write_text("Car 0 0 0 1 2 3 4 1 1 1 1 2 3 0\nCar 0 0 0 1 2 3 4 1 1 1 1 2 3\n")
    with pytest.raises(ValueError, match=r"bad.txt:2"):
        ev.read_label_file(str(bad))
    bad.write_text("Car 0 x 0 1 2 3 4 1 1 1 1 2 3 0\n")
    with pytest.raises(ValueError, match=r"bad.txt:1"):
        ev.read_label_file(str(bad))


def test_detection_rows_restate_evaluate_map(pkg):
    ev, io = pkg.evaluation, pkg.kitti_io
    rng = np.random.default_rng(6)
    block = np.zeros((2, 100, 9), np.float32)
    block[:, :, 0] = rng.uniform(-10, 10, (2, 100))
    block[:, :, 1] = rng.uniform(1, 2, (2, 100))
    block[:, :, 2] = rng.uniform(8, 50, (2, 100))
    block[:, :, 3:6] = rng.uniform(0.5, 4, (2, 100, 3))
    block[:, :, 6] = rng.uniform(-3, 3, (2, 100))
    block[:, :, 7] = rng.uniform(0, 1, (2, 100))
    cnt = np.array([40, 0], np.int32)
    p2 = np.array([[721.5, 0, 609.6, 44.9], [0, 721.5, 172.9, 0.2], [0, 0, 1, 0.003]], np.float32)
    for cls_list, shift in ((("Car",), 0), (("Pedestrian", "Cyclist"), 1)):
        rows, nl = ev.detection_rows(block, cnt, [p2, p2], cls_list=cls_list, cls_thresh=0.3)
        d = block[0, :40]
        d = d[d[:, 7] >= 0.3]
        exp = np.zeros((len(d), 14), np.float32)
        exp[:, 0] = d[:, 8] + shift
        exp[:, 1:5] = io.project_boxes_to_image(d[:, :7], p2)
        exp[:, 6:9] = d[:, :3]
        exp[:, 9], exp[:, 10], exp[:, 11], exp[:, 12], exp[:, 13] = d[:, 4], d[:, 5], d[:, 3], d[:, 6], d[:, 7]
        np.testing.assert_array_equal(rows, exp)
        assert list(nl) == [len(d), 0]


def test_kitti_ap_is_the_float32_sum_over_forty(pkg):
    p = np.random.default_rng(7).uniform(0, 1, (3, 3, 41)).astype(np.float32)
    ap = pkg.evaluation.kitti_ap(p)
    assert ap.dtype == np.float32
    np.testing.assert_array_equal(ap, np.sum(p[..., 1:], axis=-1) / 40.)
    one = np.ones((3, 3, 41), np.float32)
    np.testing.assert_array_equal(pkg.evaluation.kitti_ap(one), np.ones((3, 3), np.float32))


def test_wrappers_check_operands_before_the_library(pkg, monkeypatch):
    T = pkg.tf_ops

    class NoLib:
        def __getattr__(self, name):
            raise AssertionError("the library was called: %s" % name)

    monkeypatch.setattr(T, "lib", lambda: NoLib())
    f = lambda *s: torch.zeros(s, dtype=torch.float32)
    with pytest.raises(ValueError, match="CUDA"):
        T.calc_iou(f(1, 2, 7), f(1, 3, 7))
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    for args in ((f(1, 2, 6), f(1, 3, 7)), (f(1, 2, 7), f(2, 3, 7)), (f(2, 7), f(2, 7))):
        with pytest.raises(ValueError):
            T.calc_iou(*args)
    for args in ((f(3, 7), f(2, 7)), (f(1, 3, 7), f(1, 3, 7)), (f(3, 7).double(), f(3, 7))):
        with pytest.raises(ValueError):
            T.calc_iou_match(*args)
    n = lambda *v: torch.tensor(v, dtype=torch.int32)
    lab = [np.zeros((2, 15))]
    bad = [(f(3, 13), lab, n(3)), (f(3, 14), lab, n(2)), (f(3, 14), [np.zeros((2, 14))], n(3)), (f(3, 14), lab, n(1, 2)),
           (f(1025, 14), lab, n(1025)), (f(1, 14), [np.zeros((257, 15))], n(1)), (f(3, 14), lab, n(3).float())]
    for d, l, nl in bad:
        with pytest.raises(ValueError):
            T.evaluate_labels(d, l, nl)
    with pytest.raises(ValueError):
        T.evaluate(f(3, 14), ["a.txt", "b.txt"], n(3))
