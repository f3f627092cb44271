"""CPU tests of the BEV NMS decision arithmetic (DESIGN.md §3.5): the numpy oracle (oracle/head.py:bev_nms) and its C
twin (oracle/ssd3d_oracle.c:oracle_bev_nms) on box pairs that sit exactly at the IoU threshold, checked against the exact
IoU of their float32 rectangles, and on the scenes the GPU test (tests/test_bev_nms_gpu.py) runs through the kernel.

Every suppression is the float32 comparison IoU > thr.  Random boxes almost never put an IoU within an ulp of the
threshold, so they cannot tell two rectangle or IoU recipes apart.  The boundary pairs here do: one box of each pair is
slid along x (or z), bisecting over adjacent float32 coordinates, to the last position the numpy oracle suppresses and
the first it keeps.
"""
import functools
import math
from fractions import Fraction

import numpy as np
import pytest

from oracle import head as ohead

F32 = np.float32

# The pinned IoU recipe is a faithful rounding: iw, ih, inter, both areas, their sum, the union and the quotient are
# each rounded once, which puts the float32 IoU within 16 * 2^-24 of the exact IoU of the float32 rectangles, relatively
# (3 roundings in inter, at most 12 in the union after the cancellation inter <= min(area) allows, 1 in the quotient).
# For thr in [2^-4, 2^-3) -- 0.1 -- that is 16 ulp of float32(thr).  A decision may differ from the exact comparison
# IoU > float32(thr) only when the exact IoU lies within this bound of the threshold.
REL_BOUND = Fraction(16, 2 ** 24)


def f2ord(f):
    """float32 -> int64, monotone in the float order, with -0 and +0 both at 0."""
    b = np.asarray(f, np.float32).view(np.int32).astype(np.int64)
    return np.where(b < 0, -(b & 0x7fffffff), b)


def ord2f(o):
    o = np.asarray(o, np.int64)
    return np.where(o < 0, (-o) | 0x80000000, o).astype(np.uint32).view(np.float32)


def exact_iou(ra, rb):
    """Exact IoU of two BEV rectangles (x1, z1, x2, z2) given as float32 corners, as a Fraction (0 if either area is
    <= 0, which the NMS treats as never suppressing)."""
    x1a, z1a, x2a, z2a = (Fraction(float(v)) for v in ra)
    x1b, z1b, x2b, z2b = (Fraction(float(v)) for v in rb)
    area_a, area_b = (x2a - x1a) * (z2a - z1a), (x2b - x1b) * (z2b - z1b)
    if area_a <= 0 or area_b <= 0:
        return Fraction(0)
    inter = max(min(x2a, x2b) - max(x1a, x1b), 0) * max(min(z2a, z2b) - max(z1a, z1b), 0)
    return inter / (area_a + area_b - inter)


def near_threshold(iou, thr):
    """True when the exact IoU is within REL_BOUND (relative) of float32(thr): where a faithful float32 recipe may
    decide either way."""
    t = Fraction(float(F32(thr)))
    return abs(iou - t) <= REL_BOUND * abs(t)


def iou64(ra, rb):
    """IoU in float64 from float32 corners (relative error ~1e-15): a prefilter, exact_iou decides near the threshold."""
    ra, rb = np.asarray(ra, np.float64), np.asarray(rb, np.float64)
    area_a = (ra[..., 2] - ra[..., 0]) * (ra[..., 3] - ra[..., 1])
    area_b = (rb[..., 2] - rb[..., 0]) * (rb[..., 3] - rb[..., 1])
    iw = np.minimum(ra[..., 2], rb[..., 2]) - np.maximum(ra[..., 0], rb[..., 0])
    ih = np.minimum(ra[..., 3], rb[..., 3]) - np.maximum(ra[..., 1], rb[..., 1])
    inter = np.maximum(iw, 0) * np.maximum(ih, 0)
    with np.errstate(invalid="ignore", divide="ignore"):
        iou = inter / (area_a + area_b - inter)
    return np.where((area_a > 0) & (area_b > 0), iou, 0.0)


# ---- boundary pairs ---------------------------------------------------------------------------------------------------

def boundary_angles(rng, n_random=200):
    """0, ±π/2, ±π, the float32 values nearest kπ/4, and random angles in [-π, π]."""
    a = [0.0, math.pi / 2, -math.pi / 2, math.pi, -math.pi] + [k * math.pi / 4 for k in range(-8, 9)]
    a = list(np.asarray(a, np.float32)) + list(rng.uniform(-np.pi, np.pi, n_random).astype(np.float32))
    return np.asarray(a, np.float32)


def pair_boxes(rng, angles, kitti, axis, centers=None):
    """Box A at angle `angles`, box B of a similar size centred on A but for a small offset across `axis` (0: x, 2: z).
    Half the B boxes are axis-aligned, the others take the next angle of the list."""
    p = len(angles)
    if kitti:
        l, w = rng.uniform(3.0, 4.8, p), rng.uniform(1.4, 2.0, p)
    else:
        l, w = rng.uniform(0.2, 1.0, p), rng.uniform(0.2, 1.0, p)
    if centers is None:
        centers = (np.stack([rng.uniform(-40, 40, p), rng.uniform(0, 70, p)], -1) if kitti
                   else rng.uniform(-2, 2, (p, 2)))
    h = rng.uniform(1.4, 1.8, p)
    y = rng.uniform(-1.0, 2.5, p)
    partner = np.where(np.arange(p) % 2 == 0, 0.0, np.roll(angles, -1))
    sl, sw = rng.uniform(0.7, 1.3, p), rng.uniform(0.7, 1.3, p)
    a = np.stack([centers[:, 0], y, centers[:, 1], l, h, w, angles], -1).astype(np.float32)
    b = np.stack([centers[:, 0], y, centers[:, 1], l * sl, h, w * sw, partner], -1).astype(np.float32)
    across = 2 - axis
    b[:, across] += (rng.uniform(-0.2, 0.2, p) * np.minimum(l, w)).astype(np.float32)
    return a, b


def _suppressed(a, b, thr):
    """Whether the numpy oracle drops B (score 0.8) after keeping A (score 0.9): one two-box scene per pair."""
    boxes = np.stack([a, b], 1)
    scores = np.broadcast_to(np.array([0.9, 0.8], np.float32), (len(a), 2))
    return ohead.bev_nms(boxes, scores, thr, 2)[1] == 1


def bisect_pairs(a, b, axis, thr):
    """Slide B along `axis` from A's centre (suppressed) to beyond any overlap (kept), bisecting over float32
    coordinates.  Returns (a, b_sup, b_keep) for the pairs whose ends decide as expected (a B much smaller than A may
    stay below the threshold even on A's centre): b_sup at the last coordinate that suppresses, b_keep at the next
    float32."""
    lo = b[:, axis].copy()
    hi = (lo + (a[:, 3] + a[:, 5] + b[:, 3] + b[:, 5])).astype(np.float32)
    at = lambda c: np.concatenate([b[:, :axis], c[:, None], b[:, axis + 1:]], 1)
    valid = _suppressed(a, at(lo), thr) & ~_suppressed(a, at(hi), thr)
    a, b = a[valid], b[valid]
    at = lambda c: np.concatenate([b[:, :axis], c[:, None], b[:, axis + 1:]], 1)
    olo, ohi = f2ord(lo[valid]), f2ord(hi[valid])
    while (ohi - olo > 1).any():
        mid = (olo + ohi) // 2
        sup = _suppressed(a, at(ord2f(mid)), thr)
        olo, ohi = np.where(sup, mid, olo), np.where(sup, ohi, mid)
    return a, at(ord2f(olo)), at(ord2f(ohi))


@functools.lru_cache(maxsize=None)
def boundary_pairs(thr=0.1, seed=0, n_random=200):
    """[(a, b_sup, b_keep)] over angles x {small, KITTI-like} x {x, z}: the numpy oracle suppresses b_sup and keeps
    b_keep, whose slid coordinates are adjacent float32 values."""
    rng = np.random.default_rng(seed)
    angles = boundary_angles(rng, n_random)
    out = []
    for kitti in (False, True):
        for axis in (0, 2):
            a, b = pair_boxes(rng, angles, kitti, axis)
            out.append(bisect_pairs(a, b, axis, thr))
    a, bs, bk = (np.concatenate(v) for v in zip(*out))
    assert len(a) >= (0.9 if thr < 0.3 else 0.5) * 4 * len(angles)    # at 0.5 a rotated B often stays below it
    return a, bs, bk


# ---- scenes shared with the GPU test ------------------------------------------------------------------------------------

def clustered_boxes(rng, b, n, objects=30, jitter=0.5):
    """KITTI-like candidates: several per object, jittered in centre, size and angle, as a detection head proposes."""
    obj_c = np.stack([rng.uniform(-40, 40, (b, objects)), rng.uniform(-1, 2.5, (b, objects)),
                      rng.uniform(0, 70, (b, objects))], -1)
    obj_s = np.stack([rng.uniform(3.0, 4.8, (b, objects)), rng.uniform(1.4, 1.8, (b, objects)),
                      rng.uniform(1.4, 2.0, (b, objects))], -1)
    obj_r = rng.uniform(-np.pi, np.pi, (b, objects))
    k = rng.integers(0, objects, (b, n))
    take = lambda v: np.take_along_axis(v, k.reshape(b, n, *([1] * (v.ndim - 2))), 1)
    ctr = take(obj_c) + rng.normal(0, jitter, (b, n, 3))
    size = take(obj_s) * rng.uniform(0.85, 1.15, (b, n, 3))
    ry = take(obj_r) + rng.normal(0, 0.15, (b, n))
    return np.concatenate([ctr, size, ry[..., None]], -1).astype(np.float32)


def grid_cells(k):
    """k BEV centres (x, z) 10 m apart over x in [-65, 65], z in [2, 62]: pairs placed there do not interact."""
    gx, gz = np.meshgrid(np.arange(-65.0, 66.0, 10.0), np.arange(2.0, 63.0, 10.0))
    cells = np.stack([gx.ravel(), gz.ravel()], -1)
    assert k <= len(cells)
    return cells[:k]


def follower(b):
    """B moved on along x by a fifth of its smaller side: IoU(B, C) >= 2/3, and C is further from A than B is."""
    c = b.copy()
    c[:, 0] += F32(0.2) * np.minimum(b[:, 3], b[:, 5])
    return c


def chain_scene(rng, thr, groups=80, n=512, seed=0):
    """n candidates: `groups` boundary pairs (A, B) at the suppress or the keep position, each followed by a box C that
    overlaps B well above the threshold but not A, so B's decision decides C's; the rest are decoys.  A > B > C in
    score within a group, groups interleaved in score with each other and with the decoys."""
    cells = grid_cells(groups) + rng.uniform(-1, 1, (groups, 2))
    angles = boundary_angles(rng, groups)[rng.permutation(groups + 22)[:groups]]
    a, b = pair_boxes(rng, angles, True, 0, centers=cells)
    a, bs, bk = bisect_pairs(a, b, 0, thr)
    g = len(a)
    pick = rng.integers(0, 2, g).astype(bool)
    bb = np.where(pick[:, None], bs, bk)
    c = follower(bb)
    d = clustered_boxes(rng, 1, n - 3 * g)[0]
    boxes = np.concatenate([a, bb, c, d]).astype(np.float32)
    top = rng.uniform(0.5, 1.0, g).astype(np.float32)
    scores = np.concatenate([top, top * F32(0.999), top * F32(0.998), rng.uniform(0, 1, n - 3 * g)]).astype(np.float32)
    perm = rng.permutation(n)
    return boxes[perm], scores[perm]


def _case(name, boxes, scores, thr=0.1, max_out=100, cls_id=0):
    boxes = np.array(boxes, np.float32)
    scores = np.array(scores, np.float32)
    if boxes.ndim == 2:
        boxes, scores = boxes[None], scores[None]
    return dict(name=name, boxes=boxes, scores=scores, thr=thr, max_out=max_out, cls_id=cls_id)


def degenerate_boxes():
    """ry = 0: l = 0, w = 0, subnormal and tiny sizes (areas 0 and subnormal), boxes touching along an edge (the
    intersection is exactly 0), each next to a normal box it overlaps."""
    rows = []
    for k, (l, w) in enumerate([(0.0, 2.0), (2.0, 0.0), (1e-40, 1e-40), (1e-40, 2.0), (1e-20, 1e-20), (2e-19, 3e-19),
                                (0.0, 0.0)]):
        x = 10.0 * k
        rows += [[x, 0, 5, 2.0, 1.5, 2.0, 0], [x + 0.25, 0, 5, l, 1.5, w, 0], [x + 0.25, 0, 5, l, 1.5, w, 0]]
    for k in range(4):                      # touching: x2 of one == x1 of the next, exactly (dyadic sizes at ry = 0)
        x, z = 100.0 + 12 * k, 20.0
        rows += [[x, 0, z, 2.0, 1.5, 1.0, 0], [x + 2.0, 0, z, 2.0, 1.5, 1.0, 0], [x, 0, z + 1.0, 2.0, 1.5, 1.0, 0],
                 [x + 2.0, 0, z + 1.0, 2.0, 1.5, 1.0, 0]]
    rows += [[1e-20, 0, 1e-20, 1e-20, 1, 1e-20, 0], [1.5e-20, 0, 1e-20, 1e-20, 1, 1e-20, 0]]   # subnormal IoU terms
    return np.asarray(rows, np.float32)


@functools.lru_cache(maxsize=None)
def nms_scenes():
    """The scenes the GPU test runs through the kernel and both oracles (name -> case dict)."""
    rng = np.random.default_rng(11)
    cases = []
    for thr in (0.1, 0.5):
        for v in range(2):
            bx, sc = chain_scene(rng, thr)
            cases.append(_case("chain_thr%g_%d" % (thr, v), bx, sc, thr))
    for n in (1, 2, 31, 32, 33, 255, 256, 257, 511, 512):
        bx = clustered_boxes(rng, 2, n, objects=max(1, n // 16))
        cases.append(_case("equal_scores_n%d" % n, bx, np.stack([np.full(n, 0.5), np.full(n, 1.0)]), max_out=min(n, 100)))
    bx = clustered_boxes(rng, 2, 300, objects=20)
    sc = rng.uniform(0.2, 1.0, (2, 300))
    sc[0, 40:240] = 1.0                                                  # a long run of the saturated sigmoid
    sc[1, rng.random(300) < 0.5] = 1.0
    cases.append(_case("runs_of_one", bx, sc))
    sc = np.where(rng.random((2, 300)) < 0.5, 0.0, -0.0)               # only ±0: lower index first
    cases.append(_case("signed_zero", bx, sc))
    sc = rng.choice(np.array([1.0, 0.0, -0.0, -0.5, -1e-30, 1e-30, -1.0, 0.25], np.float32), (2, 300))
    cases.append(_case("mixed_sign_ties", bx, sc))
    cases.append(_case("negative_scores", bx, -rng.uniform(0, 5, (2, 300))))
    same = np.broadcast_to(bx[0, :1], (1, 64, 7))
    cases.append(_case("identical_boxes", same, np.full((1, 64), 0.7)))
    half = np.concatenate([same[:, :32], bx[:1, :32]], 1)
    cases.append(_case("identical_boxes_mixed", half, np.concatenate([np.full(32, 0.7), rng.uniform(0, 1, 32)])[None]))
    dg = degenerate_boxes()
    dsc = np.linspace(1.0, 0.1, len(dg))
    for thr in (0.1, 0.0, -0.1):
        cases.append(_case("degenerate_thr%g" % thr, dg, dsc, thr))
    cases.append(_case("degenerate_reversed", dg, dsc[::-1].copy()))
    bx = clustered_boxes(rng, 2, 256, objects=24)
    sc = rng.uniform(0, 1, (2, 256))
    for thr in (0.0, -0.25, 0.5, 1.0):
        cases.append(_case("thr%g" % thr, bx, sc, thr))
    bx = clustered_boxes(rng, 2, 40, objects=25, jitter=0.2)
    sc = rng.uniform(0, 1, (2, 40))
    for mo in (1, 40, 47):
        cases.append(_case("max_out%d" % mo, bx, sc, max_out=mo))
    bx = clustered_boxes(rng, 2, 512, objects=200, jitter=0.3)
    cases.append(_case("max_out_partway", bx, rng.uniform(0, 1, (2, 512)), max_out=20))
    bx = clustered_boxes(rng, 33, 100, objects=12)
    cases.append(_case("batch33_cls3", bx, rng.uniform(0, 1, (33, 100)), cls_id=3))
    cases.append(_case("batch1", bx[:1], rng.uniform(0, 1, (1, 100)), max_out=50))
    return {c["name"]: c for c in cases}


# ---- tests --------------------------------------------------------------------------------------------------------------

def test_boundary_pairs_are_adjacent_floats():
    a, bs, bk = boundary_pairs()
    moved = np.where((bs != bk).any(0))[0]
    assert set(moved) <= {0, 2}
    for axis in (0, 2):
        d = bs[:, axis] != bk[:, axis]
        assert d.any()
        assert (f2ord(bk[d, axis]) - f2ord(bs[d, axis]) == 1).all()


@pytest.mark.parametrize("thr", [0.1, 0.5])
def test_boundary_pairs_numpy_and_c_oracles_agree(oracle_ops, thr):
    a, bs, bk = boundary_pairs(thr)
    scores = np.broadcast_to(np.array([0.9, 0.8], np.float32), (2 * len(a), 2))
    boxes = np.concatenate([np.stack([a, bs], 1), np.stack([a, bk], 1)])
    nb, nc = ohead.bev_nms(boxes, scores, thr, 2)
    cb, cc = oracle_ops.bev_nms(boxes, scores, thr, 2)
    assert (nc == np.repeat([1, 2], len(a))).all()
    bad = np.flatnonzero(nc != cc)
    assert not len(bad), "numpy and C oracles decide %d of %d boundary positions differently, e.g. %r" % (
        len(bad), len(nc), boxes[bad[:3]].tolist())
    np.testing.assert_array_equal(cb, nb)


@pytest.mark.parametrize("thr", [0.1, 0.5])
def test_boundary_decisions_are_faithful_to_exact_iou(thr):
    """At every boundary position the oracle's decision equals the exact comparison IoU > float32(thr) on the float32
    rectangles, unless the exact IoU lies within REL_BOUND of the threshold."""
    a, bs, bk = boundary_pairs(thr)
    ra, rs, rk = ohead.bev_rects(a), ohead.bev_rects(bs), ohead.bev_rects(bk)
    t = Fraction(float(F32(thr)))
    worst = Fraction(0)
    for i in range(len(a)):
        for r, suppressed in ((rs[i], True), (rk[i], False)):
            e = exact_iou(ra[i], r)
            if (e > t) != suppressed:
                assert near_threshold(e, thr), "pair %d: exact IoU %r vs threshold %r, decided %s" % (
                    i, float(e), float(t), suppressed)
                worst = max(worst, abs(e - t) / t)
    assert worst <= REL_BOUND


def test_bev_rects_recipe():
    """oracle/head.py:bev_rects is the recipe of DESIGN §3.5: cos / sin in double rounded once to float32, each product
    and sum rounded, half extents by multiplication with 0.5."""
    rng = np.random.default_rng(4)
    bx = np.concatenate([rng.uniform(-40, 70, (500, 3)), rng.uniform(0.1, 5, (500, 3)),
                         rng.uniform(-np.pi, np.pi, (500, 1))], -1).astype(np.float32)
    bx[:5, 6] = np.float32([0, np.pi / 2, -np.pi, np.pi / 4, 3 * np.pi / 4])
    r = ohead.bev_rects(bx)
    for i in range(len(bx)):
        x, z, l, w, ry = (float(v) for v in bx[i, [0, 2, 3, 5, 6]])
        c, s = abs(float(F32(math.cos(ry)))), abs(float(F32(math.sin(ry))))
        dimx = F32(F32(F32(l) * F32(c)) + F32(F32(w) * F32(s)))
        dimz = F32(F32(F32(w) * F32(c)) + F32(F32(l) * F32(s)))
        exp = [F32(x) - dimx * F32(0.5), F32(z) - dimz * F32(0.5), F32(x) + dimx * F32(0.5), F32(z) + dimz * F32(0.5)]
        np.testing.assert_array_equal(r[i], np.asarray(exp, np.float32))


@pytest.mark.parametrize("name", list(nms_scenes()))
def test_scenes_numpy_and_c_oracles_agree(oracle_ops, name):
    c = nms_scenes()[name]
    nb, nc = ohead.bev_nms(c["boxes"], c["scores"], c["thr"], c["max_out"], c["cls_id"])
    cb, cc = oracle_ops.bev_nms(c["boxes"], c["scores"], c["thr"], c["max_out"], c["cls_id"])
    np.testing.assert_array_equal(cc, nc)
    np.testing.assert_array_equal(cb, nb)


def test_chain_scenes_depend_on_the_boundary_decisions():
    """The chain scenes are only worth running if their boundary decisions reach the output: with every B moved from
    the suppress to the keep position, the kept set changes."""
    rng = np.random.default_rng(5)
    cells = grid_cells(40)
    a, b = pair_boxes(rng, boundary_angles(rng, 18), True, 0, centers=cells)
    a, bs, bk = bisect_pairs(a, b, 0, 0.1)
    out = []
    for bb in (bs, bk):
        c = follower(bb)
        g = len(a)
        sc = np.concatenate([np.full(g, 0.9), np.full(g, 0.8), np.full(g, 0.7)])
        out.append(ohead.bev_nms(np.concatenate([a, bb, c])[None], sc[None].astype(np.float32), 0.1, 3 * g))
    (b0, c0), (b1, c1) = out
    assert (c0 == c1).all()                  # per group: A and C kept, or A and B kept
    assert (b0[0, :len(a)] == b1[0, :len(a)]).all()
    assert (b0[0, len(a):c0[0]] != b1[0, len(a):c1[0]]).any(-1).all()


def test_signed_zero_scores_tie_to_lower_index():
    """±0 scores are equal: the lower index goes first, whatever the sign."""
    boxes = np.zeros((1, 4, 7), np.float32)
    boxes[0, :, 3:6] = 1.0
    boxes[0, :, 0] = [0.0, 0.1, 10.0, 10.1]
    scores = np.array([[0.0, -0.0, -0.0, 0.0]], np.float32)
    blk, cnt = ohead.bev_nms(boxes, scores, 0.1, 4)
    assert cnt.tolist() == [2]
    np.testing.assert_array_equal(blk[0, :2, 0], [0.0, 10.0])
