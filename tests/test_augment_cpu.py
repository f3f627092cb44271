"""The augmentation's numpy twin (oracle/augment.py) against the reference's own kitti_forward run on recorded draws
(tests/golden/augment.npz, tests/golden/make_golden_augment.py), the point-choice rule, the draw block, the host checks
and the C-boundary calls of the tf_ops wrappers."""
import importlib
import os

import numpy as np
import pytest
import torch

from oracle import augment as OA
from test_tf_ops_abi_cpu import _QUERIES, _Recorder, abi  # noqa: F401  (abi is a fixture)

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "augment.npz")
FACE_TOL = 1e-4            # metres: points this close to a face may fall on either side of a float32 plane
COORD_TOL = 2e-4           # metres: float32 rounding of a float64 chain over coordinates up to ~70 m
A = importlib.import_module("3dssd_b200.augment")


def golden_inputs():
    """[(points, offsets, sem_labels, gt_boxes, gt_labels, draws, num_points)] of the golden scenes."""
    z = np.load(GOLDEN)
    draws = (z["scene_u"], z["loc_noise"], z["rot_u"], z["keys"], z["refill"])
    return [(z["points"], z["offsets"], z["sem_labels"], z["gt_boxes"], z["gt_labels"], draws, z["refill"].shape[1])]


@pytest.fixture(scope="module")
def golden():
    z = dict(np.load(GOLDEN))
    pts, off, sem, boxes, labels, draws, m = golden_inputs()[0]
    block, ob, rec = OA.augment(pts, off, sem, boxes, labels, draws, m)
    return z, ob, rec


def _final_face_distance(pts, boxes):
    """float64 distance of each point to the nearest face of the boxes grown by (0.5, 2, 0.5)."""
    best = np.full(len(pts), np.inf)
    for b in boxes[OA.valid_rows(boxes)].astype(np.float64):
        l, h, w = b[3] + 0.5, b[4] + 2.0, b[5] + 0.5
        c, s = np.cos(b[6]), np.sin(b[6])
        e = pts[:, :3].astype(np.float64) - b[:3]
        cx, cy, cz = c * e[:, 0] - s * e[:, 2], e[:, 1], s * e[:, 0] + c * e[:, 2]
        best = np.minimum(best, np.min(np.abs(np.stack([cx - l / 2, cx + l / 2, cy, cy + h, cz - w / 2, cz + w / 2], 1)), 1))
    return best


def test_golden_covers_its_cases(golden):
    z, _, _ = golden
    u, ch = z["scene_u"], z["ref_chosen"]
    assert (u[:, :4] == 0.5).any()
    assert (ch == 0).any() and (ch == 99).any() and (ch[OA.valid_rows(z["gt_boxes"])] == -1).any()
    assert (~OA.valid_rows(z["gt_boxes"])).all(1).any()                     # a scene without boxes
    ry = z["gt_boxes"][..., 6]
    assert (ry == np.float32(np.pi)).any() and (ry == np.float32(-np.pi)).any() and (ry[OA.valid_rows(z["gt_boxes"])] == 0).any()
    m = z["ref_moved_by"]
    assert (m >= 0).any()


def test_discrete_outcomes_equal_the_reference(golden):
    """Chosen try per box (up to the first box whose float32 and float64 searches differ), the box that moves each
    point (exhausted boxes excepted, see below), which points survive and padded rows untouched."""
    z, ob, rec = golden
    off, roff = z["offsets"], z["ref_offsets"]
    for s in range(len(off) - 1):
        valid = OA.valid_rows(z["gt_boxes"][s])
        ref, ref64, got = z["ref_chosen"][s][valid], z["ref_chosen64"][s][valid], rec["chosen"][s][valid]
        tie = np.flatnonzero(ref != ref64)
        upto = tie[0] if tie.size else len(ref)
        assert np.array_equal(got[:upto], ref[:upto]), (s, got, ref)
        assert np.all(ob[s][~valid] == 0), s
        sl = slice(off[s], off[s + 1])
        near = z["face_dist"][sl] < FACE_TOL
        near |= _final_face_distance(rec["points"][sl], ob[s]) < FACE_TOL
        exhausted = [j for j in np.flatnonzero(valid) if z["ref_chosen"][s][j] < 0]
        if z["scene_u"][s, 1] <= 0.5 and exhausted:                        # the reference filters around a zero-size box
            grown = ob[s][exhausted].copy()
            grown[:, 3:6] += OA.GROW[0], OA.GROW[1], OA.GROW[2]
            n, d = OA.planes(grown, np.float32(0))
            p = rec["points"][sl]
            for k in range(len(grown)):
                near |= OA.inside(p[:, 0], p[:, 1], p[:, 2], n[k], d[k])
        ref_mv = z["ref_moved_by"][sl].copy()
        ref_mv[np.isin(ref_mv, exhausted)] = -1                             # a failed box moves nothing here
        assert np.array_equal(rec["moved_by"][sl][~near], ref_mv[~near]), s
        kept = np.zeros(off[s + 1] - off[s], bool)
        kept[z["ref_index"][roff[s]:roff[s + 1]]] = True
        got_kept = rec["sort_keys"][sl] != OA.ALL_ONES
        assert np.array_equal(got_kept[~near], kept[~near]), s


def test_coordinates_equal_the_reference(golden):
    z, ob, rec = golden
    off, roff = z["offsets"], z["ref_offsets"]
    for s in range(len(off) - 1):
        valid = OA.valid_rows(z["gt_boxes"][s])
        good = valid & (z["ref_chosen"][s] >= 0) | ~valid
        if z["scene_u"][s, 1] > 0.5:
            good[:] = True
        assert np.abs(ob[s][good] - z["ref_boxes"][s][good]).max(initial=0) <= COORD_TOL, s
        idx = z["ref_index"][roff[s]:roff[s + 1]]
        refp = z["ref_points"][roff[s]:roff[s + 1]]
        mine = rec["points"][off[s]:off[s + 1]][idx]
        exhausted = [j for j in np.flatnonzero(valid) if z["ref_chosen"][s][j] < 0]
        collapsed = np.isin(z["ref_moved_by"][off[s]:off[s + 1]][idx], exhausted)
        assert np.abs(mine[~collapsed] - refp[~collapsed]).max(initial=0) <= COORD_TOL, s


def test_exhausted_box_diverges_from_the_reference_as_documented(golden):
    """All 100 tries of a box collide: the reference's _select_transform gives it scale 0, which zeroes its dims and
    collapses its points onto its centre; here it keeps the identity transform."""
    z, ob, rec = golden
    off, roff = z["offsets"], z["ref_offsets"]
    seen = 0
    for s in range(len(off) - 1):
        if z["scene_u"][s, 1] > 0.5:
            continue
        for j in np.flatnonzero(OA.valid_rows(z["gt_boxes"][s]) & (z["ref_chosen"][s] < 0)):
            seen += 1
            assert np.all(z["ref_boxes"][s, j, 3:6] == 0)                    # the reference: dims zeroed
            assert np.all(ob[s, j, 3:6] > 1.0)                               # here: the box keeps its size
            members = np.flatnonzero(z["ref_moved_by"][off[s]:off[s + 1]] == j)
            row = np.full(off[s + 1] - off[s], -1)
            row[z["ref_index"][roff[s]:roff[s + 1]]] = np.arange(roff[s + 1] - roff[s])
            assert members.size and np.all(row[members] >= 0)                # positives are never filtered
            refp = z["ref_points"][roff[s]:roff[s + 1]][row[members]]
            assert np.abs(refp[:, [0, 2]] - z["ref_boxes"][s, j, [0, 2]]).max(initial=0) <= COORD_TOL   # collapsed onto the centre
            assert np.all(rec["moved_by"][off[s]:off[s + 1]][members] == -1)                     # here: not moved
    assert seen >= 1


@pytest.mark.parametrize("n", [20000, 16384, 5000, 1])
def test_choice_rule(n):
    rng = np.random.default_rng(n)
    m = 16384
    pts = rng.standard_normal((n + 7, 4)).astype(np.float32)
    keys = rng.integers(0, 2 ** 32, n + 7).astype(np.uint64)
    keys[:3] = keys[3]                                                       # equal keys: the index breaks the tie
    sk = (keys << np.uint64(32)) | np.arange(n + 7, dtype=np.uint64)
    sk[n:] = OA.ALL_ONES                                                     # dropped by the filter
    refill = rng.integers(0, 2 ** 32, m).astype(np.uint32).view(np.int32)
    out = OA.choose(pts, sk, refill)
    order = np.argsort(sk[:n], kind="stable")                                # (key, index) order of the survivors
    k = min(n, m)
    assert np.array_equal(out[:k], pts[order[:k]])
    if n < m:
        r = (refill[n:].view(np.uint32).astype(np.uint64) * np.uint64(n)) >> np.uint64(32)
        assert np.array_equal(out[n:], pts[order[r.astype(np.int64)]])
    else:
        assert len(np.unique(order[:k])) == k


def test_draws_for_a_fixed_seed():
    gen = torch.Generator().manual_seed(A.draw_seed(3, 10, 1))
    d = A.draw(4, 20, 50000, 16384, gen, "cpu")
    assert d.scene_u.shape == (4, 6) and d.loc_noise.shape == (4, 20, 100, 2) and d.rot_u.shape == (4, 20, 100)
    assert d.keys.shape == (50000,) and d.refill.shape == (4, 16384) and d.keys.dtype == torch.int32
    assert d.scene_u.dtype == d.loc_noise.dtype == d.rot_u.dtype == torch.float64
    ln = d.loc_noise.numpy()
    assert abs(ln.mean()) < 0.02 and abs(ln.std() - 1) < 0.02
    ru = d.rot_u.numpy()
    assert ru.min() >= 0 and ru.max() < 1 and abs(ru.mean() - 0.5) < 0.02
    k = d.keys.numpy().view(np.uint32).astype(np.float64) / 2 ** 32
    assert abs(k.mean() - 0.5) < 0.01 and k.min() < 0.01 and k.max() > 0.99
    again = A.draw(4, 20, 50000, 16384, torch.Generator().manual_seed(A.draw_seed(3, 10, 1)), "cpu")
    assert all(torch.equal(a, b) for a, b in zip(d, again))
    assert A.draw_seed(3, 10, 1) != A.draw_seed(3, 10, 0) != A.draw_seed(3, 11, 0)


def test_host_checks_raise_before_any_launch(abi):  # noqa: F811
    T, fake = abi
    ok_off = np.array([0, 10, 30])
    with pytest.raises(ValueError):
        A.check_scenes(np.array([0, 10, 10]))                               # an empty scene
    with pytest.raises(ValueError):
        A.check_scenes(np.array([0, 131073]))
    with pytest.raises(ValueError):
        A.check_scenes(ok_off, g=257)
    with pytest.raises(ValueError):
        A.check_scenes(ok_off, np.r_[np.zeros(29, np.int32), -1])
    with pytest.raises(ValueError):
        A.Augmentor(16385)
    assert A.check_scenes(ok_off, np.zeros(30, np.int32), 256) == 20
    f = lambda *s: torch.zeros(s, dtype=torch.float32)
    d = lambda *s: torch.zeros(s, dtype=torch.float64)
    i = lambda *s: torch.zeros(s, dtype=torch.int32)
    off = i(3)
    bad = [lambda: T.augment_sem_labels(f(30, 3), off, f(2, 4, 7), i(2, 4), 20),
           lambda: T.augment_sem_labels(f(30, 4), off, f(2, 4, 7), i(2, 4), 131073),
           lambda: T.augment_sem_labels(f(30, 4), off, f(3, 4, 7), i(3, 4), 20),
           lambda: T.augment_boxes(f(2, 257, 7), d(2, 6), d(2, 257, 100, 2), d(2, 257, 100)),
           lambda: T.augment_boxes(f(2, 4, 7), d(2, 6), d(2, 4, 99, 2), d(2, 4, 100)),
           lambda: T.augment_boxes(f(2, 4, 7), f(2, 6), d(2, 4, 100, 2), d(2, 4, 100)),
           lambda: T.augment_points(f(30, 4), off, 20, i(29), i(30), torch.zeros(10000, dtype=torch.uint8), 4),
           lambda: T.augment_choose(f(30, 4), off, torch.zeros(30, dtype=torch.int64), i(2), i(2, 16385)),
           lambda: T.augment_choose(f(30, 4), i(4), torch.zeros(30, dtype=torch.int64), i(2), i(2, 64))]
    for k, call in enumerate(bad):
        fake.calls.clear()
        with pytest.raises(ValueError):
            call()
        assert not fake.calls, k


def test_wrapper_abi_trace(abi, monkeypatch):  # noqa: F811
    """The entry points, scalars and pointer placements of the augment wrappers."""
    T, fake = abi
    monkeypatch.setitem(_QUERIES, "ssd3d_augment_workspace", lambda b, g: 512 * b + 64 * g)
    rec = _Recorder(fake)
    f = lambda *s: torch.zeros(s, dtype=torch.float32)
    i = lambda *s: torch.zeros(s, dtype=torch.int32)
    d = lambda *s: torch.zeros(s, dtype=torch.float64)
    pts, off = f(30, 4), i(3)
    rec("sem", T.augment_sem_labels, pts, off, f(2, 4, 7), i(2, 4), 20)
    _, _, ws = rec("boxes", T.augment_boxes, f(2, 4, 7), d(2, 6), d(2, 4, 100, 2), d(2, 4, 100))
    rec("points", T.augment_points, pts, off, 20, i(30), i(30), ws, 4, want_moved=True)
    rec("points_nomove", T.augment_points, pts, off, 20, i(30), i(30), ws, 4)
    rec("choose", T.augment_choose, pts, off, torch.zeros(30, dtype=torch.int64), i(2), i(2, 64))
    t = rec.trace
    assert [c[0] for c in t["sem"][0]["calls"]] == ["ssd3d_augment_sem_labels"]
    assert t["sem"][0]["calls"][0][1:] == [2, 4, 20, ["a.0", 0], ["a.1", 0], ["a.2", 0], ["a.3", 0], ["r", 0], "stream"]
    assert [c[0] for c in t["boxes"][0]["calls"]] == ["ssd3d_augment_workspace", "ssd3d_augment_boxes"]
    assert t["boxes"][0]["calls"][1][1:] == [2, 4, ["a.0", 0], ["a.1", 0], ["a.2", 0], ["a.3", 0], ["r.0", 0], ["r.1", 0],
                                             ["r.2", 0], "stream"]
    assert t["boxes"][0]["returns"][2][1:3] == [[512 * 2 + 64 * 4], "torch.uint8"]
    assert t["points"][0]["calls"][-1][1:] == [2, 4, 20, ["a.0", 0], ["a.1", 0], ["a.3", 0], ["a.4", 0], ["a.5", 0], ["r.0", 0],
                                               ["r.1", 0], ["r.2", 0], ["r.3", 0], "stream"]
    assert t["points_nomove"][0]["calls"][-1][12] == 0                        # moved_by NULL
    assert t["choose"][0]["calls"][0][1:] == [2, 64, ["a.0", 0], ["a.1", 0], ["a.2", 0], ["a.3", 0], ["a.4", 0], ["r", 0], "stream"]
    assert [r[1:3] for r in t["choose"][0]["returns"]] == [[[2, 64, 4], "torch.float32"]]
