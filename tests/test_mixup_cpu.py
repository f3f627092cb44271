"""The mixup twin (oracle/mixup.py) against the reference's own database, collision test, sampler, plane reader and
mixup-on kitti_forward (tests/golden/mixup.npz, tests/golden/make_golden_mixup.py), the stateless sampler, the host
checks and the C-boundary calls of the mixup wrappers."""
import importlib
import os

import numpy as np
import pytest
import torch

from oracle import augment as OA
from oracle import mixup as OM
from test_tf_ops_abi_cpu import _Recorder, abi  # noqa: F401  (abi is a fixture)

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "mixup.npz")
FACE_TOL = 1e-4            # metres: points this close to a face may fall on either side of a float32 plane
COORD_TOL = 2e-4           # metres, as for the augmentation golden
MX = importlib.import_module("3dssd_b200.mixup")
IO = importlib.import_module("3dssd_b200.kitti_io")


def golden_db(z):
    return OM.build_db(z["db_frame_points"], z["db_frame_offsets"], z["db_frame_boxes"], z["db_frame_labels"])


def golden_draws(z, total):
    return (z["scene_u"], z["loc_noise"], z["rot_u"], z["keys"][:total], z["refill"])


@pytest.fixture(scope="module")
def golden():
    z = dict(np.load(GOLDEN))
    return z, golden_db(z)


def test_database_equals_the_reference(golden):
    """Membership, counts, order and the 4- / 5-point edge: the objects of generate_mixup_sample, Car only."""
    z, db = golden
    assert np.array_equal(db["offsets"], z["ref_db_offsets"])
    assert np.array_equal(np.stack([db["frames"], db["rows"]], 1), z["ref_db_src"])
    assert np.array_equal(db["boxes"], z["ref_db_boxes"])
    assert np.array_equal(db["points"], z["ref_db_points"])
    c = db["counts"]
    assert (c == 4).any() and (c == 5).any()                               # the four-point object is not in the database
    m = OM.members(z["db_frame_points"][z["db_frame_offsets"][1]:z["db_frame_offsets"][2]], z["db_frame_boxes"][1])
    assert (m[0] & m[1]).any()                                             # a point shared by two objects


def test_collision_outcomes_equal_the_reference(golden):
    z, db = golden
    pts, off = z["points"], z["offsets"]
    _, _, _, _, _, acc = OM.paste(pts, off, z["sem_labels"], z["gt_boxes"], z["gt_labels"], z["ids"], db, z["ref_planes"])
    assert np.array_equal(acc, z["ref_accepted"])
    drawn = z["ids"] >= 0
    assert (acc[drawn] == 0).any() and (acc[drawn] == 1).any()
    assert any(drawn[s].any() and not acc[s].any() for s in range(len(acc)))        # every drawn object dropped
    assert (~OA.valid_rows(z["gt_boxes"])).all(1).any()                                # a scene without rows


def test_planes_equal_the_reference(golden, tmp_path):
    z, _ = golden
    for i, text in enumerate(z["plane_texts"]):
        (tmp_path / ("%06d.txt" % i)).write_text(str(text))
        got = IO.read_plane(IO.plane_path(str(tmp_path), i))
        assert got.dtype == np.float64 and np.array_equal(got, z["ref_planes"][i]), i
    assert (z["plane_rows"][:, 1] > 0).any() and (np.abs(z["ref_planes"][:, [0, 2]]) > 0).any()
    with pytest.raises(FileNotFoundError, match="000099.txt"):
        IO.read_plane(IO.plane_path(str(tmp_path), 99))


def test_stateless_sampler_equals_the_recorded_sequence(golden):
    z, _ = golden
    count, num = int(z["sampler_count"]), int(z["sampler_num"])
    sizes = z["sampler_ret_sizes"]
    rets = np.split(z["sampler_rets"], np.cumsum(sizes)[:-1])
    assert count % num and len(rets) >= 3 * int(np.ceil(count / num)) and (sizes < num).any()
    for k, r in enumerate(rets):
        e, a, b = MX.Sampler.cursor(count, num, k)
        assert np.array_equal(z["sampler_perms"][e][a:b], r), k


def test_sampler_ids():
    class DB:
        def class_ids(self, c):
            return np.arange(37) * 2 if c == 1 else np.zeros(0, np.int64)
    s = MX.Sampler(DB(), seed=4)
    a = s.ids(2, 3, rank=1)
    assert a.shape == (3, 15) and a.dtype == np.int32 and np.array_equal(a, s.ids(2, 3, rank=1))
    assert (a[:, :7] >= 0).all() and (a[:, 7:] == -1).all()                 # call 2 of 3 per epoch: the 7-object tail
    seen = np.concatenate([s.ids(k, 1)[0] for k in range(3)])
    assert np.array_equal(np.sort(seen[seen >= 0]), np.arange(37) * 2)       # one epoch draws every object once
    assert not np.array_equal(s.ids(0, 2)[0], s.ids(0, 2)[1])
    e = MX.Sampler(DB(), classes=(2,), numbers=(15,))
    assert (e.ids(0, 2) == -1).all()


def test_twin_chain_equals_the_mixup_on_reference(golden):
    """kitti_forward with mixup on: the twin's survivors and coordinates (points near a face excepted)."""
    z, db = golden
    pts, off = z["points"], z["offsets"]
    _, poff, _, _, _, _ = OM.paste(pts, off, z["sem_labels"], z["gt_boxes"], z["gt_labels"], z["ids"], db, z["ref_planes"])
    block, ob, ol, rec = OM.augment(pts, off, z["sem_labels"], z["gt_boxes"], z["gt_labels"], z["ids"], db, z["ref_planes"],
                                    golden_draws(z, int(poff[-1])), 1024)
    roff = z["ref_offsets"]
    for s in range(len(off) - 1):
        sl = slice(poff[s], poff[s + 1])
        kept = np.zeros(poff[s + 1] - poff[s], bool)
        idx = z["ref_index"][roff[s]:roff[s + 1]]
        kept[idx] = True
        got = rec["sort_keys"][sl] != OA.ALL_ONES
        near = np.zeros_like(kept)
        valid = OA.valid_rows(ob[s])
        for b in ob[s][valid].astype(np.float64):
            l, h, w = b[3] + 0.5, b[4] + 2.0, b[5] + 0.5
            c, sn = np.cos(b[6]), np.sin(b[6])
            e = rec["points"][sl][:, :3].astype(np.float64) - b[:3]
            cx, cy, cz = c * e[:, 0] - sn * e[:, 2], e[:, 1], sn * e[:, 0] + c * e[:, 2]
            near |= np.min(np.abs(np.stack([cx - l / 2, cx + l / 2, cy, cy + h, cz - w / 2, cz + w / 2], 1)), 1) < FACE_TOL
        assert np.array_equal(got[~near], kept[~near]), s
        assert (rec["pasted_sem"][sl][got] >= 0).all()                          # no absent slot survives
        mine = rec["points"][sl][idx]
        ok = ~near[idx]
        assert np.abs(mine[ok] - z["ref_points"][roff[s]:roff[s + 1]][ok]).max(initial=0) <= COORD_TOL, s
        rows = int(valid.sum())
        assert np.abs(ob[s][:rows] - z["ref_boxes"][s][:rows]).max(initial=0) <= COORD_TOL, s


def test_host_checks_raise(abi):  # noqa: F811
    off = np.array([0, 100, 250])
    dbo = np.array([0, 10, 30, 60], np.int64)
    ids = np.array([[0, 2, -1], [1, -1, -1]], np.int32)
    lay = MX.layout(off, ids, dbo, 4)
    assert lay.rows == 7 and lay.total == 250 + 40 + 20 and lay.max_slots == 150 + 20
    assert np.array_equal(lay.slot_start, [[100, 110, 140, 140], [150, 170, 170, 170]])
    with pytest.raises(ValueError):
        MX.layout(off, np.array([[0, 3, -1], [1, -1, -1]]), dbo, 4)          # id out of range
    with pytest.raises(ValueError):
        MX.layout(off, np.array([[0, -2, -1], [1, -1, -1]]), dbo, 4)
    with pytest.raises(ValueError):
        MX.layout(np.array([0, 131070, 131080]), ids, dbo, 4)               # a scene over 131072 slots
    assert MX.layout(np.array([0, 131032, 131080]), ids, dbo, 4).max_slots == 131072
    with pytest.raises(ValueError):
        MX.layout(off, ids, dbo, 254)                                        # G + S > 256
    with pytest.raises(ValueError):
        MX.check_planes(np.array([[0, 0, 0, 1.65], [0, -1, 0, 1.65]]), 2)    # b = 0
    with pytest.raises(ValueError):
        MX.check_planes(np.array([[0, -1, 0, np.nan], [0, -1, 0, 1.65]]), 2)
    T, fake = abi
    f = lambda *s: torch.zeros(s, dtype=torch.float32)
    i = lambda *s: torch.zeros(s, dtype=torch.int32)
    d = lambda *s: torch.zeros(s, dtype=torch.float64)
    L = lambda *s: torch.zeros(s, dtype=torch.int64)
    bad = [lambda: T.mixup_db_count(f(30, 4), i(3), 20, f(2, 0, 7)),
           lambda: T.mixup_db_count(f(30, 4), i(3), 20, f(3, 4, 7)),
           lambda: T.mixup_db_write(f(30, 4), i(3), f(2, 4, 7), i(5, 2), L(5), 10),
           lambda: T.mixup_paste_boxes(f(2, 250, 7), i(2, 250), i(2, 15), f(9, 7), i(9), d(2, 4)),
           lambda: T.mixup_paste_boxes(f(2, 4, 7), i(2, 4), i(2, 15), f(9, 7), i(8), d(2, 4)),
           lambda: T.mixup_paste_boxes(f(2, 4, 7), i(2, 4), i(2, 15), f(9, 7), i(9), f(2, 4)),
           lambda: T.mixup_paste_points(f(30, 4), i(3), i(30), i(2, 15), f(50, 4), L(9), f(9, 7), i(9), d(2, 4), i(2, 15), i(3),
                                        i(2, 16), 40, 80),
           lambda: T.mixup_paste_points(f(30, 4), i(3), i(30), i(2, 15), f(50, 4), L(10), f(9, 7), i(9), d(2, 4), i(2, 15), i(3),
                                        i(2, 15), 40, 80)]
    for k, call in enumerate(bad):
        fake.calls.clear()
        with pytest.raises(ValueError):
            call()
        assert not fake.calls, k


def test_wrapper_abi_trace(abi):  # noqa: F811
    """The entry points, scalars and pointer placements of the mixup wrappers."""
    T, fake = abi
    rec = _Recorder(fake)
    f = lambda *s: torch.zeros(s, dtype=torch.float32)
    i = lambda *s: torch.zeros(s, dtype=torch.int32)
    d = lambda *s: torch.zeros(s, dtype=torch.float64)
    L = lambda *s: torch.zeros(s, dtype=torch.int64)
    pts, off = f(30, 4), i(3)
    rec("count", T.mixup_db_count, pts, off, 20, f(2, 4, 7))
    rec("write", T.mixup_db_write, pts, off, f(2, 4, 7), i(5, 2), L(6), 44)
    rec("boxes", T.mixup_paste_boxes, f(2, 4, 7), i(2, 4), i(2, 15), f(9, 7), i(9), d(2, 4))
    rec("points", T.mixup_paste_points, pts, off, i(30), i(2, 15), f(50, 4), L(10), f(9, 7), i(9), d(2, 4), i(2, 15), i(3),
        i(2, 16), 40, 80)
    t = rec.trace
    assert t["count"][0]["calls"] == [["ssd3d_mixup_db_count", 2, 4, 20, ["a.0", 0], ["a.1", 0], ["a.3", 0], ["r", 0], "stream"]]
    assert t["count"][0]["returns"][0][1:3] == [[2, 4], "torch.int32"]
    assert t["write"][0]["calls"] == [["ssd3d_mixup_db_write", 4, 5, ["a.0", 0], ["a.1", 0], ["a.2", 0], ["a.3", 0], ["a.4", 0],
                                       ["r", 0], "stream"]]
    assert t["write"][0]["returns"][0][1:3] == [[44, 4], "torch.float32"]
    assert t["boxes"][0]["calls"] == [["ssd3d_mixup_paste_boxes", 2, 4, 15, ["a.0", 0], ["a.1", 0], ["a.2", 0], ["a.3", 0], ["a.4", 0],
                                       ["a.5", 0], ["r.0", 0], ["r.1", 0], ["r.2", 0], "stream"]]
    assert [r[1:3] for r in t["boxes"][0]["returns"]] == [[[2, 19, 7], "torch.float32"], [[2, 19], "torch.int32"],
                                                          [[2, 15], "torch.int32"]]
    assert t["points"][0]["calls"] == [["ssd3d_mixup_paste_points", 2, 15, 40] + [["a.%d" % k, 0] for k in range(12)] +
                                       [["r.0", 0], ["r.1", 0], "stream"]]
    assert [r[1:3] for r in t["points"][0]["returns"]] == [[[80, 4], "torch.float32"], [[80], "torch.int32"]]
