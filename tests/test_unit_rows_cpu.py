"""Unit lists of 4-row units without a GPU: the lists the CPU model of the culled ball query implies at 4 rows per unit,
the checks that reject a width before any launch, and the widths the route plan gives the 3DSSD scales."""
import ctypes
import importlib

import numpy as np
import pytest
import torch


def _units(cnt, k, w):
    """The list of w-row units a ball query with these counts builds, in group order: ceil(min(cnt, k) / w) per group"""
    return [(g << 4) | j for g in range(cnt.size) for j in range((min(int(cnt[g]), k) + w - 1) // w)]


@pytest.mark.parametrize("dilated,lows,highs,ks", [
    (False, [0.0, 0.0], [0.4, 0.8], [16, 64]),
    (True, [0.0, 0.4, 0.8], [0.4, 0.8, 1.6], [32, 32, 64]),
])
def test_model_lists_at_4_rows_cover_the_same_rows(oracle_ops, dilated, lows, highs, ks):
    """From the CPU model's counts (oracle bq_grid_model, the culled kernel's restatement): a group's 4-row units are
    ceil(cnt / 4) units that together cover rows 0 .. 4 ceil(cnt / 4) - 1; every row they add beyond cnt repeats the first
    hit, so the max over them equals the max over the 8-row units and over all nsample rows."""
    rng = np.random.default_rng(7)
    xyz1 = np.concatenate([rng.normal(0, 0.3, (2, 300, 3)) + 5.0, rng.uniform(0, 20, (2, 1700, 3))], 1).astype(np.float32)
    xyz2 = np.ascontiguousarray(xyz1[:, ::10])
    idx, cnt, units8, _ = oracle_ops.query_ball_point_grid_model(lows, highs, ks, xyz1, xyz2, dilated)
    for s, k in enumerate(ks):
        c = np.asarray(cnt[s]).reshape(-1)
        ix = np.asarray(idx[s]).reshape(c.size, k)
        u8 = np.asarray(units8[s])
        assert sorted(u8[1:1 + int(u8[0])].tolist()) == _units(c, k, 8)        # the model's own 8-row lists
        u4 = _units(c, k, 4)
        per = {}
        for d in u4:
            per.setdefault(d >> 4, []).append(d & 15)
        assert sorted(per) == np.flatnonzero(c > 0).tolist()
        for g, js in per.items():
            n = min(int(c[g]), k)
            assert sorted(js) == list(range((n + 3) // 4))
            rows = [4 * j + e for j in js for e in range(4)]
            assert rows == list(range(4 * ((n + 3) // 4)))
            assert set(ix[g, rows].tolist()) == set(ix[g, :n].tolist()) == set(ix[g].tolist())
        assert len(u4) <= len(_units(c, k, 8)) * 2 and 4 * len(u4) <= 8 * len(_units(c, k, 8))


class _NoLib:
    def __getattr__(self, name):
        raise AssertionError("%s reached the library" % name)


def test_bad_widths_are_rejected_before_any_launch(pkg, monkeypatch):
    T = pkg.tf_ops
    monkeypatch.setattr(T, "lib", lambda: _NoLib())
    monkeypatch.setattr(T, "_bq_shapes", lambda a, b: (a, b))
    monkeypatch.setattr(T, "_req", lambda t, *a, **k: t)                  # CPU tensors stand in for device ones
    x1, x2 = torch.zeros((1, 64, 3)), torch.zeros((1, 8, 3))
    for rows, ks in (([4], [128]), ([4], [96]), ([2], [16]), ([16], [16]), ([8, 3], [16, 16])):
        with pytest.raises(ValueError):
            T.query_ball_point_multi([0.0] * len(ks), [0.4] * len(ks), ks, x1, x2, False, return_units=True, unit_rows=rows)
    units = torch.zeros((25,), dtype=torch.int32)
    with pytest.raises(ValueError):
        T._units_check(units, False, unit_rows=6)
    with pytest.raises(ValueError):
        T._units_check(units, False, unit_rows=4, ns=128)
    units.unit_rows = 4
    assert T._units_check(units, False) == 4 and T._units_check(units, False, unit_rows=8) == 8
    assert T._units_check(torch.zeros((25,), dtype=torch.int32), False) == 8
    with T.unit_rows([4]):
        with pytest.raises(ValueError):                        # the block's width checked against the shell's nsample
            T.query_ball_point_multi([0.0], [0.4], [128], x1, x2, False, return_units=True)


def test_c_entry_points_reject_bad_widths(pkg):
    L = pkg.lib()
    null, one = ctypes.c_void_p(None), ctypes.c_void_p(16)
    err = lambda: L.ssd3d_last_error().decode()
    assert L.ssd3d_linear_tc_units_ex(1024, 64, 32, one, one, one, one, one, one, 1, one, 0, one, 32, null, null, 0, null, 6) == -1
    assert "unit_rows" in err()
    assert L.ssd3d_linear_tc_hoisted_units_ex(1, 64, 32, 8, 128, one, one, 32, one, one, one, one, 32, one, one, one, one, 1, 0,
                                              one, 32, null, null, 0, null, 4) == -1 and "unit_rows" in err()
    assert L.ssd3d_hoist_expand_split_units_ex(1, 64, 32, 8, 96, one, one, 32, one, one, one, one, one, one, 32, null, 4) == -1
    ks = (ctypes.c_int * 1)(128)
    rad = (ctypes.c_float * 1)(0.4)
    ptr = (ctypes.c_void_p * 1)(16)
    w4 = (ctypes.c_int * 1)(4)
    cast = lambda a: ctypes.cast(a, ctypes.c_void_p)
    assert L.ssd3d_query_ball_point_multi_ws_ex(1, 64, 8, 1, 0, cast(rad), cast(rad), cast(ks), one, one, cast(ptr), cast(ptr),
                                                cast(ptr), null, 0, null, cast(w4)) == -1 and "nsample <= 64" in err()


def test_route_plan_gives_every_3dssd_scale_4_row_units(pkg):
    """Every scale of the four SA layers (nsample 16-64) takes its unit list at 4 rows per unit."""
    lu = importlib.import_module("3dssd_b200.layers_util")
    P = pkg.params
    arch = pkg.config.ARCH_3DSSD
    pp = P.prepare(P.init_params(arch, 1, seed=0), "cpu")
    assert lu.UNIT_ROWS == 4
    seen = 0
    for spec, c_feat in zip([arch[0], arch[1], arch[2], arch[5]], [1, 64, 128, 256]):
        nsample, mlp, scope = spec[3], spec[4], spec[12]
        plan = lu._route_plan(pp, scope, nsample, mlp, True, c_feat, spec[15] not in (None, -1), "tc", True, True, 2)
        assert plan.compact
        for sc, k in zip(plan.scales, nsample):
            assert sc.units and k <= 64 and sc.unit_rows == 4
            seen += 1
    assert seen == 11
