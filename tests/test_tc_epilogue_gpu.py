"""The epilogue of linear_tc_kernel (scale/shift/ReLU on the wgmma accumulator fragments, then stores or max-pools) at
the shapes the benchmark does not reach: every pooling width, unit lists that end inside a tile, row counts and widths
that are not multiples of the tile, every output combination, the gather route, and concurrent launches.

Operands are small dyadic numbers, so every product and every fp32 partial sum is exact: the kernel's results must equal
the float64 evaluation of hi.W_hi + lo.W_hi + hi.W_lo, fmaf(acc, scale, shift), ReLU and the pool bit for bit."""
import importlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _layer(cin, cout, seed):
    """A folded conv whose weights need both bf16 terms (w = integer + k/256) and power-of-two scales, dyadic shifts."""
    P = importlib.import_module("3dssd_b200.params")
    rng = np.random.default_rng(seed)
    w = rng.integers(-2, 3, (cin, cout)) + rng.integers(-3, 4, (cin, cout)) / 256.0
    scale = rng.choice([0.25, 0.5, 1.0, -0.5], cout)
    shift = rng.integers(-16, 17, cout) / 16.0
    return P.FoldedConv(*(torch.tensor(a, dtype=torch.float32, device="cuda") for a in (w, scale, shift)))


def _operand(lead, f, seed):
    """bf16 (hi, lo) operand with zero K padding: hi integers in [-3, 3], lo multiples of 1/16."""
    rng = np.random.default_rng(seed)
    shape = tuple(lead) + (f.kp,)
    hi = rng.integers(-3, 4, shape).astype(np.float64)
    lo = rng.integers(-1, 2, shape) / 16.0
    hi[..., f.cin:] = 0
    lo[..., f.cin:] = 0
    return (torch.tensor(hi, dtype=torch.bfloat16, device="cuda"), torch.tensor(lo, dtype=torch.bfloat16, device="cuda"))


def _expect(a_hi, a_lo, f, relu=True):
    """float64 y = act(fma(a_hi.W_hi + a_lo.W_hi + a_hi.W_lo, scale, shift)), exact for these operands."""
    ah, al = (t.double().cpu().numpy() for t in (a_hi, a_lo))
    bh, bl = (t.double().cpu().numpy()[:, :f.kp] for t in (f.b_hi, f.b_lo))      # (cout, kp)
    acc = ah @ bh.T + al @ bh.T + ah @ bl.T
    y = acc * f.scale.double().cpu().numpy() + f.shift.double().cpu().numpy()
    assert np.array_equal(y.astype(np.float32).astype(np.float64), y), "test operands must keep the epilogue exact"
    return np.maximum(y, 0) if relu else y


def _split(y):
    """the kernel's split: hi = bf16_rn(y), lo = bf16_rn(y - hi)"""
    t = torch.tensor(y, dtype=torch.float32)
    hi = t.to(torch.bfloat16)
    return hi, (t - hi.float()).to(torch.bfloat16)


def _same(got, exp):
    assert torch.equal(got.cpu(), exp.cpu() if torch.is_tensor(exp) else torch.tensor(exp, dtype=got.dtype))


@pytest.mark.parametrize("pool", [8, 16, 32, 64, 128])
@pytest.mark.parametrize("cout", [24, 40, 64, 200])              # 24: the 32-column tile (linear_tc_kernel<32>)
def test_pool_every_width(pkg, cuda, pool, cout):
    b, m = 2, 13                                                   # b*m*pool rows: not a multiple of 128 for pool < 128
    f = _layer(67, cout, pool + cout)
    a_hi, a_lo = _operand((b, m, pool), f, pool)
    cnt = torch.tensor(np.random.default_rng(pool).integers(0, 3, (b, m)), dtype=torch.int32, device=cuda)
    y = _expect(a_hi, a_lo, f).max(axis=2) * (cnt.cpu().numpy() > 0)[..., None]
    f32 = torch.full((b, m, cout + 40), -7.0, device=cuda)
    sh = torch.zeros((b, m, cout + 40), dtype=torch.bfloat16, device=cuda)
    sl = torch.zeros_like(sh)
    pkg.linear_tc(a_hi, a_lo, f, pool=pool, rowmask=cnt, out_f32=(f32, 24), out_split=(sh, sl, 24))
    _same(f32[..., 24:24 + cout], y.astype(np.float32))
    assert (f32[..., :24] == -7.0).all() and (f32[..., 24 + cout:] == -7.0).all()
    eh, el = _split(y)
    _same(sh[..., 24:24 + cout], eh)
    _same(sl[..., 24:24 + cout], el)


@pytest.mark.parametrize("units_n", [1, 15, 16, 17, 47, 130])
@pytest.mark.parametrize("cout", [32, 72])
def test_unit_pool_lists_ending_mid_tile(pkg, cuda, units_n, cout):
    b, m, ns = 2, 40, 32
    rng = np.random.default_rng(units_n)
    f = _layer(48, cout, units_n)
    pairs = [(g, j) for g in range(b * m) for j in range(ns // 8)]
    pick = sorted(rng.choice(len(pairs), units_n, replace=False))
    units = torch.tensor([units_n] + [(pairs[i][0] << 4) | pairs[i][1] for i in pick], dtype=torch.int32, device=cuda)
    a_hi, a_lo = _operand((b, m, ns), f, units_n + 1)                 # rows past units_n * 8 are capacity, never read
    y = _expect(a_hi.reshape(-1, f.kp)[:units_n * 8], a_lo.reshape(-1, f.kp)[:units_n * 8], f)
    exp = np.zeros((b * m, cout))
    for u, i in enumerate(pick):
        exp[pairs[i][0]] = np.maximum(exp[pairs[i][0]], y[8 * u:8 * u + 8].max(axis=0))
    out = torch.zeros((b, m, cout), device=cuda)
    pkg.linear_tc(a_hi, a_lo, f, units=units, unit_pool=True, out_f32=(out, 0))
    _same(out.reshape(-1, cout), exp.astype(np.float32))


@pytest.mark.parametrize("rows", [1, 63, 100, 129, 1000])
@pytest.mark.parametrize("cout", [24, 64, 96, 130])
@pytest.mark.parametrize("outputs", ["f32", "split", "both", "f32_unaligned"])
def test_dense_outputs(pkg, cuda, rows, cout, outputs):
    f = _layer(131 if rows % 2 else 64, cout, rows + cout)
    a_hi, a_lo = _operand((rows,), f, rows)
    y = _expect(a_hi, a_lo, f, relu=rows % 2 == 0)
    relu = rows % 2 == 0
    if outputs == "f32_unaligned":                                 # a 4-byte aligned slice: direct stores, not TMA
        buf = torch.full((rows, cout + 5), -3.0, device=cuda)
        pkg.linear_tc(a_hi, a_lo, f, relu=relu, out_f32=(buf, 1))
        _same(buf[:, 1:1 + cout], y.astype(np.float32))
        assert (buf[:, 0] == -3.0).all() and (buf[:, 1 + cout:] == -3.0).all()
        return
    y32, sp = pkg.linear_tc(a_hi, a_lo, f, relu=relu, want_f32=outputs != "split", want_split=outputs != "f32")
    if outputs != "split":
        _same(y32, y.astype(np.float32))
    if outputs != "f32":
        eh, el = _split(y)
        _same(sp[0][:, :cout], eh)
        _same(sp[1][:, :cout], el)
        assert (sp[0][:, cout:] == 0).all() and (sp[1][:, cout:] == 0).all()     # K padding of the next layer


@pytest.mark.parametrize("pool", [1, 16, 64])
def test_gather_route_resident_operand(pkg, cuda, pool):
    """The two operand routes of linear_tc_kernel on the same rows.  linear_tc streams A through the TMA ring (astat 0);
    linear_tc_gather with K = 16 (one k-block, 32 KiB) always fits the planner's A-stationary plan, so its producer
    warps build each m-tile once and it stays resident while the CTA sweeps the three 64-column n-tiles (astat 1).
    Both must give the float64 result."""
    rng = np.random.default_rng(pool)
    b, n, c, m, ns, cout = 2, 300, 13, 37, 16 if pool == 1 else pool, 160
    xyz = torch.tensor(rng.integers(0, 33, (b, n, 3)) / 8.0, dtype=torch.float32, device=cuda)
    feats = torch.tensor(rng.integers(-3, 4, (b, n, c)), dtype=torch.float32, device=cuda)
    new_xyz = xyz[:, :m].clone()
    idx = torch.tensor(rng.integers(0, n, (b, m, ns)), dtype=torch.int32, device=cuda)
    f = _layer(c + 3, cout, pool)
    a_hi, a_lo = pkg.group_concat_split(xyz, feats, new_xyz, idx)
    y = _expect(a_hi, a_lo, f)
    if pool > 1:
        y = y.max(axis=2)
    g32, _ = pkg.linear_tc_gather(xyz, feats, new_xyz, idx, f, pool=pool, want_f32=True, want_split=False)
    p32, _ = pkg.linear_tc(a_hi, a_lo, f, pool=pool)
    _same(g32, y.astype(np.float32))
    _same(p32, y.astype(np.float32))


def test_two_streams_concurrently(pkg, cuda):
    f1, f2 = _layer(64, 96, 1), _layer(131, 40, 2)
    a1, a2 = _operand((4000,), f1, 1), _operand((2, 300, 32), f2, 2)
    y1, y2 = _expect(*a1, f1), _expect(*a2, f2).max(axis=2)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    outs = []
    for _ in range(3):
        with torch.cuda.stream(s1):
            r1 = pkg.linear_tc(*a1, f1, want_f32=False, want_split=True)[1]
        with torch.cuda.stream(s2):
            r2 = pkg.linear_tc(*a2, f2, pool=32)[0]
        outs.append((r1, r2))
    torch.cuda.synchronize()
    eh, el = _split(y1)
    for (h, l), p in outs:
        _same(h[:, :96], eh)
        _same(l[:, :96], el)
        _same(p, y2.astype(np.float32))
