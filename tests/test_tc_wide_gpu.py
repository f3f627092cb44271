"""linear_tc_tma_kernel, the kernel of every linear_tc launch whose A operand is read from memory, at every tile width the
launch plan picks (32, 64 and 128 columns, chosen by N, the output kind and the tile count), with every epilogue:
TMA-store and direct outputs, the max-pools with rowmask, unit-list pools that end inside a tile, row counts around the
128-row tile, K of one k-block up to 1536, the full-size layer-4 unit-pool launch and launches on two streams at once.

The operands are the exact ones of test_tc_epilogue_gpu.py: every result must equal the float64 evaluation bit for bit."""
import numpy as np
import pytest
import torch

from test_tc_epilogue_gpu import _expect, _layer, _operand, _same, _split

pytestmark = pytest.mark.gpu

# N -> tile at 17 000 rows: 24 -> 32, 40 -> 64, 72 and wider -> 128 (one to nine n-tiles, the last one partly past N).
# TMA-store launches ("f32", "split") keep 64: a 128-column ring of 3 stages does not fit next to their store blocks.
# Below 132 tiles the plan stays at 64 columns, so the small row counts run the 64-column kernel.
WIDTHS = [24, 40, 72, 130, 200, 256, 264, 520, 1024]


def _dense(pkg, cuda, rows, cin, cout, outputs, seed):
    f = _layer(cin, cout, seed)
    a_hi, a_lo = _operand((rows,), f, seed + 1)
    relu = seed % 2 == 0
    y = _expect(a_hi, a_lo, f, relu=relu)
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
        assert (sp[0][:, cout:] == 0).all() and (sp[1][:, cout:] == 0).all()


@pytest.mark.parametrize("cout", WIDTHS)
@pytest.mark.parametrize("outputs", ["f32", "split", "both", "f32_unaligned"])
def test_every_width_and_output(pkg, cuda, cout, outputs):
    _dense(pkg, cuda, 17000, 67, cout, outputs, cout)


@pytest.mark.parametrize("rows", [1, 127, 129])
@pytest.mark.parametrize("cout", [72, 256, 1024])
@pytest.mark.parametrize("outputs", ["f32", "both"])
def test_row_counts(pkg, cuda, rows, cout, outputs):
    _dense(pkg, cuda, rows, 131, cout, outputs, rows + cout)


def test_thousand_rows(pkg, cuda):
    _dense(pkg, cuda, 1000, 131, 1024, "both", 5)


@pytest.mark.parametrize("cin", [16, 512, 1536])
@pytest.mark.parametrize("cout", [130, 1024])
def test_k_depths(pkg, cuda, cin, cout):
    _dense(pkg, cuda, 2200, cin, cout, "both", cin + cout)


@pytest.mark.parametrize("pool", [8, 16, 32, 64, 128])
@pytest.mark.parametrize("cout", [130, 256, 520, 1024])
def test_pool_every_width(pkg, cuda, pool, cout):
    b, m = 2, 8500 // (2 * pool) + 1                               # >= 132 tiles at 128 columns; rows % 128 != 0
    f = _layer(67, cout, pool + cout)
    a_hi, a_lo = _operand((b, m, pool), f, pool)
    cnt = torch.tensor(np.random.default_rng(pool).integers(0, 3, (b, m)), dtype=torch.int32, device=cuda)
    y = _expect(a_hi, a_lo, f).max(axis=2) * (cnt.cpu().numpy() > 0)[..., None]
    ld = (cout + 7) // 8 * 8 + 40                                  # split rows: a multiple of 8 elements
    f32 = torch.full((b, m, ld), -7.0, device=cuda)
    sh = torch.zeros((b, m, ld), dtype=torch.bfloat16, device=cuda)
    sl = torch.zeros_like(sh)
    pkg.linear_tc(a_hi, a_lo, f, pool=pool, rowmask=cnt, out_f32=(f32, 24), out_split=(sh, sl, 24))
    _same(f32[..., 24:24 + cout], y.astype(np.float32))
    assert (f32[..., :24] == -7.0).all() and (f32[..., 24 + cout:] == -7.0).all()
    eh, el = _split(y)
    _same(sh[..., 24:24 + cout], eh)
    _same(sl[..., 24:24 + cout], el)


def _unit_list(rng, groups, ns, units_n, cuda):
    """A list as the ball query writes it: every group's first unit, then further units of random groups, in order."""
    firsts = [(g, 0) for g in range(groups)][:units_n]
    rest = [(g, j) for g in range(groups) for j in range(1, ns // 8)]
    extra = rng.choice(len(rest), units_n - len(firsts), replace=False) if units_n > len(firsts) else []
    pairs = sorted(firsts + [rest[i] for i in extra])
    return pairs, torch.tensor([units_n] + [(g << 4) | j for g, j in pairs], dtype=torch.int32, device=cuda)


def _unit_pool(pkg, cuda, groups, ns, units_n, cin, cout, seed):
    rng = np.random.default_rng(seed)
    f = _layer(cin, cout, seed)
    pairs, units = _unit_list(rng, groups, ns, units_n, cuda)
    a_hi, a_lo = _operand((groups, ns), f, seed + 1)                  # rows past units_n * 8 are capacity, never read
    y = _expect(a_hi.reshape(-1, f.kp)[:units_n * 8], a_lo.reshape(-1, f.kp)[:units_n * 8], f)
    exp = np.zeros((groups, cout))
    for u, (g, _) in enumerate(pairs):
        exp[g] = np.maximum(exp[g], y[8 * u:8 * u + 8].max(axis=0))
    out = torch.zeros((groups, cout), device=cuda)
    pkg.linear_tc(a_hi, a_lo, f, units=units, unit_pool=True, out_f32=(out, 0))
    _same(out, exp.astype(np.float32))


@pytest.mark.parametrize("units_n", [1, 15, 17, 130])
@pytest.mark.parametrize("cout", [256, 1024])
def test_unit_pool_lists_ending_mid_tile(pkg, cuda, units_n, cout):
    _unit_pool(pkg, cuda, 300, 32, units_n, 48, cout, units_n + cout)


def test_full_size_layer4_unit_pool(pkg, cuda):
    """The 512 -> 1024 unit-pool conv of layer 4 at the benchmark's size: 2048 groups of 32 slots, about 28 900 rows."""
    _unit_pool(pkg, cuda, 2048, 32, 3612, 512, 1024, 4)


def test_two_streams_concurrently(pkg, cuda):
    f1, f2 = _layer(64, 256, 1), _layer(256, 1024, 2)
    a1 = _operand((4000,), f1, 1)
    rng = np.random.default_rng(3)
    pairs, units = _unit_list(rng, 300, 32, 700, cuda)
    a2 = _operand((300, 32), f2, 2)
    y1 = _expect(*a1, f1)
    y2u = _expect(a2[0].reshape(-1, f2.kp)[:700 * 8], a2[1].reshape(-1, f2.kp)[:700 * 8], f2)
    y2 = np.zeros((300, 1024))
    for u, (g, _) in enumerate(pairs):
        y2[g] = np.maximum(y2[g], y2u[8 * u:8 * u + 8].max(axis=0))
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    outs = []
    for _ in range(3):
        with torch.cuda.stream(s1):
            r1 = pkg.linear_tc(*a1, f1, want_f32=False, want_split=True)[1]
        with torch.cuda.stream(s2):
            r2 = torch.zeros((300, 1024), device=cuda)
            pkg.linear_tc(*a2, f2, units=units, unit_pool=True, out_f32=(r2, 0))
        outs.append((r1, r2))
    torch.cuda.synchronize()
    eh, el = _split(y1)
    for (h, l), p in outs:
        _same(h[:, :256], eh)
        _same(l[:, :256], el)
        _same(p, y2.astype(np.float32))
