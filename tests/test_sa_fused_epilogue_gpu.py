"""The fragment epilogue of sa_fused_kernel (scale/shift/ReLU/split written in place as the next layer's operand, and the
max-pool of the last layer on the wgmma accumulator fragments) at the shapes the benchmark does not reach: every
compile-time twin and the run-time-shape kernel, every pooling width, unit lists that end inside a tile, row counts
that are not tile multiples, every tail-block width, every output combination, pool-before / after the affine, negative
scales and concurrent launches.

Operands are small dyadic numbers (operand and weight lo terms included), so every product and every fp32 partial sum is
exact: the kernel's result must equal the float64 evaluation of hi.W_hi + lo.W_hi + hi.W_lo, fmaf(acc, scale, shift),
ReLU, the kernel's bf16 split between layers and the pool, bit for bit.  _layer_exact checks that premise per layer."""
import importlib

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _P():
    return importlib.import_module("3dssd_b200.params")


def _grid(a):
    """smallest e with a * 2^e integral everywhere"""
    for e in range(48):
        if np.array_equal(np.round(a * 2.0 ** e), a * 2.0 ** e):
            return e
    raise AssertionError("operand is not dyadic")


def _conv(cin, cout, rng, lo_terms):
    """A folded conv: weights in {-1, 0, 1} (+-2^-9 lo terms where nonzero when lo_terms), scales 1/4 or 1/2 with every
    third negative, shifts multiples of 1/16."""
    w = rng.integers(-1, 2, (cin, cout)).astype(np.float64)
    if lo_terms:
        w += (w != 0) * rng.integers(-1, 2, (cin, cout)) * 2.0 ** -9
    scale = rng.choice([0.25, 0.5], cout)
    scale[1::3] *= -1.0
    shift = rng.integers(-8, 9, cout) / 16.0
    return _P().FoldedConv(*(torch.tensor(a, dtype=torch.float32, device="cuda") for a in (w, scale, shift)))


def _split(y):
    """the kernel's split: hi = bf16_rn(y), lo = bf16_rn(y - hi), as float64 arrays"""
    t = torch.tensor(y, dtype=torch.float32)
    hi = t.to(torch.bfloat16)
    return hi.double().numpy(), (t - hi.float()).to(torch.bfloat16).double().numpy()


def _layer_exact(hi, lo, f):
    """float64 relu(fma(hi.W_hi + lo.W_hi + hi.W_lo, scale, shift)); asserts that fp32 computes it exactly"""
    bh, bl = (t.double().cpu().numpy()[:, :f.cin] for t in (f.b_hi, f.b_lo))      # (cout, cin)
    # every product is a multiple of 2^-e; partial sums below 2^(24-e) in magnitude are then exact in fp32
    e = max(_grid(a) + _grid(w) for a, w in ((hi, bh), (lo, bh), (hi, bl)) if a.any() and w.any())
    bound = np.abs(hi) @ np.abs(bh).T + np.abs(lo) @ np.abs(bh).T + np.abs(hi) @ np.abs(bl).T
    assert bound.max() < 2.0 ** (24 - e), "test operands must keep every fp32 partial sum exact"
    acc = hi @ bh.T + lo @ bh.T + hi @ bl.T
    y = acc * f.scale.double().cpu().numpy() + f.shift.double().cpu().numpy()
    assert np.array_equal(y.astype(np.float32).astype(np.float64), y), "test operands must keep the epilogue exact"
    return np.maximum(y, 0)


def _stack_rows(x, convs):
    """per-row float64 result of the stack on the fp32 operand rows x (..., K0)"""
    hi, lo = _split(x)
    for li, f in enumerate(convs):
        y = _layer_exact(hi, lo, f)
        if li < len(convs) - 1:
            hi, lo = _split(y)
    return y


class Scale:
    """One SA scale with exactly representable inputs: (b, n) points, m centres, ns neighbours, a conv stack `mlp`, either
    plain (operand concat(features, xyz - centre)) or hoisted (operand relu(z + (xyz - centre) . Wx))."""

    def __init__(self, b, n, c, m, ns, mlp, hoist, seed):
        rng = np.random.default_rng(seed)
        self.b, self.m, self.ns, self.hoist = b, m, ns, hoist
        xyz = rng.integers(0, 3, (b, n, 3)).astype(np.float64)
        new_xyz = xyz[:, :m].copy()
        idx = rng.integers(0, n, (b, m, ns))
        self.cnt = rng.integers(0, 3, (b, m))
        gx = np.take_along_axis(xyz[:, :, None], idx.reshape(b, -1, 1, 1), 1).reshape(b, m, ns, 3)
        d = gx - new_xyz[:, :, None]
        if hoist:
            z = rng.integers(-2, 3, (b, n, c)).astype(np.float64)              # lo terms in the weights only (the ReLU
            wx = rng.integers(-1, 2, (3, c)).astype(np.float64)               # could make an operand's hi a fraction)
            gz = np.take_along_axis(z[:, :, None], idx.reshape(b, -1, 1, 1), 1).reshape(b, m, ns, c)
            x = np.maximum(gz + d @ wx, 0)
            self.src = (torch.tensor(z, dtype=torch.float32, device="cuda"), torch.tensor(wx, dtype=torch.float32, device="cuda"))
            cin = c
        else:
            h = rng.integers(-1, 2, (b, n, c)).astype(np.float64)
            feats = h + (h != 0) * rng.integers(-1, 2, (b, n, c)) * 2.0 ** -9   # bf16 hi = the integer (a tie), lo = +-2^-9
            gf = np.take_along_axis(feats[:, :, None], idx.reshape(b, -1, 1, 1), 1).reshape(b, m, ns, c)
            x = np.concatenate([gf, d], -1)
            self.src = torch.tensor(feats, dtype=torch.float32, device="cuda")
            cin = c + 3
        self.convs = []
        for j, cout in enumerate(mlp):
            self.convs.append(_conv(cin, cout, rng, lo_terms=j == 0))
            cin = cout
        self.stack = _P().FusedStack(self.convs, c if hoist else c + 3)
        self.rows = _stack_rows(x, self.convs)                                  # (b, m, ns, C)
        self.t = {k: torch.tensor(v, dtype=torch.int32 if k in ("idx", "cnt") else torch.float32, device="cuda")
                  for k, v in (("xyz", xyz), ("new_xyz", new_xyz), ("idx", idx), ("cnt", self.cnt))}

    def expect(self):
        return self.rows.max(axis=2) * (self.cnt > 0)[..., None]

    def run(self, pkg, **kw):
        t = self.t
        if self.hoist:
            z, wx = self.src
            return pkg.sa_mlp_fused_hoisted(t["xyz"], z, 0, wx, t["new_xyz"], t["idx"], t["cnt"], self.stack, **kw)
        return pkg.sa_mlp_fused(t["xyz"], self.src, t["new_xyz"], t["idx"], t["cnt"], self.stack, **kw)


def _same(got, exp):
    assert torch.equal(got.cpu(), exp.cpu() if torch.is_tensor(exp) else torch.tensor(exp, dtype=got.dtype))


SCALES = {  # b, n, c, m, ns, mlp, hoist
    "L1s1": (2, 300, 16, 50, 32, [16, 32], True),            # SfStat<16, 16, 32, 32>: one warpgroup, both halves in turn
    "L1s3": (2, 300, 32, 35, 64, [32, 64], True),            # SfStat<32, 32, 64, 64>
    "L2s1": (2, 600, 64, 70, 32, [64, 128], True),           # SfStat<64, 64, 128, 32>: two slots, a warpgroup per half
    "L2s3": (2, 600, 64, 45, 64, [96, 128], True),           # SfStat<64, 96, 128, 64>: 64 + 32-column hidden chunks
    "pool8": (2, 300, 5, 17, 8, [16]),                       # run-time shapes from here on; one layer, 8-row groups
    "pool16_tails": (3, 300, 45, 33, 16, [112, 80, 64]),     # K = 48 / 112 / 80: tail rows of 128 / 128 / 32 bytes
    "k96": (2, 300, 93, 21, 64, [48, 32]),                   # K = 96 / 48: tail rows of 64 / 128 bytes
    "pool128_wg1": (1, 400, 8, 9, 128, [32, 32, 64]),        # a group is the whole tile, one warpgroup
    "pool128_wg2": (2, 500, 64, 5, 128, [64, 64, 128]),      # ... and two warpgroups (the halves meet across them)
}


def _scale(name, seed=0):
    b, n, c, m, ns, mlp, *hoist = SCALES[name]
    return Scale(b, n, c, m, ns, mlp, bool(hoist and hoist[0]), seed=len(name) + 7 * seed)


@pytest.mark.parametrize("name", sorted(SCALES))
@pytest.mark.parametrize("pool_first", [True, False])
def test_fused_scale_every_output(pkg, cuda, name, pool_first):
    """fp32 only, split only and both outputs, into slices of wider buffers; pool_first False runs the affine + ReLU on
    every accumulator before the pool (the last layer's scales are non-negative in a FusedStack, so both agree)."""
    s = _scale(name)
    s.stack.last_scale_nonneg = pool_first
    y = s.expect()
    cout = y.shape[-1]
    eh, el = (torch.tensor(a, dtype=torch.bfloat16) for a in _split(y))
    _same(s.run(pkg), y.astype(np.float32))
    for outputs in ("split", "both"):
        f32 = torch.full((s.b, s.m, cout + 40), -7.0, device=cuda)
        sh = torch.zeros((s.b, s.m, cout + 40), dtype=torch.bfloat16, device=cuda)
        sl = torch.zeros_like(sh)
        s.run(pkg, out_f32=(f32, 24) if outputs == "both" else None, out_split=(sh, sl, 24))
        _same(sh[..., 24:24 + cout], eh)
        _same(sl[..., 24:24 + cout], el)
        assert (sh[..., :24] == 0).all() and (sh[..., 24 + cout:] == 0).all()
        if outputs == "both":
            _same(f32[..., 24:24 + cout], y.astype(np.float32))
            assert (f32[..., :24] == -7.0).all() and (f32[..., 24 + cout:] == -7.0).all()


@pytest.mark.parametrize("name", ["L1s1", "L2s1", "pool16_tails"])
@pytest.mark.parametrize("units_n", [1, 17, 130])
def test_fused_unit_lists_ending_mid_tile(pkg, cuda, name, units_n):
    """A tile of 16 listed 8-row units; the list ends inside a tile.  A group's result is the max over its listed units
    (zero when none is listed: the caller's zero fill)."""
    s = _scale(name, seed=units_n)
    rng = np.random.default_rng(units_n)
    pairs = [(g, j) for g in range(s.b * s.m) for j in range(s.ns // 8)]
    pick = sorted(rng.choice(len(pairs), min(units_n, len(pairs)), replace=False))
    units = torch.tensor([len(pick)] + [(pairs[i][0] << 4) | pairs[i][1] for i in pick], dtype=torch.int32, device=cuda)
    rows = s.rows.reshape(s.b * s.m, s.ns, -1)
    exp = np.zeros((s.b * s.m, rows.shape[-1]))
    for i in pick:
        g, j = pairs[i]
        exp[g] = np.maximum(exp[g], rows[g, 8 * j:8 * j + 8].max(axis=0))
    out = torch.zeros((s.b, s.m, rows.shape[-1]), device=cuda)
    s.run(pkg, out_f32=(out, 0), units=units)
    _same(out.reshape(s.b * s.m, -1), exp.astype(np.float32))


def test_fused_two_streams_concurrently(pkg, cuda):
    s1, s2 = _scale("L2s3"), _scale("L1s3")
    y1, y2 = s1.expect().astype(np.float32), s2.expect().astype(np.float32)
    st1, st2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    outs = []
    for _ in range(3):
        with torch.cuda.stream(st1):
            r1 = s1.run(pkg)
        with torch.cuda.stream(st2):
            r2 = s2.run(pkg)
        outs.append((r1, r2))
    torch.cuda.synchronize()
    for r1, r2 in outs:
        _same(r1, y1)
        _same(r2, y2)
