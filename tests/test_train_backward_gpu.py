"""The training backward on the GPU (-m gpu) at the shapes of the real step: every backward kernel at every call shape
of one ARCH_3DSSD step at b = 8 x 16384 (tests/golden/train_backward_shapes.json, pinned by
tests/test_train_backward_cpu.py) plus edge shapes, against float64.  linear_wgrad, bn_train(_grad), rowgroup_max_grad,
group_concat_grad and vote_translate_grad are called through the C ABI with strided operands as well.

* linear_wgrad on exact operands (test_train_backward_cpu.wgrad_operands): bit for bit float32(float64 x^T dz), with
  NaN-filled workspace and outputs, grad_b = NULL, and ldx > cin / lddz > cout with NaN in the gaps.
* bn_train_grad element by element against the float64 header formula (<= 1 ulp + 1e-12 of the terms), with planted
  rows where the forward's fma(x, scale, shift) is exactly 0; bn_train's y bit for bit against fmaf (+ReLU), its
  statistics within 1 ulp of a two-pass float64 restatement, the moving statistics bit for bit, and x == out in place.
* rowgroup_max_grad bit for bit against the float32 restatement of test_train_grad_gpu, with ties of 3, 5 and 7 rows
  and all-zero groups.
* group_concat_grad, gather_point_grad, vote_translate_grad on dyadic gradients with back-filled indices: bit for bit.
* linear_tc with W^T (the data gradient) at every recorded (rows, K = cout, N = cin), on the exact operands of
  test_tc_epilogue_gpu, bit for bit.
* One real step at b = 8 calls exactly the pinned shapes.
* Full size: every trainable gradient of ARCH_3DSSD + conv1d_0 + head at b = 2 x 16384 within 1e-3 of the
  teacher-forced float64 restatement of test_train_grad_cpu."""
import ctypes
import importlib

import numpy as np
import pytest
import torch

from test_tc_epilogue_gpu import _expect, _layer, _operand
from test_train_grad_gpu import rowgroup_max_grad_f32
from test_train_backward_cpu import (EDGES, load_shapes, record_step, recorded, wgrad_operands, wgrad_plan,
                                     wgrad_shapes)

pytestmark = pytest.mark.gpu
B = 8                                             # the batch of tools/time_train.py
NAN = float("nan")


def _lib():
    return importlib.import_module("3dssd_b200._lib")


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def _s():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _call(name, *args):
    L = _lib()
    L.check(getattr(L.lib(), "ssd3d_" + name)(*args), name)


def _strided(t, extra, fill=NAN):
    """t (rows, c) copied into the first c columns of a (rows, c + extra) buffer filled with `fill`."""
    buf = torch.full((t.shape[0], t.shape[1] + extra), fill, dtype=t.dtype, device=t.device)
    buf[:, :t.shape[1]] = t
    return buf


def _bits(t):
    """The bits of t with -0 read as +0: a sum of one product -0 x y is -0 in float64 but +0 from an accumulator that
    starts at 0."""
    return (t.contiguous() + 0.0).view(torch.int32)


def _same_bits(got, exp, what):
    assert got.shape == exp.shape, what
    bad = (_bits(got) != _bits(exp.float())).sum().item()
    assert bad == 0, "%s: %d of %d elements differ (max |diff| %g)" % (what, bad, got.numel(),
                                                                       (got.double() - exp.double()).abs().max().item())


def _ulp32(ref):
    """ulp of float32(ref) in float64."""
    a = ref.float().abs()
    return (torch.nextafter(a, torch.full_like(a, float("inf"))).double() - a.double())


# ---- A: the step calls exactly the pinned shapes ---------------------------------------------------------------------

def test_real_step_calls_the_pinned_backward_shapes(pkg, cuda):
    rec = record_step(pkg, B, cuda)
    torch.cuda.synchronize()
    assert rec == load_shapes(B)


# ---- B: linear_wgrad -------------------------------------------------------------------------------------------------

def _wgrad(rows, cin, cout, x, ldx, dz, lddz, bias=True):
    """ssd3d_linear_wgrad with a NaN-filled workspace and NaN-filled outputs."""
    ws_bytes = int(_lib().lib().ssd3d_linear_wgrad_workspace(rows, cin, cout))
    ws = torch.full((ws_bytes,), 0xFF, dtype=torch.uint8, device=x.device)          # NaN as float and as double
    gw = torch.full((cin, cout), NAN, device=x.device)
    gb = torch.full((cout,), NAN, device=x.device) if bias else None
    _call("linear_wgrad", rows, cin, cout, _p(x), ldx, _p(dz), lddz, _p(ws), ws_bytes, _p(gw), _p(gb), _s())
    return gw, gb


@pytest.mark.parametrize("variant", ["x_bf16", "dz_bf16"])
def test_linear_wgrad_bit_exact_at_step_and_edge_shapes(pkg, cuda, variant):
    for i, (rows, cin, cout) in enumerate(wgrad_shapes(B)):
        what = "%s rows=%d cin=%d cout=%d" % (variant, rows, cin, cout)
        x, dz = wgrad_operands(rows, cin, cout, variant, 100 * i + len(variant), cuda)
        rps, _ = wgrad_plan(rows, cin, cout)
        assert rps * x.abs().max().item() * dz.abs().max().item() * 256 < 2 ** 24, what    # every split's partial exact
        ew = x.double().t() @ dz.double()
        eb = dz.double().sum(0)
        if rows >= 2 ** 20:                          # the non-negative block's totals pass 2^24 units of 2^-8
            assert ew[0, :16].min().item() * 256 > 2 ** 24, what
        gw, gb = _wgrad(rows, cin, cout, x, cin, dz, cout)
        _same_bits(gw, ew, what + " grad_w")
        _same_bits(gb, eb, what + " grad_b")
        if variant == "x_bf16":
            xs, ds = _strided(x, 5), _strided(dz, 3)
            sw, sb = _wgrad(rows, cin, cout, xs, cin + 5, ds, cout + 3)
            _same_bits(sw, gw, what + " strided grad_w")
            _same_bits(sb, gb, what + " strided grad_b")
            nw, _ = _wgrad(rows, cin, cout, xs, cin + 5, ds, cout + 3, bias=False)
            _same_bits(nw, gw, what + " grad_b = NULL")
        del x, dz, ew


def test_linear_wgrad_wrapper_is_the_dense_call(pkg, cuda):
    x, dz = wgrad_operands(4099, 131, 64, "dz_bf16", 7, cuda)
    gw, gb = pkg.tf_ops.linear_wgrad(x.view(1, 4099, 131), dz.view(1, 4099, 64))
    _same_bits(gw, x.double().t() @ dz.double(), "grad_w")
    _same_bits(gb, dz.double().sum(0), "grad_b")


# ---- C: bn_train and bn_train_grad -------------------------------------------------------------------------------------

EPS = float(np.float32(1e-3))                    # the kernels take eps as a float: r = 1 / sqrt(var + (double)eps)


def _bn_shapes():
    out = []
    for s in recorded("bn_train_grad", B):
        t = (int(np.prod(s[:-2])), s[-2])
        if t not in out:
            out.append(t)
    return out + EDGES["bn_train_grad"]


def _bn_input(rows, c, seed, dev):
    """Pre-BN conv outputs: per-channel offsets and spreads; channel 1 has a mean ~10^3 times its spread and channel 2 is
    constant (var = 0)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn((rows, c), generator=g, device=dev) * (torch.rand((c,), generator=g, device=dev) * 2 + 0.1) \
        + torch.randn((c,), generator=g, device=dev)
    if c > 1:
        x[:, 1] = 1000.0 + torch.randn((rows,), generator=g, device=dev)
    if c > 2:
        x[:, 2] = 0.75
    gamma = torch.rand((c,), generator=g, device=dev) + 0.5
    beta = 0.1 * torch.randn((c,), generator=g, device=dev)
    go = torch.randn((rows, c), generator=g, device=dev)
    return x, gamma, beta, go


def _fma32(x, s, t):
    """float32 fmaf(x, s, t), correctly rounded: the float64 sum with its exact error (TwoSum) decides float32 ties."""
    p = x.double() * s.double()                          # exact
    t64 = t.double().expand_as(p)
    sm = p + t64
    bb = sm - p
    err = (p - (sm - bb)) + (t64 - bb)
    r = sm.float()
    toward = torch.where(sm > r.double(), torch.full_like(r, float("inf")), torch.full_like(r, -float("inf")))
    other = torch.nextafter(r, toward)
    tie = ((r.double() + other.double()) * 0.5 == sm) & (err != 0)
    up = torch.maximum(r, other)
    down = torch.minimum(r, other)
    return torch.where(tie, torch.where(err > 0, up, down), r)


def _bn_train(x, ldx, gamma, beta, mm, mv, decay, relu, out, ldo):
    rows, c = x.shape[0], gamma.shape[0]
    dev = x.device
    ws = torch.full((int(_lib().lib().ssd3d_bn_train_workspace(c)),), 0xFF, dtype=torch.uint8, device=dev)
    scale, shift, mean, var = (torch.full((c,), NAN, device=dev) for _ in range(4))
    _call("bn_train", rows, c, _p(x), ldx, _p(gamma), _p(beta), _p(mm), _p(mv), ctypes.c_float(decay), ctypes.c_float(EPS),
          _p(ws), _p(scale), _p(shift), _p(mean), _p(var), int(relu), _p(out), ldo, _s())
    return scale, shift, mean, var


def _bn_grad(x, ldx, go, ldg, scale, shift, mean, var, gamma, relu, gx, ldgx, want_sums=True):
    rows, c = x.shape[0], gamma.shape[0]
    dev = x.device
    ws = torch.full((int(_lib().lib().ssd3d_bn_train_grad_workspace(c)),), 0xFF, dtype=torch.uint8, device=dev)
    gg, gb = (torch.full((c,), NAN, device=dev) for _ in range(2)) if want_sums else (None, None)
    _call("bn_train_grad", rows, c, _p(x), ldx, _p(go), ldg, _p(scale), _p(shift), _p(mean), _p(var), _p(gamma),
          ctypes.c_float(EPS), int(relu), _p(ws), _p(gg), _p(gb), _p(gx), ldgx, _s())
    return gg, gb


def _bn_grad_check(x, go, scale, shift, mean, var, gamma, relu, gx, gg, gb, what):
    """The header formula in float64 from the kernel's own inputs; <= 1 ulp of float32(ref) + 1e-12 of the terms."""
    rows = x.shape[0]
    g = go.double()
    if relu:
        g = g * ((x.double() * scale.double() + shift.double()) > 0)       # the sign of the exact fma
    r = 1.0 / torch.sqrt(var.double() + EPS)
    xh = (x.double() - mean.double()) * r
    sg, sgx = g.sum(0), (g * xh).sum(0)
    gam = gamma.double()
    ref = gam * r / rows * (rows * g - sg - xh * sgx)
    terms = gam.abs() * r / rows * (rows * g.abs() + sg.abs() + (xh * sgx).abs())
    err = (gx.double() - ref).abs()
    lim = _ulp32(ref) + 1e-12 * terms
    assert (err <= lim).all(), "%s grad_x: worst err / bound %g" % (what, (err / lim).max().item())
    for got, exp, mag, name in ((gb, sg, g.abs().sum(0), "grad_beta"), (gg, sgx, (g * xh).abs().sum(0), "grad_gamma")):
        if got is None:
            continue
        e = (got.double() - exp).abs()
        lim = _ulp32(exp) + 1e-12 * mag
        assert (e <= lim).all(), "%s %s: worst err / bound %g" % (what, name, (e / lim).max().item())


def _ulp_close(got, exp, what):
    e = (got.double() - exp).abs()
    assert (e <= _ulp32(exp)).all(), "%s: worst err %g ulp" % (what, (e / _ulp32(exp)).max().item())


def test_bn_train_and_grad_at_step_and_edge_shapes(pkg, cuda):
    decay = 0.9
    for i, (rows, c) in enumerate(_bn_shapes()):
        what = "rows=%d c=%d" % (rows, c)
        x, gamma, beta, go = _bn_input(rows, c, i, cuda)
        # forward: statistics, moving statistics, y
        g = torch.Generator(device=cuda).manual_seed(1000 + i)
        mm0, mv0 = torch.randn((c,), generator=g, device=cuda), torch.rand((c,), generator=g, device=cuda) + 0.5
        mm, mv = mm0.clone(), mv0.clone()
        y = torch.full_like(x, NAN)
        scale, shift, mean, var = _bn_train(x, c, gamma, beta, mm, mv, decay, True, y, c)
        x64 = x.double()
        emean = x64.mean(0)
        evar = ((x64 - emean) ** 2).mean(0)                                  # two passes
        _ulp_close(mean, emean, what + " batch mean")
        _ulp_close(var, evar, what + " batch var")
        om = np.float32(1.0) - np.float32(decay)
        for got, old, st in ((mm, mm0, mean), (mv, mv0, var)):
            o, s_ = old.cpu().numpy(), st.cpu().numpy()
            exp = o - (o - s_) * om                                          # float32 numpy: the kernel's order
            assert np.array_equal(got.cpu().numpy().view(np.int32), exp.astype(np.float32).view(np.int32)), what
        ey = torch.clamp_min(_fma32(x, scale, shift), 0.0)
        assert torch.equal(y, ey), what + " y"
        xin = x.clone()
        _bn_train(xin, c, gamma, beta, None, None, decay, True, xin, c)     # x == out
        assert torch.equal(xin, y), what + " in place"
        # backward, dense and strided with NaN gaps, and without the parameter sums
        gx = torch.full_like(x, NAN)
        gg, gb = _bn_grad(x, c, go, c, scale, shift, mean, var, gamma, True, gx, c)
        _bn_grad_check(x, go, scale, shift, mean, var, gamma, True, gx, gg, gb, what)
        xs, gos = _strided(x, 3), _strided(go, 5)
        gxs = torch.full((rows, c + 7), -7.0, device=cuda)
        sgg, sgb = _bn_grad(xs, c + 3, gos, c + 5, scale, shift, mean, var, gamma, True, gxs, c + 7)
        _same_bits(gxs[:, :c], gx, what + " strided grad_x")
        assert (gxs[:, c:] == -7.0).all(), what + " strided grad_x gaps"
        _same_bits(sgg, gg, what + " strided grad_gamma")
        _same_bits(sgb, gb, what + " strided grad_beta")
        if i % 4 == 0:
            gxn = torch.full_like(x, NAN)
            _bn_grad(x, c, go, c, scale, shift, mean, var, gamma, True, gxn, c, want_sums=False)
            _same_bits(gxn, gx, what + " grad_gamma = grad_beta = NULL")
        del x, go, y, gx, xs, gos, gxs, xin


@pytest.mark.parametrize("relu", [True, False])
def test_bn_train_grad_relu_decision_at_exact_zero(pkg, cuda, relu):
    """Rows where fma(x, scale, shift) is exactly 0: the forward's ReLU output is 0 there, so its gradient is masked
    (the rule is `> 0`); without the ReLU they count like any other row."""
    rows, c = 20011, 40
    g = torch.Generator(device=cuda).manual_seed(5)
    scale = torch.tensor([0.75, -1.5, 0.5, 2.0] * 10, device=cuda)
    x0 = torch.randint(-64, 64, (c,), generator=g, device=cuda).float() / 16
    shift = -x0 * scale                                                      # exact: fma(x0, scale, shift) == 0
    x = torch.randn((rows, c), generator=g, device=cuda) + x0
    x[::3] = x0                                                              # a third of the rows on the decision
    assert (_fma32(x[::3], scale, shift) == 0).all()
    mean, var = x.double().mean(0).float(), x.double().var(0, unbiased=False).float()
    gamma = torch.rand((c,), generator=g, device=cuda) + 0.5
    go = torch.randn((rows, c), generator=g, device=cuda)
    gx = torch.full_like(x, NAN)
    gg, gb = _bn_grad(x, c, go, c, scale, shift, mean, var, gamma, relu, gx, c)
    _bn_grad_check(x, go, scale, shift, mean, var, gamma, relu, gx, gg, gb, "relu=%s" % relu)
    assert (go[::3].double().sum(0).abs() > 1e-3).all()                     # the planted rows move grad_beta visibly
    exp = (go.double() * ((x.double() * scale.double() + shift.double()) > 0)).sum(0) if relu else go.double().sum(0)
    assert ((gb.double() - exp).abs() <= _ulp32(exp) + 1e-12 * go.double().abs().sum(0)).all()


# ---- D: rowgroup_max_grad ----------------------------------------------------------------------------------------------

def _rowgroup_case(groups, pool, c, seed, dev):
    """Post-ReLU-like groups: 1/8-steps with random ties; every 4th group from 1 has its maximum tied in exactly 3, 5 or 7
    rows (1/num not dyadic), every 4th from 2 is all zero (num = pool)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    y = torch.clamp_min(torch.randint(-40, 40, (groups, pool, c), generator=g, device=dev).float() / 8, 0.0)
    k = torch.tensor([3, 5, 7], device=dev)[torch.arange(groups, device=dev) % 3]
    tie = torch.arange(pool, device=dev).view(1, pool, 1) < torch.minimum(k, torch.tensor(pool, device=dev)).view(-1, 1, 1)
    sel = (torch.arange(groups, device=dev) % 4 == 1).view(-1, 1, 1)
    y = torch.where(sel & tie, torch.full_like(y, 6.0), torch.where(sel, torch.clamp_max(y, 5.0), y))
    y[2::4] = 0.0
    cnt = torch.randint(0, 3, (groups,), generator=g, device=dev, dtype=torch.int32)
    go = torch.randn((groups, c), generator=g, device=dev)
    return y, cnt, go


def test_rowgroup_max_grad_at_step_shapes_strided(pkg, cuda):
    shapes = [tuple(s) for s in recorded("rowgroup_max_grad", B)] + EDGES["rowgroup_max_grad"]
    for i, (b, m, pool, c, mask) in enumerate(shapes):
        what = "b=%d m=%d pool=%d c=%d" % (b, m, pool, c)
        groups = b * m
        y, cnt, go = _rowgroup_case(groups, pool, c, i, cuda)
        exp = torch.from_numpy(rowgroup_max_grad_f32(y.cpu().numpy(), go.cpu().numpy(),
                                                     cnt.cpu().numpy() if mask else None)).to(cuda)
        if pool >= 7:
            assert {3, 5, 7} <= set((y == y.amax(1, keepdim=True)).sum(1).unique().tolist())
        gy = torch.full_like(y, NAN)
        cnt = cnt if mask else None
        _call("rowgroup_max_grad", groups, pool, c, _p(y), c, _p(cnt), _p(go), _p(gy), c, _s())
        _same_bits(gy, exp, what)
        ys = _strided(y.view(-1, c), 4)
        gys = torch.full((groups * pool, c + 2), -7.0, device=cuda)
        _call("rowgroup_max_grad", groups, pool, c, _p(ys), c + 4, _p(cnt), _p(go), _p(gys), c + 2, _s())
        _same_bits(gys[:, :c].reshape(y.shape), exp, what + " strided")
        assert (gys[:, c:] == -7.0).all(), what + " gaps"


# ---- E: the scatters ---------------------------------------------------------------------------------------------------

def _backfilled_idx(b, m, ns, n, seed, dev):
    """Neighbour lists as ball query writes them: a random number of found points, the rest back-filled with the first."""
    g = torch.Generator(device=dev).manual_seed(seed)
    idx = torch.randint(0, n, (b, m, ns), generator=g, device=dev, dtype=torch.int32)
    found = torch.randint(1, ns + 1, (b, m, 1), generator=g, device=dev)
    return torch.where(torch.arange(ns, device=dev).view(1, 1, ns) < found, idx, idx[..., :1])


def _dyadic(shape, seed, dev):
    g = torch.Generator(device=dev).manual_seed(seed)
    return torch.randint(-8, 9, shape, generator=g, device=dev).float() / 16


def _scatter_expect(src, idx, b, n):
    """float64 scatter-add of src rows (b, rows, w) into (b, n, w); exact for dyadic sums."""
    w = src.shape[-1]
    flat = (idx.long().reshape(b, -1) + torch.arange(b, device=src.device).view(b, 1) * n).reshape(-1)
    out = torch.zeros((b * n, w), dtype=torch.float64, device=src.device)
    out.index_add_(0, flat, src.reshape(-1, w).double())
    counts = torch.bincount(flat, minlength=b * n)
    assert counts.max().item() * 8 < 2 ** 24                  # |each term| <= 8/16: every fp32 partial sum is exact
    return out.view(b, n, w)


def _group_concat_grad(b, n, c, m, ns, idx, gx, ldx, want):
    dev = gx.device
    gp = torch.full((b, n, max(c, 1)), NAN, device=dev) if want[0] else None
    gxyz = torch.full((b, n, 3), NAN, device=dev) if want[1] else None
    gnew = torch.full((b, m, 3), NAN, device=dev) if want[2] else None
    _call("group_concat_grad", b, n, c, m, ns, _p(idx), _p(gx), ldx, _p(gp), _p(gxyz), _p(gnew), _s())
    return gp, gxyz, gnew


def _group_concat_check(b, n, c, m, ns, seed, dev, ldx, wants):
    idx = _backfilled_idx(b, m, ns, n, seed, dev)
    g = _dyadic((b * m * ns, c + 3), seed, dev)
    gxs = _strided(g, ldx - c - 3)
    ep = _scatter_expect(g[:, :c].view(b, -1, c), idx, b, n) if c else None
    exyz = _scatter_expect(g[:, c:].view(b, -1, 3), idx, b, n)
    enew = -g[:, c:].double().view(b, m, ns, 3).sum(2)
    for want in wants:
        what = "b=%d n=%d c=%d m=%d ns=%d ldx=%d want=%s" % (b, n, c, m, ns, ldx, want)
        gp, gxyz, gnew = _group_concat_grad(b, n, c, m, ns, idx, gxs, ldx, want)
        if gp is not None and c:
            _same_bits(gp, ep, what + " grad_points")
        if gp is not None and not c:
            assert torch.isnan(gp).all(), what + " grad_points with c = 0 is not written"
        if gxyz is not None:
            _same_bits(gxyz, exyz, what + " grad_xyz")
        if gnew is not None:
            _same_bits(gnew, enew, what + " grad_new_xyz")


def test_group_concat_grad_at_step_shapes_strided(pkg, cuda):
    for i, (b, m, ns, ldx, n, c, wp, wx, wn) in enumerate(recorded("group_concat_grad", B)):
        assert ldx == c + 3
        _group_concat_check(b, n, c, m, ns, i, cuda, c + 3 + 4, [(wp, wx, wn)])


def test_group_concat_grad_every_output_combination(pkg, cuda):
    combos = [(p, x, w) for p in (0, 1) for x in (0, 1) for w in (0, 1)]
    _group_concat_check(2, 300, 13, 40, 16, 1, cuda, 13 + 3 + 6, combos)
    _group_concat_check(2, 300, 13, 40, 16, 2, cuda, 13 + 3, combos)
    _group_concat_check(2, 300, 0, 40, 16, 3, cuda, 5, combos)                 # c = 0: only the xyz columns


def test_gather_point_grad_at_step_shapes(pkg, cuda):
    for i, (b, n, c, m) in enumerate(recorded("gather_point_grad", B)):
        g = torch.Generator(device=cuda).manual_seed(i)
        idx = torch.randint(0, n, (b, m), generator=g, device=cuda, dtype=torch.int32)
        idx[:, m // 2:] = idx[:, :1]                                          # duplicated samples
        og = _dyadic((b, m, c), i, cuda)
        got = pkg.tf_ops.gather_point_grad(torch.empty((b, n, c), device="meta"), idx, og)
        _same_bits(got, _scatter_expect(og, idx, b, n), "b=%d n=%d c=%d m=%d" % (b, n, c, m))


def test_vote_translate_grad_at_step_shapes_strided(pkg, cuda):
    lo = (-3.0, -3.0, -2.0)
    for i, (b, n, w) in enumerate(recorded("vote_translate_grad", B) + EDGES["vote_translate_grad"]):
        g = torch.Generator(device=cuda).manual_seed(i)
        off = (torch.rand((b * n, 3), generator=g, device=cuda) * 8 - 4)
        lim = torch.tensor(lo, device=cuda)
        off[::5] = lim
        off[1::5] = -lim
        off[2::5] = torch.nextafter(lim, torch.full_like(lim, -10.0))
        go = torch.randn((b * n, 3), generator=g, device=cuda)
        exp = torch.where((off >= lim) & (off <= -lim), go, torch.zeros_like(go))
        for ld in (3, 7):
            offs = _strided(off, ld - 3)
            got = torch.full_like(go, NAN)
            _call("vote_translate_grad", b * n, _p(offs), ld, _p(go), ctypes.c_float(lo[0]), ctypes.c_float(lo[1]),
                  ctypes.c_float(lo[2]), _p(got), _s())
            _same_bits(got, exp, "b=%d n=%d ld_offsets=%d" % (b, n, ld))


# ---- F: the data-gradient GEMM ---------------------------------------------------------------------------------------

def test_linear_tc_transposed_at_step_shapes(pkg, cuda):
    """grad_x = dz.W^T as _ConvTrain.backward runs it: linear_tc with the fold of W^T (scale 1, shift 0, no ReLU), at every
    recorded (rows, K = cout, N = cin), on the exact operands of test_tc_epilogue_gpu (W = integer + k/256, dz split into
    an integer hi and a lo in 1/16 steps): bit for bit float32 of the float64 hi.W_hi + lo.W_hi + hi.W_lo."""
    seen = []
    for s in recorded("linear_tc_t", B):
        rows, k, n = int(np.prod(s[:-2])), s[-2], s[-1]
        if (rows, k, n) in seen:
            continue
        seen.append((rows, k, n))
        w = _layer(n, k, len(seen)).w                                     # layer weights (cin = N, cout = K)
        f = pkg.params.FoldedConv(w.t().contiguous(), torch.ones((n,), device=cuda), torch.zeros((n,), device=cuda))
        a_hi, a_lo = _operand((rows,), f, len(seen))
        y, _ = pkg.tf_ops.linear_tc(a_hi, a_lo, f, relu=False, want_f32=True, want_split=False)
        _same_bits(y, torch.from_numpy(_expect(a_hi, a_lo, f, relu=False)).to(cuda), "rows=%d K=%d N=%d" % (rows, k, n))
        del a_hi, a_lo, y


# ---- G: full-size gradients against the teacher-forced float64 restatement ------------------------------------------

def test_full_size_gradients_teacher_forced(pkg, cuda):
    """Two KITTI-like scenes (full_size_gradients_teacher_forced)."""
    synth = importlib.import_module("3dssd_b200.synth")
    full_size_gradients_teacher_forced(pkg, cuda, synth.kitti_like(2, 16384, seed=3))


def full_size_gradients_teacher_forced(pkg, cuda, points):
    """ARCH_3DSSD + conv1d_0 + head on points [b, 16384, 4] through the trainable path, loss = a random linear
    functional of the head outputs and the vote offsets.  The layer loop of backbone.train_forward is driven here with return_debug, so
    that sampling, neighbour lists, ReLU masks and pooling winners can be handed to the float64 restatement of
    test_train_grad_cpu (run on the GPU); its outputs must first equal train_forward's bit for bit.  Every trainable
    tensor's gradient is then held to 1e-3 (compare_grads)."""
    from test_train_grad_cpu import compare_grads, gather_rows, recording, ref_conv, ref_head, ref_leaves, ref_sa_msg, ref_vote
    cfg, L = pkg.config, pkg.layers_util
    arch = cfg.ARCH_3DSSD
    assert cfg.AGGREGATION_SA_FEATURE
    xyz, feat = pkg.tf_ops.split_points(torch.from_numpy(np.ascontiguousarray(points, dtype=np.float32)).to(cuda))
    d = pkg.params.init_params(arch, 1, seed=5, random_bias=True)
    d.update(pkg.params.init_head_params(cfg.layer_channels(arch, 1)[-1], seed=6))
    with torch.no_grad():
        o = pkg.backbone.train_forward(arch, pkg.params.TrainableParams(d, cuda), xyz, feat)

    tp = pkg.params.TrainableParams(d, cuda)
    rec = recording(pkg, tp)
    xyz_l, feat_l, fps_l, dbg_l, offs = [xyz], [feat], [None], [None], []
    for (xyz_i, feat_i, radius, nsample, mlps, bn, rng, method, npoint, former, attn, ltype, scope, dilated, vote_idx,
         agg) in arch:
        if ltype == "SA_Layer":
            r = L.pointnet_sa_module_msg(xyz_l[xyz_i[0]], feat_l[feat_i[0]], radius, nsample, mlps, True, None, bn, rng, method,
                                         npoint, fps_l[former] if former != -1 else None, attn, scope, dilated,
                                         xyz_l[vote_idx] if vote_idx != -1 else None, agg, params=tp, return_debug=True)
            xyz_l.append(r[0]); feat_l.append(r[1]); fps_l.append(r[2]); dbg_l.append(r[3])
        else:
            assert ltype == "Vote_Layer"
            nx, nf, off = L.vote_layer(xyz_l[xyz_i[0]], feat_l[feat_i[0]], mlps, True, None, bn, scope, params=tp)
            xyz_l.append(nx); feat_l.append(nf); fps_l.append(None); dbg_l.append(None); offs.append(off)
    head = pkg.head.box_regression_head(tp.conv_train("conv1d_0", feat_l[-1], True), 1, 1, 6, True, True, params=tp)
    outs = list(head) + offs
    assert len(outs) == len(o.head) + len(o.vote_offsets)
    for got, exp in zip(outs, list(o.head) + list(o.vote_offsets)):
        assert torch.equal(got.detach(), exp)
    del o

    g = torch.Generator(device=cuda).manual_seed(8)
    R = [torch.randn(tuple(t.shape), generator=g, device=cuda) for t in outs]
    sum((t * r).sum() for t, r in zip(outs, R)).backward()

    P = ref_leaves(tp, cuda)
    xr_l, fr_l, offs_r = [xyz.double()], [feat.double()], []
    for li, (xyz_i, feat_i, radius, nsample, mlps, bn, rng, method, npoint, former, attn, ltype, scope, dilated, vote_idx,
             agg) in enumerate(arch, 1):
        if ltype == "SA_Layer":
            new_xyz = gather_rows(xr_l[vote_idx] if vote_idx != -1 else xr_l[xyz_i[0]], fps_l[li])      # :116-119
            if radius:
                out = ref_sa_msg(P, rec, xr_l[xyz_i[0]], fr_l[feat_i[0]], new_xyz, dbg_l[li]["idx"], dbg_l[li]["cnt"], mlps,
                                 scope, agg not in (None, -1))
            else:
                out = gather_rows(fr_l[feat_i[0]], fps_l[li])                                          # :186-187
            xr_l.append(new_xyz); fr_l.append(out)
        else:
            ctr, pts, off = ref_vote(P, rec, xr_l[xyz_i[0]], fr_l[feat_i[0]], len(mlps), scope, cfg.MAX_TRANSLATE_RANGE)
            xr_l.append(ctr); fr_l.append(pts); offs_r.append(off)
    cls, reg = ref_head(P, rec, ref_conv(P, rec, "conv1d_0", fr_l[-1], True, True))
    reg = reg.view(tuple(head[1].shape[:3]) + (-1,))
    exp = [cls, reg[..., :6], reg[..., 6:18], reg[..., 18:]] + offs_r
    sum((e * r.double()).sum() for e, r in zip(exp, R)).backward()
    ratio = compare_grads(tp, P, tol=1e-3)
    worst = {}
    for k, v in ratio.items():
        layer = k.split("/")[0]
        if v >= worst.get(layer, (-1.0, ""))[0]:
            worst[layer] = (v, k)
    print("\nfull-size gradients, worst error / bound per layer (bound: 1e-3 of max|ref|, biases before BN 1e-5 of "
          "max|grad_w|):")
    for layer, (v, k) in worst.items():
        print("  %-10s %.3e  (%s)" % (layer, v, k))
