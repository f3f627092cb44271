"""The shapes and the arithmetic plan of the training backward, on the CPU.

* The backward entry points of tf_ops are wrapped to record their call shapes (the `_Timed` wrapper of
  tools/time_train.py, shapes only) while one ARCH_3DSSD step of tools/time_train.py runs through the CPU dry fixture.
  The list is pinned in tests/golden/train_backward_shapes.json; tests/test_train_backward_gpu.py checks that one real
  step on the GPU calls exactly these shapes and runs every kernel at each of them.
* `wgrad_plan` restates the split-K plan of csrc/train_grad.cu (132 SMs, 3 CTAs per SM, 64-row chunks); it is checked
  against ssd3d_linear_wgrad_workspace = splits * cout * (8 + 4 cin), a host-only query of the library.
* The exact-operand construction of the linear_wgrad test: operands whose three bf16 product terms carry bits, whose
  dropped lo*lo term is 0 and whose per-split fp32 partials are integers below 2^24 units, so the kernel's result is
  float32 of the float64 product, bit for bit.

Recorded shapes: every entry's first number is the batch.  The dry run records at b = 1 (its CPU stand-ins take about
7 s per scene); the step at batch b calls the same list with b in place of the leading 1, because every per-scene size
of the step (points, samples, neighbours, channels) is independent of b.  The golden holds exactly what the step calls,
so that the dry run and a real step can be compared with it as they stand; the synthetic edge shapes the GPU tests add
are listed here instead, in EDGES and wgrad_edge_shapes (whose one-row-tail row counts are derived from the split plan).
SSD3D_RECORD_TRAIN_SHAPES=1 rewrites the golden."""
import importlib
import importlib.util
import json
import os

import numpy as np
import pytest
import torch

from test_train_grad_cpu import gdry  # noqa: F401  (fixture)
from test_orchestration_cpu import dry  # noqa: F401  (fixture used by gdry)

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "train_backward_shapes.json")
POINTS = 16384

BACKWARD_OPS = ("linear_wgrad", "bn_train_grad", "rowgroup_max_grad", "group_concat_grad", "gather_point_grad",
                "vote_translate_grad")


# ---- call shapes ------------------------------------------------------------------------------------------------------

def _shape(name, a, k):
    """One call as a JSON-able list whose first number is the batch."""
    if name == "linear_wgrad":                     # x (b, .., cin), dz (b, .., cout)
        return list(a[0].shape) + [a[1].shape[-1]]
    if name == "bn_train_grad":                    # x (b, .., c), relu
        return list(a[0].shape) + [int(k.get("relu", True))]
    if name == "rowgroup_max_grad":                # y (b, m, pool, c), rowmask given
        return list(a[0].shape) + [int((a[3] if len(a) > 3 else k.get("rowmask")) is not None)]
    if name == "group_concat_grad":                # grad_x (b, m, ns, ldx), n, c, wanted outputs
        want = list(a[4:7]) + [k[w] for w in ("want_points", "want_xyz", "want_new_xyz") if w in k]
        want += [True] * (3 - len(want))
        return list(a[0].shape) + [int(a[2]), int(a[3])] + [int(bool(w)) for w in want]
    if name == "gather_point_grad":                # inp (b, n, c), idx (b, m)
        return list(a[0].shape) + [a[1].shape[1]]
    if name == "vote_translate_grad":              # offsets (b, n, >= 3)
        return list(a[0].shape)
    if name == "linear_tc_t":                      # d_hi (b, .., kp), W^T fold: K = f.cin (layer cout), N = f.cout
        return list(a[0].shape[:-1]) + [a[2].cin, a[2].cout]
    raise KeyError(name)


class ShapeRecorder:
    """Wraps the backward entry points of tf_ops (and the transposed linear_tc of _ConvTrain.backward) so that every
    call appends [name, shape]; the wrapped functions run unchanged."""

    def __init__(self, T):
        self.T, self.rec, self.orig, self.in_backward = T, [], {}, 0

    def _wrap(self, name, f, only_in_backward=False, as_name=None):
        def wrap(*a, **k):
            if not only_in_backward or self.in_backward:
                self.rec.append([as_name or name, _shape(as_name or name, a, k)])
            return f(*a, **k)
        return wrap

    def __enter__(self):
        T = self.T
        for n in BACKWARD_OPS:
            self.orig[n] = getattr(T, n)
            setattr(T, n, self._wrap(n, self.orig[n]))
        self.orig["linear_tc"] = T.linear_tc
        T.linear_tc = self._wrap("linear_tc", T.linear_tc, only_in_backward=True, as_name="linear_tc_t")
        back = T._ConvTrain.backward

        def backward(ctx, g):
            self.in_backward += 1
            try:
                return back(ctx, g)
            finally:
                self.in_backward -= 1
        self.orig["_ConvTrain.backward"] = T._ConvTrain.__dict__["backward"]
        T._ConvTrain.backward = staticmethod(backward)
        return self

    def __exit__(self, *a):
        for n, f in self.orig.items():
            if n == "_ConvTrain.backward":
                self.T._ConvTrain.backward = f
            else:
                setattr(self.T, n, f)


def time_train():
    spec = importlib.util.spec_from_file_location("time_train", os.path.join(os.path.dirname(HERE), "tools", "time_train.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def record_step(pkg, batch, device):
    """One step of tools/time_train.py (ARCH_3DSSD, kitti_like scenes, the squares loss) with the recorder in place."""
    tt = time_train()
    synth = importlib.import_module("3dssd_b200.synth")
    pts = torch.from_numpy(synth.kitti_like(batch, POINTS, seed=1)).to(device)
    xyz, feat = pkg.tf_ops.split_points(pts)
    tp = tt.trainable(pkg.config.ARCH_3DSSD, device)
    with ShapeRecorder(pkg.tf_ops) as r:
        tt.step(pkg.config.ARCH_3DSSD, tp, xyz, feat)
    return r.rec


def load_shapes(batch=1):
    with open(GOLDEN) as f:
        rec = json.load(f)["calls"]
    return [[n, [batch] + s[1:]] for n, s in rec]


def recorded(name, batch=1):
    """Distinct shapes of one entry point, in first-call order."""
    out = []
    for n, s in load_shapes(batch):
        if n == name and s not in out:
            out.append(s)
    return out


# synthetic shapes beyond the step, run by tests/test_train_backward_gpu.py next to the recorded ones
EDGES = {
    # (rows, c): one column, either side of the 32-wide column block, the widest layer; rows at and past the 256-block
    # cap of the partial sums (512 rows per block)
    "bn_train_grad": [(4099, 1), (4099, 31), (4099, 33), (4099, 1024), (131072, 33), (131073, 33), (300001, 5)],
    # (b, m, pool, c, rowmask): a pool narrower than the planted ties, one column without a rowmask
    "rowgroup_max_grad": [(2, 7, 3, 33, 1), (2, 5, 7, 1, 0)],
    # (b, n, 3): a row count that is not a multiple of the block
    "vote_translate_grad": [(2, 1001, 3)],
}


# ---- the split-K plan of linear_wgrad -------------------------------------------------------------------------------

NUM_SMS, CTAS_PER_SM, WG_BM, WG_BK = 132, 3, 64, 64


def wgrad_bn(cout):
    return 16 if cout <= 16 else (32 if cout <= 32 else 64)


def wgrad_plan(rows, cin, cout):
    """(rows per split, splits) of wgrad_plan in csrc/train_grad.cu."""
    cdiv = lambda a, b: -(-a // b)
    tiles = cdiv(cin, WG_BM) * cdiv(cout, wgrad_bn(cout))
    chunks = cdiv(rows, WG_BK)
    s = max(1, min(cdiv(NUM_SMS * CTAS_PER_SM, tiles), chunks))
    rps = cdiv(chunks, s) * WG_BK
    return rps, max(1, cdiv(rows, rps))


def wgrad_edge_shapes():
    """(rows, cin, cout) beyond the step: tiny row counts, a last split of one row, cout either side of the 16/32/64
    tile widths and cin either side of the 64-row m-tile."""
    out = [(r, 67, 32) for r in (1, 63, 64, 65)]
    out += [(one_row_tail(cin, cout), cin, cout) for cin, cout in ((4, 32), (131, 64), (64, 16))]
    out += [(4099, 64, co) for co in (15, 16, 17, 31, 32, 33, 63, 64, 65)]
    out += [(777, ci, 48) for ci in (64, 65)]
    return out


def one_row_tail(cin, cout, lo=100000):
    """The smallest row count >= lo whose plan ends with a split of exactly one row."""
    rows = lo
    while True:
        rps, splits = wgrad_plan(rows, cin, cout)
        if splits > 1 and rows - (splits - 1) * rps == 1:
            return rows
        rows += 1


def wgrad_shapes(batch=8):
    """Every distinct (rows, cin, cout) of the recorded step at `batch`, then the edges."""
    out = []
    for s in recorded("linear_wgrad", batch):
        t = (int(np.prod(s[:-2])), s[-2], s[-1])
        if t not in out:
            out.append(t)
    return out + [t for t in wgrad_edge_shapes() if t not in out]


def wgrad_magnitude(rows, cin, cout):
    """(A, bound): the integer magnitude of the exact linear_wgrad operands at one shape and the bound, in units of
    2^-8, of one split's fp32 partial.  One operand is an integer in [-A, A], the other an integer in [-A, A] plus k/256,
    so one product is below A (A + 1) units of 2^-8 times 256 and a split adds at most rps of them.  A is the largest of
    3, 2, 1 that keeps the bound below 2^24, where fp32 holds every such sum exactly."""
    rps, _ = wgrad_plan(rows, cin, cout)
    for a in (3, 2, 1):
        bound = rps * a * (a + 1) * 256
        if bound < 2 ** 24:
            return a, bound
    raise AssertionError("no exact operand magnitude for rows=%d cin=%d cout=%d (rows per split %d)" % (rows, cin, cout, rps))


def wgrad_operands(rows, cin, cout, variant, seed, device):
    """Exact float32 operands (x, dz) for linear_wgrad.  variant "x_bf16": x is an integer (exact in bf16, lo = 0) and
    dz = integer + k/256 (hi and lo both carry bits); "dz_bf16": the converse.  hi.hi + lo.hi + hi.lo then carries all
    of x^T dz and the dropped lo.lo is exactly 0.  Column 0 of x and columns 0:16 of dz are non-negative, so the block
    grad_w[0, 0:16] sums non-negative products: at the large row counts its totals exceed 2^24 units although every
    split's partial stays below (a reduce in float would round them)."""
    a, _ = wgrad_magnitude(rows, cin, cout)
    g = torch.Generator(device=device).manual_seed(seed)
    ints = lambda c: torch.randint(-a, a + 1, (rows, c), generator=g, device=device).float()
    frac = lambda c: torch.randint(0, 256, (rows, c), generator=g, device=device).float() / 256
    x, dz = ints(cin), ints(cout)
    x[:, 0] = x[:, 0].abs()
    dz[:, :16] = dz[:, :16].abs()
    if variant == "x_bf16":
        dz += frac(cout)
    else:
        x += frac(cin)
    return x, dz


# ---- tests ----------------------------------------------------------------------------------------------------------

def test_wgrad_plan_matches_workspace_query(pkg):
    q = pkg.lib().ssd3d_linear_wgrad_workspace
    shapes = wgrad_shapes(8) + wgrad_shapes(1) + [(r, ci, co) for r in (1, 64, 65, 4095, 4096, 4097, 2 ** 21 + 37)
                                                   for ci in (1, 4, 64, 65, 1536) for co in (1, 3, 16, 17, 64, 65, 512)]
    seen = set()
    for rows, cin, cout in shapes:
        rps, splits = wgrad_plan(rows, cin, cout)
        assert rps % WG_BK == 0 and (splits - 1) * rps < rows <= splits * rps, (rows, cin, cout)
        assert q(rows, cin, cout) == splits * cout * (8 + 4 * cin), (rows, cin, cout, rps, splits)
        seen.add(splits)
    assert max(seen) > 300 and 1 in seen                     # the layer-1 shape splits ~400 ways; tiny row counts once
    assert wgrad_plan(8 * 4096 * 64, 4, 32) == (5312, 395)   # layer-1 conv0_0 at b = 8: 2,097,152 rows
    for rows, cin, cout in wgrad_edge_shapes():
        if rows >= 100000:
            rps, splits = wgrad_plan(rows, cin, cout)
            assert rows - (splits - 1) * rps == 1


def wgrad_block_total(rows, cin, cout):
    """Expected value, in units of 2^-8, of one entry of the non-negative block grad_w[0, 0:16] of wgrad_operands (either
    variant): rows * E|i| * (E|i| + E[k/256]) with i uniform on -A..A and k uniform on 0..255."""
    a, _ = wgrad_magnitude(rows, cin, cout)
    e_int = a * (a + 1) / (2 * a + 1)
    return rows * e_int * (e_int + 255 / 512) * 256


def test_wgrad_operand_bounds_at_every_shape():
    """Every shape the GPU test runs has an exact operand magnitude: one split's fp32 partial stays below 2^24 units of
    2^-8 (wgrad_magnitude raises otherwise).  At the layer-1 shapes (>= 2^20 rows, ~400 splits) the expected total of
    the non-negative block is at least 8 times 2^24 units, so its cross-split sums cannot all be exact in fp32: a reduce
    in float would round them where the double reduce does not (the GPU test asserts the realised totals as well)."""
    big = []
    for rows, cin, cout in wgrad_shapes(8):
        _, bound = wgrad_magnitude(rows, cin, cout)
        assert bound < 2 ** 24
        if rows >= 2 ** 20:
            assert wgrad_block_total(rows, cin, cout) > 8 * 2 ** 24, (rows, cin, cout)
            big.append((rows, cin, cout))
    assert len(big) == 6 and (2097152, 4, 32) in big


@pytest.mark.parametrize("variant", ["x_bf16", "dz_bf16"])
def test_wgrad_operands_are_exact(variant):
    """The operand construction of the GPU test: both values are float32, hi + lo = value for the bf16 split, one of
    the two lo terms is zero everywhere and the other is not, and the block grad_w[0, 0:16] sums non-negative products."""
    for i, (rows, cin, cout) in enumerate([(4099, 64, 33), (777, 65, 48), (65, 67, 32), (100609, 131, 64)]):
        x, dz = wgrad_operands(rows, cin, cout, variant, i, "cpu")
        hi = [t.to(torch.bfloat16).float() for t in (x, dz)]
        lo = [(t - h).to(torch.bfloat16).float() for t, h in zip((x, dz), hi)]
        for t, h, l in zip((x, dz), hi, lo):
            assert torch.equal(h + l, t)
        assert (lo[0].abs().max() == 0) != (lo[1].abs().max() == 0)
        assert (x[:, 0] >= 0).all() and (dz[:, :16] >= 0).all()


def test_dry_step_calls_the_pinned_backward_shapes(gdry, monkeypatch):
    """The backward of one ARCH_3DSSD step of tools/time_train.py at b = 1 x 16384 points through the CPU dry fixture
    calls exactly the pinned shapes.  gather_point goes through the real autograd Function here (the gdry fixture
    replaces it with a torch gather), with float64 stand-ins of its forward and backward."""
    pkg = gdry
    T = pkg.tf_ops

    def gather_point(inp, idx):
        if inp.requires_grad and torch.is_grad_enabled():
            return T._GatherPoint.apply(inp, idx)
        return T._gather_point_fwd(inp, idx)

    def gather_point_grad(inp, idx, out_g):
        b, n, c = inp.shape
        flat = (idx.long() + torch.arange(b).view(b, 1) * n).reshape(-1)
        return torch.zeros(b * n, c, dtype=torch.float64).index_add_(0, flat, out_g.reshape(-1, c).double()).float().view(b, n, c)

    from test_train_grad_cpu import gather_rows
    monkeypatch.setattr(T, "_gather_point_fwd", lambda inp, idx: gather_rows(inp.detach(), idx))
    monkeypatch.setattr(T, "gather_point", gather_point)
    monkeypatch.setattr(T, "gather_point_grad", gather_point_grad)
    rec = record_step(pkg, 1, "cpu")
    if os.environ.get("SSD3D_RECORD_TRAIN_SHAPES"):
        head = {"batch": 1, "points": POINTS, "arch": "ARCH_3DSSD",
                "note": "backward calls of one tools/time_train.py step in call order; the first number of every shape is "
                        "the batch (tests/test_train_backward_cpu.py)"}
        with open(GOLDEN, "w") as f:
            f.write(json.dumps(head)[:-1] + ', "calls": [\n' + ",\n".join(json.dumps(c) for c in rec) + "\n]}\n")
    assert rec == load_shapes(1)
    names = {n for n, _ in rec}
    assert names == set(BACKWARD_OPS) | {"linear_tc_t"}
