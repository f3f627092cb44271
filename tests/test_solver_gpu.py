"""GPU checks of the solver (csrc/solver.cu, 3dssd_b200/solver.py, DESIGN.md section 3.11): the Adam kernel and the
operand rebuild bit for bit against oracle/solver.py and params.FoldedConv, the operand cache against the uncached
forward, resume from a checkpoint, the scheduled BatchNorm decay reaching the layers, a short training run, and a Trainer
over a given DataParallel (world 1; fresh process and CTA bound as in test_data_parallel_gpu.py) against the oracles of
the exchange and of Adam chained."""
import importlib
import os

import numpy as np
import pytest
import torch

from oracle import data_parallel as ODP
from oracle import solver as O
from test_backbone_gpu import scaled_arch
from test_data_parallel_gpu import N, sim_ctas

pytestmark = pytest.mark.gpu
synth = importlib.import_module("3dssd_b200.synth")
S = importlib.import_module("3dssd_b200.solver")
F = np.float32


def same_bits(got, want, what):
    """Equal bit patterns; a NaN matches any NaN (the payload of a generated NaN is the hardware's)."""
    g, w = np.ascontiguousarray(got).reshape(-1), np.ascontiguousarray(want).reshape(-1)
    assert g.dtype.itemsize == w.dtype.itemsize and g.size == w.size, what
    it = {2: np.uint16, 4: np.uint32, 8: np.uint64}[g.dtype.itemsize]
    bad = g.view(it) != w.view(it)
    if g.dtype.kind == "f":
        bad &= ~(np.isnan(g) & np.isnan(w))
    idx = np.flatnonzero(bad)
    assert idx.size == 0, "%s: %d of %d differ, first at %d: %r vs %r" % (what, idx.size, g.size, idx[0], g[idx[0]], w[idx[0]])


def isolated(call):
    """Run `call` over this module's functions in a fresh process with eager module loading (test_data_parallel_gpu.py)."""
    import subprocess
    import sys
    tests = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(tests)
    code = ("import sys; sys.path[:0] = [%r, %r]; import importlib, torch; import test_solver_gpu as t; "
            "pkg = importlib.import_module('3dssd_b200'); cuda = torch.device('cuda:0'); t.%s" % (root, tests, call))
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, CUDA_MODULE_LOADING="EAGER"), cwd=root,
                       capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, (r.stdout[-3000:] + "\n" + r.stderr[-6000:])


def _model(pkg, arch, seed=5):
    d = pkg.params.init_params(arch, 1, seed=seed, random_bias=True)
    d.update(pkg.params.init_head_params(pkg.config.layer_channels(arch, 1)[-1], seed=seed + 1))
    return d


def _scenes(pkg, cuda, batch, npoints, seed):
    p, b, l = synth.kitti_like_with_boxes(batch, npoints, 20, seed=seed)
    pts, boxes, labels = (torch.from_numpy(a).to(cuda) for a in (p, b, l))
    xyz, feat = pkg.tf_ops.split_points(pts)
    return xyz, feat, boxes, labels


def _special_grad(rng, n, scale):
    g = (rng.standard_normal(n) * scale).astype(F)
    special = np.array([0.0, -0.0, 1e-42, -3e-45, np.inf, -np.inf, np.nan, 1e-30, 3e38], F)
    g[: min(n, special.size)] = special[: min(n, special.size)]
    return g


@pytest.mark.parametrize("n", [2513858, 1003, 2])
def test_adam_step_bitwise(pkg, cuda, n):
    """Three launches over a schedule whose boundary lies between them (lr changes at the third), gradients with zeros,
    denormals, infinities and NaN; the state block after each launch; then the same three launches as one CUDA graph."""
    T = pkg.tf_ops
    rng = np.random.default_rng(n)
    boundaries, values = (1,), (0.002, 0.0005)
    p0 = rng.standard_normal(n).astype(F)
    grads = [_special_grad(rng, n, s) for s in (0.1, 1e-6, 3.0)]
    dev = lambda a: torch.from_numpy(np.array(a, copy=True)).to(cuda)

    def fresh():
        return dev(p0), torch.zeros(n, device=cuda), torch.zeros(n, device=cuda), dev(S.pack_state(0, F(0.9), F(0.999)))

    p, m, v, st = fresh()
    g = torch.zeros(n, device=cuda)
    op, om, ov, ost = p0, np.zeros(n, F), np.zeros(n, F), O.new_state()
    want = []
    for i, gi in enumerate(grads):
        g.copy_(dev(gi))
        T.adam_step(p, g, m, v, st, boundaries, values)
        op, om, ov, ost = O.adam_step(op, gi, om, ov, ost, boundaries, values)
        want.append((op, om, ov, ost))
        for name, got, exp in (("param", p, op), ("m", m, om), ("v", v, ov)):
            same_bits(N(got), exp, "n=%d launch %d %s" % (n, i, name))
        words = N(st)
        assert S.unpack_state(words) == (ost["global_step"], ost["beta1_power"], ost["beta2_power"], ost["lr_used"]), (i, words)
        assert (words[5:] == 0).all()
    assert [w[3]["lr_used"] for w in want] == [F(0.002), F(0.002), F(0.0005)]
    if n > 9:                                                        # Inf / NaN gradients poison their own element only
        assert np.isnan(op[4:7]).all() and np.isfinite(op[:4]).all() and np.isfinite(op[9:]).all()

    p, m, v, st = fresh()
    gs = [dev(gi) for gi in grads]
    graph = torch.cuda.CUDAGraph()
    stream = torch.cuda.Stream(device=cuda)
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        with torch.cuda.graph(graph, stream=stream):
            for gi in gs:
                T.adam_step(p, gi, m, v, st, boundaries, values)
    torch.cuda.synchronize()
    same_bits(N(p), p0, "capture runs nothing")
    graph.replay()
    torch.cuda.synchronize()
    for name, got, exp in (("param", p, op), ("m", m, om), ("v", v, ov)):
        same_bits(N(got), exp, "n=%d graph %s" % (n, name))
    assert S.unpack_state(N(st))[0] == 3


def test_adam_step_rejects_bad_arguments(pkg, cuda):
    T = pkg.tf_ops
    z = lambda n: torch.zeros(n, device=cuda)
    st = torch.from_numpy(S.pack_state(0, 0.9, 0.999)).to(cuda)
    with pytest.raises(ValueError):
        T.adam_step(z(8), z(8), z(8), z(7), st, (), (0.1,))
    with pytest.raises(ValueError):
        T.adam_step(z(8), z(8), z(8), z(8), st, (3, 2), (0.1, 0.1, 0.1))
    with pytest.raises(ValueError):
        T.adam_step(z(9)[1:], z(8), z(8), z(8), st, (), (0.1,))
    with pytest.raises(ValueError):
        T.adam_step(z(8), z(8), z(8), z(8), st, tuple(range(9)), (0.1,) * 10)


def test_weight_operands_bitwise_after_a_step(pkg, cuda):
    """Every weight of ARCH_3DSSD + head (cin 4, 67, 131, 259 ...: the paddings that are not multiples of 16), read
    straight after an adam_step on the same stream: both operands equal params.FoldedConv's, padding included."""
    P = pkg.params
    arch = pkg.config.ARCH_3DSSD
    tp = P.TrainableParams(_model(pkg, arch), cuda)
    adam = S.Adam(tp, S.Solver())
    assert adam.param.numel() == 2513858
    first = tp.operand_arena.clone()
    g = torch.Generator(device=cuda).manual_seed(1)
    adam.grad.copy_(torch.randn(adam.grad.shape, generator=g, device=cuda) * 0.1)
    adam.step()
    assert not torch.equal(first, tp.operand_arena)
    seen = set()
    for scope in tp.weight_scopes():
        w = tp.tensors[scope + "/weights"].detach()
        cin, cout = w.shape
        seen.add(cin)
        fwd, bwd = tp.operand_cache[scope]
        ones = lambda c: torch.ones(c, device=cuda)
        ref_f, ref_b = P.FoldedConv(w, ones(cout), ones(cout)), P.FoldedConv(w.t().contiguous(), ones(cin), ones(cin))
        for name, got, exp in (("fwd hi", fwd.b_hi, ref_f.b_hi), ("fwd lo", fwd.b_lo, ref_f.b_lo),
                               ("bwd hi", bwd.b_hi, ref_b.b_hi), ("bwd lo", bwd.b_lo, ref_b.b_lo)):
            assert got.shape == exp.shape and got.is_contiguous(), (scope, name)
            same_bits(N(got.view(torch.int16)), N(exp.view(torch.int16)), "%s %s" % (scope, name))
        hi, lo = O.split_operand(N(w))
        same_bits(N(fwd.b_hi.view(torch.int16)), hi, scope + " oracle hi"); same_bits(N(fwd.b_lo.view(torch.int16)), lo, scope + " oracle lo")
        assert fwd.kp == P.round16(cin) and bwd.kp == P.round16(cout) and fwd.cout == cout and bwd.cout == cin
        b = tp.tensors.get(scope + "/biases")
        assert b is None or fwd.shift.data_ptr() == b.data_ptr()          # the live bias, not a copy
    assert {4, 67, 131, 259} <= seen


def _forward_backward(pkg, arch, tp, scene, bn_decay=None):
    xyz, feat, boxes, labels = scene
    o = pkg.backbone.train_forward(arch, tp, xyz, feat, bn_decay=bn_decay)
    tg = pkg.loss.assign_targets(o.base_xyz, o.vote_base, boxes, labels)
    losses = pkg.loss.detection_loss(o.base_xyz, *o.head, o.vote_offsets[-1], tg)
    losses["total"].backward()
    return o, losses


def test_operand_cache_gives_the_uncached_forward(pkg, cuda):
    """Same weights, with and without the cache: the forward is bit-identical (outputs, losses, moving statistics).  The
    gradients are held to 1e-3 of each tensor's largest entry (biases before BN: 1e-5 of the weight gradient's), the
    bound of the backward tests: group_concat_grad and
    gather_point_grad accumulate with float atomics, so two runs of the SAME path already differ in the last bits."""
    arch = scaled_arch(pkg, 8)
    d = _model(pkg, arch)
    scene = _scenes(pkg, cuda, 2, 2048, seed=3)
    plain, cached = pkg.params.TrainableParams(d, cuda), pkg.params.TrainableParams(d, cuda)
    cached.enable_operand_cache()
    calls = []
    orig = pkg.params.FoldedConv.__init__
    try:
        pkg.params.FoldedConv.__init__ = lambda self, *a: (calls.append(1), orig(self, *a))[1]
        oc, lc = _forward_backward(pkg, arch, cached, scene)
        assert not calls                                                 # no operand was built on the way
        op, lp = _forward_backward(pkg, arch, plain, scene)
        assert len(calls) >= len(plain.weight_scopes())                  # one per forward, one per grad-x
    finally:
        pkg.params.FoldedConv.__init__ = orig
    for a, b in zip(list(oc.head) + list(oc.vote_offsets), list(op.head) + list(op.vote_offsets)):
        same_bits(N(a), N(b), "forward output")
    for k in lp:
        same_bits(N(lc[k]).reshape(1), N(lp[k]).reshape(1), "loss " + k)
    for k, t in plain.tensors.items():
        if not t.requires_grad:
            same_bits(N(cached.tensors[k]), N(t), k)
    for (k, a), (_, b) in zip(cached.named_parameters(), plain.named_parameters()):
        assert a.grad is not None and b.grad is not None, k
        err, bound = (a.grad - b.grad).abs().max().item(), 1e-3 * b.grad.abs().max().item()
        scope = k[: -len("/biases")]
        if k.endswith("/biases") and scope + "/bn/gamma" in plain.tensors:   # a bias before BatchNorm has gradient 0 up to
            bound = 1e-5 * plain.tensors[scope + "/weights"].grad.abs().max().item()   # rounding: held to the weight's scale
        assert err <= bound + 1e-12, (k, err, bound)


def _trainer(pkg, cuda, arch, d, solver):
    return S.Trainer(arch, pkg.params.TrainableParams(d, cuda), solver)


def _everything(tr):
    out = {k: N(t) for k, t in tr.tp.tensors.items()}
    out.update(m=N(tr.adam.m), v=N(tr.adam.v), state=N(tr.adam.state), arena=N(tr.tp.operand_arena.view(torch.int16)),
               flat=N(tr.adam.param))
    return out


def test_resume_is_bit_for_bit(pkg, cuda, tmp_path):
    """Three steps, save, load into fresh objects: every tensor is identical, and one more Adam step from the SAME
    injected gradient gives identical results.  (A recomputed training step cannot be compared bit for bit: its backward
    accumulates with float atomics.)"""
    arch = scaled_arch(pkg, 8)
    solver = S.Solver(steps=(1,))
    a = _trainer(pkg, cuda, arch, _model(pkg, arch), solver)
    for i in range(3):
        a.step(*_scenes(pkg, cuda, 2, 2048, seed=10 + i))
    path = str(tmp_path / "model-00000003.npz")
    a.save(path)
    b = _trainer(pkg, cuda, arch, _model(pkg, arch, seed=50), solver)
    assert not np.array_equal(N(b.adam.param), N(a.adam.param))
    b.load(path)
    torch.cuda.synchronize()
    assert b.global_step == a.global_step == 3 and S.unpack_state(N(b.adam.state)) == S.unpack_state(N(a.adam.state))
    ea, eb = _everything(a), _everything(b)
    assert set(ea) == set(eb)
    for k in ea:
        same_bits(eb[k], ea[k], "after load: " + k)
    g = torch.randn(a.adam.grad.shape, generator=torch.Generator(device=cuda).manual_seed(4), device=cuda) * 0.05
    for tr in (a, b):
        tr.adam.grad.copy_(g)
        tr.adam.step()
    ea, eb = _everything(a), _everything(b)
    for k in ea:
        same_bits(eb[k], ea[k], "one step after load: " + k)
    assert S.unpack_state(ea["state"])[3] == solver.learning_rate(3) == F(0.002 * 0.1)
    with np.load(path) as z:                                            # the file is a model for the inference path as it is
        prm = pkg.kitti_io.params_from_tf_variables({k: z[k] for k in z.files})
    assert set(prm) == set(a.tp.tensors)


def test_scheduled_bn_decay_reaches_every_layer(pkg, cuda):
    """steps=(1,): the forwards at global_step 0 and 1 use decay 0.5, the one at step 2 uses 0.75.  The batch statistics
    come from the exchange's BN record; the moving statistics must equal the oracle's update at exactly those decays."""
    arch = scaled_arch(pkg, 8)
    solver = S.Solver(steps=(1,))
    tr = _trainer(pkg, cuda, arch, _model(pkg, arch), solver)
    stats = N(tr.tp.stats_flat).copy()
    for step, decay in enumerate((0.5, 0.5, 0.75)):
        assert float(solver.bn_decay(step)) == decay
        tr.step(*_scenes(pkg, cuda, 2, 2048, seed=20 + step))
        h = pkg.dist._HEAD_FLOATS
        record = N(tr.dp.gathered[:, h:h + tr.dp.nstats]).copy()
        want = ODP.bn_update(stats, record, decay)
        assert not np.array_equal(want, ODP.bn_update(stats, record, 0.9))
        same_bits(N(tr.tp.stats_flat), want, "moving statistics after step %d" % step)
        stats = want
    assert tr.dp.timeouts() == 0


def test_it_trains(pkg, cuda):
    """Two fixed scenes, the 1/8-scale model, 20 steps at the reference's 0.002: the loss goes down and nothing blows up."""
    arch = scaled_arch(pkg, 8)
    tr = _trainer(pkg, cuda, arch, _model(pkg, arch), S.Solver())
    scene = _scenes(pkg, cuda, 2, 2048, seed=31)
    totals = [tr.step(*scene)["total"] for _ in range(20)]
    totals = [float(t) for t in totals]
    assert np.isfinite(totals).all(), totals
    assert np.mean(totals[-5:]) < np.mean(totals[:5]), totals
    assert torch.isfinite(tr.adam.param).all() and torch.isfinite(tr.tp.stats_flat).all()
    assert S.unpack_state(N(tr.adam.state))[0] == tr.global_step == 20


def test_world_one_trainer_through_a_given_data_parallel():
    isolated("replicas(pkg, cuda, 1)")


def replicas(pkg, cuda, world, steps=3):
    """`world` ranks simulated on one device (streams, plain allocations as symmetric buffers, CTAs bounded by
    dist.simulated_ctas so every spinning CTA's peers are placed), each a Trainer over its own DataParallel, fed RECORDED
    per-rank gradients and BN records: after three exchanges + Adam steps the replicas hold the same bits, and rank 0
    equals the oracle's exchange followed by the oracle's Adam."""
    D = pkg.dist
    arch = scaled_arch(pkg, 8)
    ctas = sim_ctas(pkg, world)
    d = _model(pkg, arch)
    tps = [pkg.params.TrainableParams(d, cuda) for _ in range(world)]
    nbytes = D.DataParallel.symmetric_bytes(tps[0], world, ctas)
    sym = [torch.zeros((nbytes,), dtype=torch.uint8, device=cuda) for _ in range(world)]
    dps = [D.DataParallel(tp, peers=[t.data_ptr() for t in sym], world=world, rank=r, ctas=ctas) for r, tp in enumerate(tps)]
    solver = S.Solver(steps=(1,))
    trs = [S.Trainer(arch, tp, solver, dp) for tp, dp in zip(tps, dps)]
    streams = [torch.cuda.Stream(device=cuda) for _ in range(world)]
    n, ns = trs[0].adam.param.numel(), dps[0].nstats
    rng = np.random.default_rng(world)
    op, om, ov, ost = N(trs[0].adam.param).copy(), np.zeros(n, F), np.zeros(n, F), O.new_state()
    ostats = N(tps[0].stats_flat).copy()
    zero = torch.zeros((), device=cuda)
    losses = {k: zero for k in pkg.loss.LOSS_NAMES + ("total",)}
    for step in range(steps):
        grads = [(rng.standard_normal(n) * (0.01 if (r + step) % 2 else 0.5)).astype(F) for r in range(world)]
        records = [rng.uniform(0.1, 1.0, ns).astype(F) for _ in range(world)]
        decay = float(solver.bn_decay(step))
        for r in range(world):
            dps[r].grad.copy_(torch.from_numpy(grads[r]))
            dps[r].record.copy_(torch.from_numpy(records[r]))
            dps[r].decay = decay                                         # what recording() leaves behind
        torch.cuda.synchronize()
        for r in reversed(range(world)):                                 # launch order != rank order
            with torch.cuda.stream(streams[r]):
                dps[r].exchange(losses)
        torch.cuda.synchronize()
        mean, ostats, _, _ = ODP.exchange(grads, records, ostats, decay)
        for r in range(world):
            same_bits(N(dps[r].grad), mean, "mean gradient rank %d step %d" % (r, step))
            with torch.cuda.stream(streams[r]):
                trs[r].adam.step()
        torch.cuda.synchronize()
        op, om, ov, ost = O.adam_step(op, mean, om, ov, ost, solver.steps, solver.lr_values())
    for r in range(world):
        same_bits(N(trs[r].adam.param), op, "parameters rank %d" % r)
        same_bits(N(trs[r].adam.m), om, "m rank %d" % r); same_bits(N(trs[r].adam.v), ov, "v rank %d" % r)
        same_bits(N(tps[r].stats_flat), ostats, "statistics rank %d" % r)
        same_bits(N(tps[r].operand_arena.view(torch.int16)), N(tps[0].operand_arena.view(torch.int16)), "arena rank %d" % r)
        assert S.unpack_state(N(trs[r].adam.state))[:3] == (steps, ost["beta1_power"], ost["beta2_power"])
    ref = pkg.params.FoldedConv(tps[0].tensors["layer1/conv0_0/weights"].detach(), torch.ones(16, device=cuda), torch.ones(16, device=cuda))
    same_bits(N(tps[0].operand_cache["layer1/conv0_0"][0].b_hi.view(torch.int16)), N(ref.b_hi.view(torch.int16)), "arena is current")
    assert sum(dp.timeouts() for dp in dps) == 0
