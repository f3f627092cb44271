"""GPU checks of fine-tuning and the Momentum solver (DESIGN.md section 3.19): ssd3d_momentum_step bit for bit against
the float32 restatement of test_finetune_cpu.py; three Trainer steps on the real-scan scenes with the candidate-generation
layer and the head trained and everything below frozen (frozen tensors unchanged, their moving statistics those of plain
training forwards, step-0 gradients and clip norm those of the trained tensors of a full step); layer 1 trained under
frozen layers (the dgrad-only path); the backward's entry points with and without a frozen set; resume bit for bit with
Adam and Momentum; and two simulated data-parallel ranks over a frozen set, with and without SyncBN."""
import importlib
import json
import os

import numpy as np
import pytest
import torch

from oracle import data_parallel as ODP
from test_data_parallel_gpu import N, sim_ctas
from test_finetune_cpu import TOP, model, momentum_step
from test_realscan_cpu import realscan_scenes
from test_solver_gpu import _special_grad, same_bits

pytestmark = pytest.mark.gpu
S = importlib.import_module("3dssd_b200.solver")
F = np.float32
BOTTOM = ("layer1", "layer2", "layer3", "vote")


def isolated(call):
    """Run `call` over this module's functions in a fresh process with eager module loading (test_data_parallel_gpu.py)."""
    import subprocess
    import sys
    tests = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(tests)
    code = ("import sys; sys.path[:0] = [%r, %r]; import importlib, torch; import test_finetune_gpu as t; "
            "pkg = importlib.import_module('3dssd_b200'); cuda = torch.device('cuda:0'); t.%s" % (root, tests, call))
    r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, CUDA_MODULE_LOADING="EAGER"), cwd=root,
                       capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, (r.stdout[-3000:] + "\n" + r.stderr[-6000:])


@pytest.mark.parametrize("n", [2513858, 1003, 2])
def test_momentum_step_bitwise(pkg, cuda, n):
    """Three launches over a schedule whose boundary lies between them, gradients with zeros, denormals, infinities and
    NaN; the state block after each launch (beta powers untouched); then the same launches as one CUDA graph."""
    T = pkg.tf_ops
    rng = np.random.default_rng(n)
    boundaries, values = (1,), (0.002, 0.0005)
    p0 = rng.standard_normal(n).astype(F)
    grads = [_special_grad(rng, n, s) for s in (0.1, 1e-6, 3.0)]
    dev = lambda a: torch.from_numpy(np.array(a, copy=True)).to(cuda)
    fresh = lambda: (dev(p0), torch.zeros(n, device=cuda), dev(S.pack_state(0, F(0.25), F(0.5))))
    p, a, st = fresh()
    op, oa, ost = p0, np.zeros(n, F), {"global_step": 0}
    g = torch.zeros(n, device=cuda)
    for i, gi in enumerate(grads):
        g.copy_(dev(gi))
        T.momentum_step(p, g, a, st, boundaries, values, momentum=0.9)
        op, oa, ost = momentum_step(op, gi, oa, ost, boundaries, values, 0.9)
        same_bits(N(p), op, "n=%d launch %d param" % (n, i))
        same_bits(N(a), oa, "n=%d launch %d accum" % (n, i))
        words = N(st)
        assert S.unpack_state(words) == (ost["global_step"], F(0.25), F(0.5), ost["lr_used"]), (i, words)
        assert (words[5:] == 0).all()
    assert ost["lr_used"] == F(0.0005)
    if n > 9:                                                        # Inf / NaN gradients poison their own element only
        assert not np.isfinite(op[4:7]).any() and np.isfinite(op[:4]).all() and np.isfinite(op[9:]).all()

    p, a, st = fresh()
    gs = [dev(gi) for gi in grads]
    graph, stream = torch.cuda.CUDAGraph(), torch.cuda.Stream(device=cuda)
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        with torch.cuda.graph(graph, stream=stream):
            for gi in gs:
                T.momentum_step(p, gi, a, st, boundaries, values, momentum=0.9)
    graph.replay()
    torch.cuda.synchronize()
    same_bits(N(p), op, "graph param")
    same_bits(N(a), oa, "graph accum")
    assert S.unpack_state(N(st))[0] == 3


def test_momentum_step_rejects_bad_arguments(pkg, cuda):
    T = pkg.tf_ops
    z = lambda n: torch.zeros(n, device=cuda)
    st = torch.from_numpy(S.pack_state(0, 0, 0)).to(cuda)
    for bad in (lambda: T.momentum_step(z(8), z(8), z(7), st, (), (0.1,)),
                lambda: T.momentum_step(z(8), z(8), z(8), st, (3, 2), (0.1, 0.1, 0.1)),
                lambda: T.momentum_step(z(9)[1:], z(8), z(8), st, (), (0.1,)),
                lambda: T.momentum_step(z(8), z(8), z(8), st, tuple(range(9)), (0.1,) * 10)):
        with pytest.raises(ValueError):
            bad()


# ---- training on the real-scan scenes ---------------------------------------------------------------------------------
def real_batch(pkg, cuda, step, batch=4):
    """`batch` of the eight real-scan scenes (step 0: S0-S3, step 1: S4-S7, ...) with car boxes standing around some of
    their points, so that every scene has positives."""
    pts = realscan_scenes()[0]
    idx = [(step * batch + i) % len(pts) for i in range(batch)]
    p = np.ascontiguousarray(pts[idx])
    boxes = np.zeros((batch, 8, 7), F)
    labels = np.zeros((batch, 8), np.int32)
    for s in range(batch):
        rng = np.random.default_rng(100 + idx[s])
        for j, r in enumerate(rng.choice(p.shape[1], 8, replace=False)):
            x, y, z = p[s, r, :3]
            boxes[s, j] = (x, y + 0.78, z, 3.9, 1.56, 1.6, rng.uniform(-np.pi, np.pi))
            labels[s, j] = 1
    xyz, feat = pkg.tf_ops.split_points(torch.from_numpy(p).to(cuda))
    return xyz, feat, torch.from_numpy(boxes).to(cuda), torch.from_numpy(labels).to(cuda)


def trainer(pkg, cuda, trainable=None, solver=None, seed=5):
    tp = pkg.params.TrainableParams(model(pkg, seed), cuda, trainable=trainable)
    return S.Trainer(pkg.config.ARCH_3DSSD, tp, solver or S.Solver(steps=(1,)))


class PreClip:
    """Snapshots of the flat gradient as the backward left it, before the exchange clips and averages it."""

    def __init__(self, tr):
        self.grads, orig = [], tr.dp.exchange

        def exchange(losses):
            self.grads.append(tr.dp.grad.clone())
            return orig(losses)
        tr.dp.exchange = exchange


def per_tensor(tr, flat):
    return {k: flat[o:o + tr.tp.tensors[k].numel()] for k, o in tr.tp.grad_offsets.items()}


def test_trained_on_top_frozen_below(pkg, cuda):
    """trainable = CG layer + head, three steps: frozen tensors keep their bits; the moving statistics of layers 1-3 and
    the vote layer are those of three plain training forwards of the initial weights at the same decays; the step-0
    gradient of every trained tensor equals the full step's bit for bit (no atomic scatter lies between these weights
    and the loss) and the clip norm is the norm over those tensors alone."""
    d = model(pkg)
    tr = trainer(pkg, cuda, TOP)
    full = trainer(pkg, cuda)
    snap, fsnap = PreClip(tr), PreClip(full)
    init = {k: N(t).copy() for k, t in tr.tp.tensors.items()}
    for step in range(3):
        tr.step(*real_batch(pkg, cuda, step))
        if step == 0:
            norm0 = float(tr.dp.norms()[0])
    full.step(*real_batch(pkg, cuda, 0))
    torch.cuda.synchronize()
    frozen = tr.tp.frozen_names()
    assert frozen and all(k.startswith(BOTTOM) for k in frozen)
    for k in frozen:
        same_bits(N(tr.tp.tensors[k]), init[k], "frozen " + k)
        assert tr.tp.tensors[k].grad is None, k
    for k in tr.tp.weight_scopes():
        assert not np.array_equal(N(tr.tp.tensors[k + "/weights"]), init[k + "/weights"]), "trained %s did not move" % k

    plain = pkg.params.TrainableParams(d, cuda)
    with torch.no_grad():
        for step in range(3):
            xyz, feat, _, _ = real_batch(pkg, cuda, step)
            pkg.backbone.train_forward(pkg.config.ARCH_3DSSD, plain, xyz, feat, bn_decay=float(tr.solver.bn_decay(step)))
    for s in tr.tp.bn_scopes():
        if s.startswith(BOTTOM):
            for suf in tr.tp._STATS:
                same_bits(N(tr.tp.tensors[s + suf]), N(plain.tensors[s + suf]), "moving statistics " + s + suf)

    g, gf = per_tensor(tr, snap.grads[0]), per_tensor(full, fsnap.grads[0])
    for k, t in g.items():
        same_bits(N(t), N(gf[k]), "step-0 gradient " + k)
    g64 = N(snap.grads[0]).astype(np.float64)
    want = np.sqrt((g64 * g64).sum())
    full64 = N(fsnap.grads[0]).astype(np.float64)
    assert abs(norm0 - want) <= 1e-5 * want, (norm0, want)
    assert np.sqrt((full64 * full64).sum()) > want * (1 + 1e-4)           # the frozen tensors' share is really left out


def test_trained_at_the_bottom_frozen_above(pkg, cuda):
    """trainable = layer 1: the gradient reaches it through frozen layers (dgrad only).  Its step-0 gradients equal a full
    step's to within the spread of two identical full steps (the group-point scatter adds with float atomics); the frozen
    tensors get no gradient."""
    tr = trainer(pkg, cuda, ["layer1"])
    fulls = [trainer(pkg, cuda) for _ in range(2)]
    snaps = [PreClip(t) for t in [tr] + fulls]
    batch = real_batch(pkg, cuda, 0)
    for t in [tr] + fulls:
        t.step(*batch)
    torch.cuda.synchronize()
    g = per_tensor(tr, snaps[0].grads[0])
    f1, f2 = per_tensor(fulls[0], snaps[1].grads[0]), per_tensor(fulls[1], snaps[2].grads[0])
    assert set(g) == {k for k in tr.tp.tensors if k.startswith("layer1/") and not k.endswith(tr.tp._STATS)}
    for k in g:
        a, b, c = N(g[k]).astype(np.float64), N(f1[k]).astype(np.float64), N(f2[k]).astype(np.float64)
        spread = np.abs(b - c).max()
        scale = np.abs(b).max()
        err = np.abs(a - b).max()
        assert err <= 4 * spread + 1e-6 * scale + 1e-30, (k, err, spread, scale)
    for k in tr.tp.frozen_names():
        assert tr.tp.tensors[k].grad is None, k


class Recorder:
    """tf_ops.lib wrapped by a stand-in that records each entry point called (with its arguments) and passes it through."""

    def __init__(self, T):
        self.T, self.calls, self.real = T, [], T.lib

    def __getattr__(self, name):
        f = getattr(self.real(), name)

        def fn(*a):
            self.calls.append((name, a))
            return f(*a)
        return fn

    def __enter__(self):
        self.T.lib = lambda: self
        return self

    def __exit__(self, *a):
        self.T.lib = self.real


def backward_trace(pkg, cuda, trainable):
    """One training step of a Trainer with `trainable`, the backward's library calls recorded; also (scope, rows, cin,
    cout) of every conv of the forward."""
    tr = trainer(pkg, cuda, trainable)
    xyz, feat, boxes, labels = real_batch(pkg, cuda, 0)
    convs, orig = [], tr.tp.conv_train

    def conv_train(scope, x, *a, **k):
        convs.append((scope, x.numel() // x.shape[-1]) + tuple(tr.tp.tensors[scope + "/weights"].shape))
        return orig(scope, x, *a, **k)
    tr.tp.conv_train = conv_train
    tr.dp.zero_grad()
    with tr.dp.recording():
        o = pkg.backbone.train_forward(tr.arch, tr.tp, xyz, feat, bn_decay=0.5)
    tg = pkg.loss.assign_targets(o.base_xyz, o.vote_base, boxes, labels)
    losses = pkg.loss.detection_loss(o.base_xyz, *o.head, o.vote_offsets[-1], tg)
    with Recorder(pkg.tf_ops) as rec:
        losses["total"].backward()
    torch.cuda.synchronize()
    tr.dp.exchange(losses)
    return tr, convs, rec.calls


def test_backward_runs_only_for_the_trained_layers(pkg, cuda):
    """With the CG layer and the head trained, the weight-gradient GEMMs run for exactly the trained weight scopes and no
    BatchNorm backward, weight gradient or grouping backward of layers 1-3 or the vote layer runs; with nothing frozen
    every conv runs one weight gradient and every BatchNorm one backward, and the ordered list of entry points (with
    their first three integer arguments: rows and widths) is tests/golden/finetune_full_backward_trace.json, recorded
    on the same scene from the code as it was before the frozen set existed."""
    full, fconvs, fcalls = backward_trace(pkg, cuda, None)
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "finetune_full_backward_trace.json")) as f:
        pinned = json.load(f)
    got = [[c] + [x for x in a if isinstance(x, int)][:3] for c, a in fcalls]
    assert got == pinned, "the full-training backward's entry points changed"
    top, tconvs, tcalls = backward_trace(pkg, cuda, TOP)
    names = lambda calls, n: [a for c, a in calls if c == n]
    wshape = lambda tr, s: tuple(tr.tp.tensors[s + "/weights"].shape)
    scope_rows = {(s, r, ci, co) for s, r, ci, co in fconvs}

    assert len(names(fcalls, "ssd3d_linear_wgrad")) == len(full.tp.weight_scopes()) == len(fconvs)
    assert len(names(fcalls, "ssd3d_bn_train_grad")) == len(full.tp.bn_scopes())
    got = sorted((a[0], a[1], a[2]) for a in names(fcalls, "ssd3d_linear_wgrad"))
    assert got == sorted((r, ci, co) for _, r, ci, co in scope_rows)

    trained_scopes = top.tp.weight_scopes()
    assert trained_scopes and not any(s.startswith(BOTTOM) for s in trained_scopes)
    got = sorted((a[0], a[1], a[2]) for a in names(tcalls, "ssd3d_linear_wgrad"))
    want = sorted((r, ci, co) for s, r, ci, co in tconvs if s in trained_scopes)
    assert got == want and len(got) == len(trained_scopes)
    top_bn = sorted((r, co) for s, r, _, co in tconvs if s in top.tp.bn_scopes() and not s.startswith(BOTTOM))
    assert sorted((a[0], a[1]) for a in names(tcalls, "ssd3d_bn_train_grad")) == top_bn     # no BatchNorm of layers 1-3 / vote
    assert len(names(tcalls, "ssd3d_group_concat_grad")) < len(names(fcalls, "ssd3d_group_concat_grad"))
    assert len(names(tcalls, "ssd3d_rowgroup_max_grad")) < len(names(fcalls, "ssd3d_rowgroup_max_grad"))
    assert len(tcalls) < len(fcalls) / 2


@pytest.mark.parametrize("kind", ["adam", "momentum"])
def test_resume_is_bit_for_bit(pkg, cuda, tmp_path, kind):
    """The trained-on-top set (its step has no atomic scatter): three uninterrupted steps against two steps, save, load
    into a fresh Trainer, and the third step there; every tensor and the optimizer's state agree bit for bit."""
    solver = S.Solver(steps=(1,), type=kind)
    a = trainer(pkg, cuda, TOP, solver)
    b = trainer(pkg, cuda, TOP, solver)
    for step in range(2):
        b.step(*real_batch(pkg, cuda, step))
    path = str(tmp_path / "model-00000002.npz")
    b.save(path)
    with np.load(path) as z:
        slots = {k for k in z.files if k.endswith(("/Adam", "/Adam_1", "/Momentum"))}
    assert slots == {k + s for k, _ in b.tp.named_parameters() for s in S.OPTIMIZERS[kind].SLOTS}
    c = trainer(pkg, cuda, TOP, solver, seed=50)
    c.load(path)
    for step in range(3):
        a.step(*real_batch(pkg, cuda, step))
    c.step(*real_batch(pkg, cuda, 2))
    torch.cuda.synchronize()
    assert a.global_step == c.global_step == 3
    for k, t in a.tp.tensors.items():
        same_bits(N(c.tp.tensors[k]), N(t), "%s step 3: %s" % (kind, k))
    sa, sc = a.optimizer.state_dict(), c.optimizer.state_dict()
    for k in sa:
        same_bits(np.asarray(sc[k]), np.asarray(sa[k]), "%s state %s" % (kind, k))
    wrong = trainer(pkg, cuda, TOP, S.Solver(steps=(1,), type="momentum" if kind == "adam" else "adam"))
    with pytest.raises(ValueError, match="another optimizer"):
        wrong.load(path)


@pytest.mark.parametrize("sync_bn", [False, True])
def test_data_parallel_with_a_frozen_set(sync_bn):
    isolated("frozen_ranks(pkg, cuda, 2, %r)" % sync_bn)


def frozen_ranks(pkg, cuda, world, sync_bn, steps=3):
    """`world` simulated ranks (test_data_parallel_gpu.run_simulated; with SyncBN test_sync_bn_gpu.trainer_replicas, each
    rank on its own thread and stream, meeting before every forward exchange) train the 1/8-scale model on shards of one
    batch with trainable=TOP and Momentum.  The exchange covers the trained gradient only; without SyncBN the first
    exchange equals the oracle's on the captured gradients and BN records.  After three steps every rank holds the same
    trained tensors and moving statistics, the frozen tensors keep their initial bits, and the statistics of the frozen
    layers have moved: they are still exchanged."""
    import threading
    from test_backbone_gpu import scaled_arch
    D = pkg.dist
    synth = importlib.import_module("3dssd_b200.synth")
    arch = scaled_arch(pkg, 8)
    d = pkg.params.init_params(arch, 1, seed=5, random_bias=True)
    d.update(pkg.params.init_head_params(pkg.config.layer_channels(arch, 1)[-1], seed=6))
    ctas = sim_ctas(pkg, world)
    barrier = threading.Barrier(world, timeout=300)

    def meet(scope, direction):
        if direction == 0:                                 # the backward runs inside autograd (test_sync_bn_gpu)
            torch.cuda.current_stream().synchronize()
            barrier.wait()

    tps = [pkg.params.TrainableParams(d, cuda, trainable=TOP) for _ in range(world)]
    n = sum(t.numel() for t in tps[0].parameters())
    full = pkg.params.TrainableParams(d, "cpu")
    assert n < sum(t.numel() for t in full.parameters())
    nbytes = D.DataParallel.symmetric_bytes(tps[0], world, ctas, sync_bn=sync_bn)
    assert nbytes < D.DataParallel.symmetric_bytes(full, world, ctas, sync_bn=sync_bn)
    sym = [torch.zeros((nbytes,), dtype=torch.uint8, device=cuda) for _ in range(world)]
    solver = S.Solver(steps=(1,), type="momentum")
    dps = [D.DataParallel(tp, peers=[t.data_ptr() for t in sym], world=world, rank=r, ctas=ctas, clip_norm=solver.clip_norm,
                          sync_bn=sync_bn, before_exchange=meet if sync_bn else None) for r, tp in enumerate(tps)]
    trs = [S.Trainer(arch, tp, solver, dp, sync_bn=sync_bn) for tp, dp in zip(tps, dps)]
    assert all(dp.grad.numel() == tr.optimizer.param.numel() == n for dp, tr in zip(dps, trs))
    init = {k: N(tps[0].tensors[k]).copy() for k in tps[0].frozen_names()}
    stats0 = N(tps[0].stats_flat).copy()
    p, b, l = synth.kitti_like_with_boxes(2 * world, 2048, 20, seed=12)
    pts, boxes, labels = (torch.from_numpy(a).to(cuda) for a in (p, b, l))
    streams = [torch.cuda.Stream(device=cuda) for _ in range(world)]
    shard = lambda r: [D.shard_batch(t, r, world) for t in (pts, boxes, labels)]

    if sync_bn:
        errs = []

        def run(r):
            try:
                sp, sb, sl = shard(r)
                with torch.cuda.stream(streams[r]):
                    xyz, feat = pkg.tf_ops.split_points(sp)
                    for _ in range(steps):
                        trs[r].step(xyz, feat, sb, sl)
                streams[r].synchronize()
            except BaseException as e:                    # noqa: B902  (re-raised below)
                errs.append(e)
                barrier.abort()

        th = [threading.Thread(target=run, args=(r,)) for r in range(world)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        if errs:
            raise errs[0]
    else:
        for step in range(steps):
            losses = []
            for r, tr in enumerate(trs):
                sp, sb, sl = shard(r)
                xyz, feat = pkg.tf_ops.split_points(sp)
                tr.dp.zero_grad()
                with tr.dp.recording():
                    o = pkg.backbone.train_forward(arch, tr.tp, xyz, feat, bn_decay=float(solver.bn_decay(step)))
                tg = pkg.loss.assign_targets(o.base_xyz, o.vote_base, sb, sl)
                lo = pkg.loss.detection_loss(o.base_xyz, *o.head, o.vote_offsets[-1], tg)
                lo["total"].backward()
                losses.append(lo)
            torch.cuda.synchronize()
            if step == 0:
                grads = [N(dp.grad).copy() for dp in dps]
                records = [N(dp.record).copy() for dp in dps]
            for r in reversed(range(world)):                            # launch order != rank order
                with torch.cuda.stream(streams[r]):
                    dps[r].exchange(losses[r])
            torch.cuda.synchronize()
            if step == 0:
                want_g, want_s, _, _ = ODP.exchange(grads, records, stats0, float(solver.bn_decay(0)))
                for r in range(world):
                    same_bits(N(dps[r].grad), want_g, "mean gradient rank %d" % r)
                    same_bits(N(tps[r].stats_flat), want_s, "moving statistics rank %d" % r)
            for r in range(world):
                with torch.cuda.stream(streams[r]):
                    trs[r].optimizer.step()
                trs[r].global_step += 1
            torch.cuda.synchronize()
    torch.cuda.synchronize()
    assert sum(dp.timeouts() for dp in dps) == 0
    for r in range(world):
        for k, v in init.items():
            same_bits(N(tps[r].tensors[k]), v, "frozen %s rank %d" % (k, r))
        same_bits(N(tps[r].stats_flat), N(tps[0].stats_flat), "statistics rank %d" % r)
        for (k, a), (_, b2) in zip(tps[0].named_parameters(), tps[r].named_parameters()):
            same_bits(N(b2), N(a), "trained %s rank %d after %d steps" % (k, r, steps))
    off = tps[0].bn_offsets
    for s in tps[0].bn_scopes():
        if s.startswith(BOTTOM):
            o, c = off[s]
            assert not np.array_equal(N(tps[0].stats_flat)[o:o + 2 * c], stats0[o:o + 2 * c]), "statistics of %s did not move" % s
    assert all(not np.array_equal(N(tps[0].tensors[k]), d[k]) for k, _ in tps[0].named_parameters() if k.endswith("/weights"))
