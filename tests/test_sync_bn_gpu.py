"""GPU checks of SyncBN (csrc/bn.cu ssd3d_bn_train_sync / ssd3d_bn_train_grad_sync, dist.BnSync, DataParallel(sync_bn=True);
DESIGN.md section 3.18) on ranks simulated on one device: every rank is a host thread with its own stream and its own
"symmetric" buffer (a plain allocation of this process -- the kernels only see addresses).

The ranks' exchange CTAs spin on each other, so nothing another rank still has to run may wait behind them.  Every
simulated rank therefore drains its own stream and meets the others at a threading.Barrier before each forward exchange
(the handle's before_exchange hook), so spinners only ever wait on other exchange kernels, and the tests assert from the
occupancy API that all G x ceil(C / 128) of them fit.  Backward exchanges of the full step run inside autograd, which
executes every CUDA node of the device on one engine thread, where a barrier would wait forever; their ranks are
enqueued without host synchronisation instead and the spinners (one or two CTAs) leave the rest of the device free.
Each test runs in a fresh process with every module loaded up front (CUDA_MODULE_LOADING=EAGER: a lazily loaded
kernel may synchronise the context).  No test withholds a rank: the time-out path is covered by the CPU model."""
import importlib
import json
import os
import subprocess
import sys
import threading

import numpy as np
import pytest
import torch

from oracle import sync_bn as O

pytestmark = pytest.mark.gpu
TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)
EPS = 1e-3


def isolated(call):
    env = dict(os.environ, CUDA_MODULE_LOADING="EAGER")
    code = ("import sys; sys.path[:0] = [%r, %r]; import importlib, torch; import test_sync_bn_gpu as t; "
            "pkg = importlib.import_module('3dssd_b200'); cuda = torch.device('cuda:0'); t.%s" % (ROOT, TESTS, call))
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, (r.stdout[-3000:] + "\n" + r.stderr[-6000:])


def N(t):
    return t.detach().cpu().numpy()


def same_bits(got, want, what):
    g, w = np.asarray(got, np.float32).reshape(-1).view(np.int32), np.asarray(want, np.float32).reshape(-1).view(np.int32)
    bad = np.flatnonzero(g != w)
    assert bad.size == 0, "%s: %d of %d differ, first at %d: %r vs %r" % (what, bad.size, g.size, bad[0],
                                                                         np.asarray(got).reshape(-1)[bad[0]],
                                                                         np.asarray(want).reshape(-1)[bad[0]])


def within_ulp(got, want, what, ulps=1):
    g, w = np.asarray(got, np.float32).reshape(-1), np.asarray(want, np.float32).reshape(-1)
    d = np.abs(g.view(np.int32).astype(np.int64) - w.view(np.int32).astype(np.int64))
    same_sign = np.sign(g) == np.sign(w)
    ok = (d <= ulps) & same_sign | (g == w)
    assert ok.all(), "%s: %d of %d beyond %d ulp, first %r vs %r" % (what, (~ok).sum(), g.size, ulps, g[~ok][0], w[~ok][0])


def bn_shapes():
    """(rows, c) of every BatchNorm of one ARCH_3DSSD step at 8 x 16384 points, then edge shapes."""
    d = json.load(open(os.path.join(TESTS, "golden", "train_backward_shapes.json")))
    out = []
    for name, s in d["calls"]:
        t = (8 * int(np.prod(s[1:-2])), int(s[-2]))
        if name == "bn_train_grad" and t not in out:
            out.append(t)
    return out + [(1, 1), (5, 3), (7, 40), (33, 1024), (1000, 1024), (300, 100)]


class Ranks:
    """`world` simulated ranks: symmetric buffers, peers and the forward / backward slots of one BN of c channels."""

    def __init__(self, pkg, world, c, cuda):
        T, D = pkg.tf_ops, pkg.dist
        self.world, self.c = world, c
        area = int(T.lib().ssd3d_bn_sync_area_bytes(world, c))
        assert area == D.bn_sync_area_bytes(world, c)
        assert world * -(-c // 128) <= T.bn_sync_resident_ctas()
        self.sym = [torch.zeros((2 * area,), dtype=torch.uint8, device=cuda) for _ in range(world)]
        self.peers = torch.tensor([t.data_ptr() for t in self.sym], dtype=torch.int64, device=cuda)
        self.state = torch.zeros((world, 2, 4), dtype=torch.int32, device=cuda)
        self.barrier = threading.Barrier(world, timeout=300)
        self.streams = [torch.cuda.Stream(device=cuda) for _ in range(world)]
        self.slots = [[T.BnSyncSlot(self.peers, world, r, d * area, self.state[r, d], self._meet) for d in (0, 1)]
                      for r in range(world)]

    def _meet(self):
        torch.cuda.current_stream().synchronize()
        self.barrier.wait()

    def run(self, fn):
        """fn(rank) on every rank at once, each from its own thread and stream; returns the results in rank order."""
        out, err = [None] * self.world, []

        def body(r):
            try:
                with torch.cuda.stream(self.streams[r]):
                    out[r] = fn(r)
                self.streams[r].synchronize()
            except BaseException as e:                    # noqa: B902  (re-raised below)
                err.append(e)
                self.barrier.abort()

        th = [threading.Thread(target=body, args=(r,)) for r in range(self.world)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        if err:
            raise err[0]
        return out

    def timeouts(self):
        return int(self.state[:, :, 2].sum().item())


def _input(rng, rows, c):
    x = rng.standard_normal((rows, c)) * (rng.random(c) * 2 + 0.1) + rng.standard_normal(c)
    if c > 2:
        x[:, 1] += 1e3                                    # mean ~10^3 times the spread
        x[:, 2] = 0.75                                    # constant: var = 0
    return x.astype(np.float32)


def _vecs(rng, c, cuda):
    g = torch.from_numpy((rng.random(c) + 0.5).astype(np.float32)).to(cuda)
    b = torch.from_numpy(rng.standard_normal(c).astype(np.float32)).to(cuda)
    mm = torch.from_numpy(rng.standard_normal(c).astype(np.float32)).to(cuda)
    mv = torch.from_numpy((rng.random(c) + 0.5).astype(np.float32)).to(cuda)
    return g, b, mm, mv


# ---- world 1: the same bits as the plain path ----------------------------------------------------------------------

def test_world_one_equals_plain_path():
    isolated("world_one(pkg, cuda)")


def world_one(pkg, cuda):
    T = pkg.tf_ops
    rng = np.random.default_rng(1)
    for rows, c in bn_shapes():
        rk = Ranks(pkg, 1, c, cuda)
        x = torch.from_numpy(_input(rng, rows, c)).to(cuda)
        g, b, mm, mv = _vecs(rng, c, cuda)
        mm2, mv2 = mm.clone(), mv.clone()
        for relu in (True, False):
            plain = T.bn_train(x, g, b, mm, mv, decay=0.9, relu=relu)
            sync = T.bn_train_sync(x, g, b, rk.slots[0][0], mm2, mv2, decay=0.9, relu=relu)
            for name, p, s in zip(("y", "scale", "shift", "mean", "var"), plain, sync):
                same_bits(N(s), N(p), "forward %s rows=%d c=%d relu=%d" % (name, rows, c, relu))
            same_bits(N(mm2), N(mm), "moving mean rows=%d c=%d" % (rows, c))
            same_bits(N(mv2), N(mv), "moving var rows=%d c=%d" % (rows, c))
            go = torch.randn((rows, c), device=cuda)
            pg = T.bn_train_grad(x, go, *plain[1:], g, relu=relu)
            sg = T.bn_train_grad_sync(x, go, *plain[1:], g, rk.slots[0][1], relu=relu)
            for name, p, s in zip(("grad_x", "grad_gamma", "grad_beta"), pg, sg):
                same_bits(N(s), N(p), "backward %s rows=%d c=%d relu=%d" % (name, rows, c, relu))
        torch.cuda.synchronize()
        assert N(rk.state[0])[:, :3].tolist() == [[2, 0, 0], [2, 0, 0]], (rows, c)


# ---- simulated ranks: forward, backward, moving statistics ---------------------------------------------------------

@pytest.mark.parametrize("world", [2, 3, 4])
def test_simulated_ranks(world):
    isolated("simulated(pkg, cuda, %d)" % world)


def simulated(pkg, cuda, world):
    T = pkg.tf_ops
    rng = np.random.default_rng(world)
    for c, sizes in ((200, [3000] * world), (200, [5000, 17, 2600, 1][:world]), (1024, [700, 3][:world] + [64] * (world - 2))):
        rk = Ranks(pkg, world, c, cuda)
        xs = [_input(rng, n, c) for n in sizes]
        g, b, mm, mv = _vecs(rng, c, cuda)
        mms, mvs = [mm.clone() for _ in range(world)], [mv.clone() for _ in range(world)]
        xd = [torch.from_numpy(x).to(cuda) for x in xs]
        outs = rk.run(lambda r: T.bn_train_sync(xd[r], g, b, rk.slots[r][0], mms[r], mvs[r], decay=0.9))
        what = "G=%d c=%d shards=%s" % (world, c, sizes)
        want = O.forward(xs, N(g), N(b), EPS)
        for r in range(world):
            for name, got, w in zip(("scale", "shift", "mean", "var"), outs[r][1:], want):
                same_bits(N(got), w, "%s %s rank %d vs oracle" % (what, name, r))
            same_bits(N(mms[r]), N(mms[0]), "%s moving mean rank %d" % (what, r))
            same_bits(N(mvs[r]), N(mvs[0]), "%s moving var rank %d" % (what, r))
        # one bn_train over the concatenated rows: the same statistics up to the order of the sums
        cat = torch.cat(xd)
        mm1, mv1 = mm.clone(), mv.clone()
        whole = T.bn_train(cat, g, b, mm1, mv1, decay=0.9)
        for name, i in (("scale", 1), ("mean", 3), ("var", 4)):
            within_ulp(N(outs[0][i]), N(whole[i]), "%s %s vs whole batch" % (what, name))
        within_ulp(N(mms[0]), N(mm1), "%s moving mean vs one whole-batch update" % what)
        within_ulp(N(mvs[0]), N(mv1), "%s moving var vs one whole-batch update" % what)
        y = torch.cat([o[0] for o in outs])
        torch.testing.assert_close(y, whole[0], rtol=1e-5, atol=1e-4)

        # backward against the oracle and float64 autograd of the whole batch
        scale, shift, mean, var = outs[0][1:]
        gos = [torch.randn_like(x) for x in xd]
        grads = rk.run(lambda r: T.bn_train_grad_sync(xd[r], gos[r], scale, shift, mean, var, g, rk.slots[r][1]))
        ow = O.backward(xs, [N(t) for t in gos], N(scale), N(shift), N(mean), N(var), N(g), eps=EPS)
        xa = cat.double().requires_grad_(True)
        ga = g.double().requires_grad_(True)
        ba = b.double().requires_grad_(True)
        mu = xa.mean(0)
        ya = (xa - mu) / torch.sqrt((xa * xa).mean(0) - mu * mu + EPS) * ga + ba
        keep = torch.cat([torch.addcmul(shift, x, scale) > 0 for x in xd])
        torch.where(keep, ya, torch.zeros_like(ya)).backward(torch.cat(gos).double())
        gx_all = xa.grad.split(sizes)
        for r in range(world):
            gx, gg, gb = (N(t) for t in grads[r])
            tol = 1e-5 * max(1.0, np.abs(ow[r][0]).max())
            np.testing.assert_allclose(gx, ow[r][0], rtol=1e-5, atol=tol, err_msg="%s grad_x rank %d vs oracle" % (what, r))
            np.testing.assert_allclose(gx, N(gx_all[r]), rtol=1e-3, atol=1e-3 * np.abs(N(xa.grad)).max(),
                                       err_msg="%s grad_x rank %d vs autograd" % (what, r))
            np.testing.assert_allclose(gg, ow[r][1], rtol=1e-5, atol=1e-3, err_msg="%s grad_gamma rank %d" % (what, r))
            np.testing.assert_allclose(gb, ow[r][2], rtol=1e-5, atol=1e-3, err_msg="%s grad_beta rank %d" % (what, r))
        # grad_gamma / grad_beta are each rank's own share: they add up to the whole batch's, and are not it
        np.testing.assert_allclose(sum(N(gr[2]).astype(np.float64) for gr in grads), N(ba.grad), rtol=1e-4, atol=1e-3)
        np.testing.assert_allclose(sum(N(gr[1]).astype(np.float64) for gr in grads), N(ga.grad), rtol=1e-4, atol=1e-3)
        assert not np.allclose(N(grads[0][2]), N(ba.grad), rtol=1e-3, atol=1e-3)
        torch.cuda.synchronize()
        assert rk.timeouts() == 0
        assert (N(rk.state)[:, :, 0] == 1).all()


# ---- CUDA graphs: each rank's call captured, replayed in lockstep ----------------------------------------------------

def test_graph_replay_in_lockstep():
    isolated("graph_replay(pkg, cuda, 3, 200)")


def graph_replay(pkg, cuda, world, c):
    T = pkg.tf_ops
    rng = np.random.default_rng(5)
    rk = Ranks(pkg, world, c, cuda)
    sizes = [900, 31, 400][:world]
    xd = [torch.from_numpy(_input(rng, n, c)).to(cuda) for n in sizes]
    g, b, _, _ = _vecs(rng, c, cuda)
    quiet = [T.BnSyncSlot(s.peers, s.world, s.rank, s.area, s.state) for s, _ in rk.slots]      # no hook inside a capture
    rk.run(lambda r: T.bn_train_sync(xd[r], g, b, rk.slots[r][0]))                              # warm-up, eager
    graphs, outs = [], []
    for r in range(world):
        gr = torch.cuda.CUDAGraph()
        with torch.cuda.stream(rk.streams[r]):
            with torch.cuda.graph(gr, stream=rk.streams[r]):
                outs.append(T.bn_train_sync(xd[r], g, b, quiet[r]))
        graphs.append(gr)
    torch.cuda.synchronize()
    for rep in range(3):
        xs = [_input(rng, n, c) for n in sizes]
        for r in range(world):
            xd[r].copy_(torch.from_numpy(xs[r]))
        torch.cuda.synchronize()

        def replay(r):
            rk._meet()
            graphs[r].replay()

        rk.run(replay)
        want = O.forward(xs, N(g), N(b), EPS)
        for r in range(world):
            for name, got, w in zip(("scale", "shift", "mean", "var"), outs[r][1:], want):
                same_bits(N(got), w, "replay %d %s rank %d" % (rep, name, r))
        assert (N(rk.state)[:, 0, 0] == 2 + rep).all(), N(rk.state)
    assert rk.timeouts() == 0
    del graphs


# ---- the full step ----------------------------------------------------------------------------------------------------

def _params(pkg, arch):
    d = pkg.params.init_params(arch, 1, seed=5, random_bias=True)
    d.update(pkg.params.init_head_params(pkg.config.layer_channels(arch, 1)[-1], seed=6))
    return d


def _losses(pkg, o, boxes, labels, lo, hi):
    sl = lambda t: t[lo:hi]
    tg = pkg.loss.assign_targets(sl(o.base_xyz), sl(o.vote_base), boxes[lo:hi], labels[lo:hi])
    return pkg.loss.detection_loss(sl(o.base_xyz), *[sl(t) for t in o.head], sl(o.vote_offsets[-1]), tg)


def _data_parallel_grads(pkg, cuda, arch, d, pts, boxes, labels, world, sync_bn):
    """The rank-averaged gradient of `world` simulated ranks on shards of the batch, with clipping inactive."""
    D, T = pkg.dist, pkg.tf_ops
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctas = D.simulated_ctas(world, sms)
    barrier = threading.Barrier(world, timeout=300)

    def meet(scope, direction):
        if direction == 0:                                 # the backward runs inside autograd (module doc)
            torch.cuda.current_stream().synchronize()
            barrier.wait()

    tps = [pkg.params.TrainableParams(d, cuda) for _ in range(world)]
    nbytes = D.DataParallel.symmetric_bytes(tps[0], world, ctas, sync_bn=sync_bn)
    sym = [torch.zeros((nbytes,), dtype=torch.uint8, device=cuda) for _ in range(world)]
    dps = [D.DataParallel(tp, peers=[t.data_ptr() for t in sym], world=world, rank=r, ctas=ctas, clip_norm=2.0 ** 100,
                          sync_bn=sync_bn, before_exchange=meet) for r, tp in enumerate(tps)]
    if sync_bn:
        assert world * max(-(-c // 128) for _, c in D._bn_channels(tps[0])) <= T.bn_sync_resident_ctas()
    streams = [torch.cuda.Stream(device=cuda) for _ in range(world)]
    losses = [None] * world

    def fwd(r):
        with torch.cuda.stream(streams[r]):
            dps[r].zero_grad()
            lo, hi = D.shard_bounds(pts.shape[0], r, world)
            with dps[r].recording():
                xyz, feat = T.split_points(pts[lo:hi])
                o = pkg.backbone.train_forward(arch, tps[r], xyz, feat)
            losses[r] = _losses(pkg, o, boxes[lo:hi], labels[lo:hi], 0, hi - lo)
        streams[r].synchronize()

    th = [threading.Thread(target=fwd, args=(r,)) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert all(lo is not None for lo in losses), "a rank's forward failed"
    torch.autograd.backward([lo["total"] for lo in losses])
    torch.cuda.synchronize()
    for r in reversed(range(world)):
        with torch.cuda.stream(streams[r]):
            dps[r].exchange(losses[r])
    torch.cuda.synchronize()
    assert (N(torch.stack([dp.scale for dp in dps])) == 1).all()                  # clipping inactive
    assert sum(dp.timeouts() for dp in dps) == 0
    for r in range(1, world):
        same_bits(N(dps[r].grad), N(dps[0].grad), "averaged gradient rank %d" % r)
    return tps[0], N(dps[0].grad)


def _whole_batch_grads(pkg, cuda, arch, d, pts, boxes, labels, world):
    """One device, BatchNorm over every row, loss = the mean of the per-shard det_loss totals."""
    D, T = pkg.dist, pkg.tf_ops
    tp = pkg.params.TrainableParams(d, cuda)
    xyz, feat = T.split_points(pts)
    o = pkg.backbone.train_forward(arch, tp, xyz, feat)
    tot = 0
    for r in range(world):
        lo, hi = D.shard_bounds(pts.shape[0], r, world)
        tot = tot + _losses(pkg, o, boxes, labels, lo, hi)["total"]
    (tot / world).backward()
    torch.cuda.synchronize()
    return {k: N(t.grad) for k, t in tp.named_parameters()}


def _worst(tp, flat, want):
    """max over the tensors of max |got - want| / max |want|, and the tensor where it is reached.  The bias of a conv
    that feeds a BatchNorm is left out: the normalisation removes it, so its gradient is zero up to rounding."""
    worst = (0.0, None)
    for k, t in tp.named_parameters():
        if k.endswith("/biases") and k[:-len("/biases")] + "/bn/gamma" in tp.tensors:
            continue
        o = tp.grad_offsets[k]
        got = flat[o:o + t.numel()].reshape(t.shape)
        scale = np.abs(want[k]).max()
        if scale > 0:
            worst = max(worst, (float(np.abs(got - want[k]).max() / scale), k))
    return worst


def coordinate_sampled(arch):
    """`arch` with the F-FPS and fusion sampling of layers 2 and 3 replaced by D-FPS.  F-FPS picks points by feature
    distance, and the two runs compared below normalise with statistics that agree to about 1 ulp, not bit for bit
    (their sums run in different orders): a feature-distance tie broken differently would pick other points and compare
    other steps.  A fusion-sampling entry of n points becomes one D-FPS of 2n, so every layer keeps its point counts.
    (The vote layer's F-FPS entry takes all of its rows, which is no sampling.)"""
    out = [list(spec) for spec in arch]
    for spec in out:
        if spec[12] in ("layer2", "layer3"):
            spec[8] = [2 * n if m == "FS" else n for m, n in zip(spec[7], spec[8])]
            spec[7] = ["D-FPS" if m in ("F-FPS", "FS") else m for m in spec[7]]
    return out


def test_full_step_matches_whole_batch():
    isolated("full_step(pkg, cuda)")


def full_step(pkg, cuda):
    from test_backbone_gpu import scaled_arch
    synth = importlib.import_module("3dssd_b200.synth")
    arch, world = coordinate_sampled(scaled_arch(pkg, 8)), 2
    d = _params(pkg, arch)
    p, b, l = synth.kitti_like_with_boxes(2 * world, 2048, 20, seed=11)
    pts, boxes, labels = (torch.from_numpy(a).to(cuda) for a in (p, b, l))
    want = _whole_batch_grads(pkg, cuda, arch, d, pts, boxes, labels, world)
    tp, got = _data_parallel_grads(pkg, cuda, arch, d, pts, boxes, labels, world, sync_bn=True)
    err = _worst(tp, got, want)
    tp, got = _data_parallel_grads(pkg, cuda, arch, d, pts, boxes, labels, world, sync_bn=False)
    control = _worst(tp, got, want)
    print("sync_bn worst %.3g (%s), per-shard BN worst %.3g (%s)" % (err + control))
    assert err[0] <= 1e-3, err
    assert control[0] > 30 * max(err[0], 1e-4), (control, err)                # per-shard statistics: a different gradient


def test_trainer_replicas_stay_identical():
    isolated("trainer_replicas(pkg, cuda)")


def trainer_replicas(pkg, cuda, steps=3):
    from test_backbone_gpu import scaled_arch
    D, S = pkg.dist, pkg.solver
    synth = importlib.import_module("3dssd_b200.synth")
    arch, world = scaled_arch(pkg, 8), 2
    d = _params(pkg, arch)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctas = D.simulated_ctas(world, sms)
    barrier = threading.Barrier(world, timeout=300)

    def meet(scope, direction):
        if direction == 0:
            torch.cuda.current_stream().synchronize()
            barrier.wait()

    tps = [pkg.params.TrainableParams(d, cuda) for _ in range(world)]
    nbytes = D.DataParallel.symmetric_bytes(tps[0], world, ctas, sync_bn=True)
    sym = [torch.zeros((nbytes,), dtype=torch.uint8, device=cuda) for _ in range(world)]
    solver = S.Solver()
    dps = [D.DataParallel(tp, peers=[t.data_ptr() for t in sym], world=world, rank=r, ctas=ctas, clip_norm=solver.clip_norm,
                          sync_bn=True, before_exchange=meet) for r, tp in enumerate(tps)]
    trs = [S.Trainer(arch, tp, solver, dp, sync_bn=True) for tp, dp in zip(tps, dps)]
    p, b, l = synth.kitti_like_with_boxes(2 * world, 2048, 20, seed=12)
    pts, boxes, labels = (torch.from_numpy(a).to(cuda) for a in (p, b, l))
    stats0 = N(tps[0].stats_flat).copy()
    streams = [torch.cuda.Stream(device=cuda) for _ in range(world)]
    means, errs = [[] for _ in range(world)], []

    def run(r):
        try:
            lo, hi = D.shard_bounds(pts.shape[0], r, world)
            with torch.cuda.stream(streams[r]):
                xyz, feat = pkg.tf_ops.split_points(pts[lo:hi])
                for _ in range(steps):
                    m = trs[r].step(xyz, feat, boxes[lo:hi], labels[lo:hi])
                    means[r].append(float(m["total"]))
            streams[r].synchronize()
        except BaseException as e:                        # noqa: B902  (re-raised below)
            errs.append(e)
            barrier.abort()

    th = [threading.Thread(target=run, args=(r,)) for r in range(world)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    if errs:
        raise errs[0]
    torch.cuda.synchronize()
    for r in range(1, world):
        for (k, a), (_, b2) in zip(tps[0].named_parameters(), tps[r].named_parameters()):
            same_bits(N(b2), N(a), "parameter %s rank %d after %d steps" % (k, r, steps))
        same_bits(N(tps[r].stats_flat), N(tps[0].stats_flat), "statistics rank %d" % r)
        assert means[r] == means[0]
    assert not np.array_equal(N(tps[0].stats_flat), stats0)
    assert (N(dps[0].bn_sync.replays()) == steps).all()
    assert sum(dp.timeouts() for dp in dps) == 0


# ---- two processes -----------------------------------------------------------------------------------------------------

def two_process_rank(outdir):
    """One rank of test_two_process_sync_bn_step, started with torchrun's environment variables."""
    from test_backbone_gpu import scaled_arch
    pkg = importlib.import_module("3dssd_b200")
    D, S = pkg.dist, pkg.solver
    synth = importlib.import_module("3dssd_b200.synth")
    rank, world, local = D.init_from_env(backend="nccl")
    dev = torch.device("cuda", local)
    arch = scaled_arch(pkg, 8)
    tp = pkg.params.TrainableParams(_params(pkg, arch), dev)
    solver = S.Solver()
    dp = D.DataParallel(tp, D.PeerArena(D.DataParallel.symmetric_bytes(tp, world, sync_bn=True), dev), sync_bn=True,
                        clip_norm=solver.clip_norm)
    tr = S.Trainer(arch, tp, solver, dp)
    p, b, l = synth.kitti_like_with_boxes(2 * world, 2048, 20, seed=7)
    pts, boxes, labels = (D.shard_batch(torch.from_numpy(a), rank, world).to(dev) for a in (p, b, l))
    xyz, feat = pkg.tf_ops.split_points(pts)
    m = tr.step(xyz, feat, boxes, labels)
    torch.cuda.synchronize()
    np.savez(os.path.join(outdir, "rank%d.npz" % rank), stats=N(tp.stats_flat),
             losses=np.array([float(m[k]) for k in pkg.loss.LOSS_NAMES + ("total",)], np.float32),
             timeouts=np.array([dp.timeouts()]))
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_process_sync_bn_step(tmp_path):
    """DataParallel(sync_bn=True) in two processes over PeerArena symmetric memory: both ranks report the same losses
    and statistics.  Both processes are waited for (killed on a time-out): none is left behind."""
    import socket
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    code = "import sys; sys.path[:0] = [%r, %r]; import test_sync_bn_gpu as t; t.two_process_rank(%r)" % (ROOT, TESTS, str(tmp_path))
    procs = []
    try:
        for r in range(2):
            env = dict(os.environ, RANK=str(r), LOCAL_RANK=str(r), WORLD_SIZE="2", LOCAL_WORLD_SIZE="2",
                       MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
            procs.append(subprocess.Popen([sys.executable, "-c", code], env=env, cwd=ROOT, stdout=subprocess.PIPE,
                                          stderr=subprocess.STDOUT, text=True))
        logs = [p.communicate(timeout=900)[0] for p in procs]
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
                p.wait()
    for r, (p, log) in enumerate(zip(procs, logs)):
        assert p.returncode == 0, "rank %d:\n%s" % (r, log[-6000:])
    a, b = (np.load(os.path.join(str(tmp_path), "rank%d.npz" % r)) for r in range(2))
    same_bits(b["losses"], a["losses"], "losses")
    same_bits(b["stats"], a["stats"], "moving statistics")
    assert int(a["timeouts"][0]) == 0 and int(b["timeouts"][0]) == 0
