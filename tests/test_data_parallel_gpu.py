"""GPU checks of data-parallel training (csrc/grad_exchange.cu, dist.DataParallel) on ranks simulated on one device:
every rank is a stream with its own "symmetric" buffer (a plain allocation of this process -- the kernels only see
addresses).  Before any exchange the test asserts from the occupancy API that the world's CTAs fit co-resident, so a
wait can never outlast the time-out; no test withholds a rank (the CPU model covers that path).

The ranks spin on each other, so their kernels must truly run at the same time on the one device, which two things
can prevent; neither exists between the processes of a real run.  Loading a kernel lazily may synchronise the context:
each test runs in a fresh process with every module loaded up front (CUDA_MODULE_LOADING=EAGER).  And once the other
ranks' spinning CTAs cover every SM, the kernels a late rank runs before its allreduce are not placed until the
spinners give up: the ranks use dist.simulated_ctas CTAs, so that (G - 1) x ctas stays below the SM count (DataParallel
refuses more)."""
import importlib
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import data_parallel as O
from test_backbone_gpu import scaled_arch

pytestmark = pytest.mark.gpu
synth = importlib.import_module("3dssd_b200.synth")
TESTS = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(TESTS)


def isolated(call):
    """Run `call` (an expression over this module's functions, given pkg and cuda) in a fresh process (module doc)."""
    env = dict(os.environ, CUDA_MODULE_LOADING="EAGER")
    code = ("import sys; sys.path[:0] = [%r, %r]; import importlib, torch; import test_data_parallel_gpu as t; "
            "pkg = importlib.import_module('3dssd_b200'); cuda = torch.device('cuda:0'); t.%s" % (ROOT, TESTS, call))
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, capture_output=True, text=True, timeout=1500)
    assert r.returncode == 0, (r.stdout[-3000:] + "\n" + r.stderr[-6000:])


def N(t):
    return t.detach().cpu().numpy()


def same_bits(got, want, what):
    g, w = np.asarray(got, np.float32).view(np.int32), np.asarray(want, np.float32).view(np.int32)
    bad = np.flatnonzero(g.reshape(-1) != w.reshape(-1))
    assert bad.size == 0, "%s: %d of %d differ, first at %d: %r vs %r" % (what, bad.size, g.size, bad[0],
                                                                         got.reshape(-1)[bad[0]], want.reshape(-1)[bad[0]])


def sim_ctas(pkg, world):
    """CTAs per simulated rank, checked against the occupancy API (all G x ctas co-resident) and the SM count."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ctas = pkg.dist.simulated_ctas(world, sms)
    fit = pkg.tf_ops.peer_allreduce_resident_ctas()
    assert world * ctas <= fit and (world - 1) * ctas < sms, (world, ctas, fit, sms)
    return ctas


# Elements 0 and 1 of the crafted replay, per rank (ranks >= 3 hold 0): every rank's norm is below 5, so every scale
# is 1 and the values reach the sum unchanged.  Column 0 sums exactly in double but not in float32 (1 + 2^-30 rounds
# to 1); column 1 spans more than 53 bits, so its double sum depends on the order (2^-60 + 1 - 1 = 0 in rank order,
# -1 + 1 + 2^-60 = 2^-60 reversed).
CRAFTED = ((1.0, 2.0 ** -60), (2.0 ** -30, 1.0), (-1.0, -1.0))


def crafted_grads(world, n):
    out = []
    for r in range(world):
        g = np.zeros(n, np.float32)
        if r < len(CRAFTED):
            g[: min(n, 2)] = CRAFTED[r][: min(n, 2)]
        out.append(g)
    return out


def float32_sum_mean(gs, scales):
    acc = (gs[0] * scales[0]).astype(np.float32)
    for g, s in zip(gs[1:], scales[1:]):
        acc = (acc + (g * s).astype(np.float32)).astype(np.float32)
    return (acc / np.float32(len(gs))).astype(np.float32)


def reversed_mean(gs, scales):
    return O.allreduce_mean(gs[::-1], scales[::-1])


def rank_grads(rng, world, n, replay):
    """Per-rank gradients: replay 0 is the crafted one (G >= 3), the others random, with some ranks clipping."""
    if replay == 0 and world >= 3:
        return crafted_grads(world, n)
    out = []
    for r in range(world):
        g = (rng.standard_normal(n) * (0.01 if (r + replay) % 2 else 0.5)).astype(np.float32)
        g[: min(n, 4)] = [1.0, 2.0 ** -30, -1.0, 1e8][: min(n, 4)] if r % 2 == 0 else [2.0 ** -30, 1.0, 1e-8, -1e8][: min(n, 4)]
        out.append(g)
    return out


@pytest.mark.parametrize("world", [1, 2, 3, 4])
def test_kernels_bitwise_on_simulated_ranks(world):
    isolated("kernels_bitwise(pkg, cuda, %d)" % world)


def kernels_bitwise(pkg, cuda, world):
    T, D = pkg.tf_ops, pkg.dist
    ctas = sim_ctas(pkg, world)
    streams = [torch.cuda.Stream(device=cuda) for _ in range(world)]
    order = list(range(world))[::-1]                                  # launch order != rank order
    rng = np.random.default_rng(world)
    for n in (1, 37, 2513858):
        L = D.allreduce_layout(n, world, ctas)
        sym = [torch.zeros((L.nbytes,), dtype=torch.uint8, device=cuda) for _ in range(world)]
        peers = torch.tensor([t.data_ptr() for t in sym], dtype=torch.int64, device=cuda)
        grad = [torch.zeros((n,), dtype=torch.float32, device=cuda) for _ in range(world)]
        norm = [torch.zeros((1,), dtype=torch.float32, device=cuda) for _ in range(world)]
        scale = [torch.zeros((1,), dtype=torch.float32, device=cuda) for _ in range(world)]
        ws = [torch.empty((2048,), dtype=torch.uint8, device=cuda) for _ in range(world)]
        state = [torch.zeros((4,), dtype=torch.int32, device=cuda) for _ in range(world)]

        def step(r):
            T.grad_clip_scale(grad[r], norm[r], scale[r], 5.0, ws[r])
            T.peer_allreduce_mean(grad[r], scale[r], peers, world, r, L, state[r])

        def check(gs, what, crafted=False):
            want, _, norms, scales = O.exchange(gs, [np.zeros(1, np.float32)] * world, np.zeros(1, np.float32), 0.9)
            if crafted and world >= 3:                                   # the crafted operands discriminate
                assert (scales == 1).all()
                assert not np.array_equal(want.view(np.int32), float32_sum_mean(gs, scales).view(np.int32))
                if n >= 2:
                    assert not np.array_equal(want.view(np.int32), reversed_mean(gs, scales).view(np.int32))
            for r in range(world):
                same_bits(N(norm[r]), norms[r:r + 1], "%s norm rank %d" % (what, r))
                same_bits(N(scale[r]), scales[r:r + 1], "%s scale rank %d" % (what, r))
                same_bits(N(grad[r]), want, "%s mean rank %d (state %s)" % (what, r, N(state[r]).tolist()))

        def load(replay):
            gs = rank_grads(rng, world, n, replay)
            for r in range(world):
                grad[r].copy_(torch.from_numpy(gs[r]))
            torch.cuda.synchronize()
            return gs

        replays = 0
        for replay in range(6):
            gs = load(replay)
            for r in order:
                with torch.cuda.stream(streams[r]):
                    step(r)
            torch.cuda.synchronize()
            replays += 1
            check(gs, "n=%d replay %d" % (n, replay), crafted=replay == 0)
        graphs = []
        for r in range(world):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.stream(streams[r]):
                with torch.cuda.graph(g, stream=streams[r]):
                    step(r)
            graphs.append(g)
        torch.cuda.synchronize()
        for replay in range(3):
            gs = load(10 + replay)
            for r in order:
                with torch.cuda.stream(streams[r]):
                    graphs[r].replay()
            torch.cuda.synchronize()
            replays += 1
            check(gs, "n=%d graph replay %d" % (n, replay))
        for r in range(world):
            assert N(state[r])[:3].tolist() == [replays, 0, 0]
        del graphs


def test_bn_moving_update_ranks_bitwise(pkg, cuda):
    rng = np.random.default_rng(3)
    for world in (1, 2, 3, 4):
        v = rng.standard_normal(14144).astype(np.float32)
        b = rng.standard_normal((world, 14160)).astype(np.float32)
        st = torch.from_numpy(v).to(cuda)
        pkg.tf_ops.bn_moving_update_ranks(st, torch.from_numpy(b).to(cuda)[:, :14144], world, 0.9)
        same_bits(N(st), O.bn_update(v, b[:, :14144], 0.9), "bn world %d" % world)


# ---- the training step ----------------------------------------------------------------------------------------------

def _params(pkg, arch):
    cfg = pkg.config
    d = pkg.params.init_params(arch, 1, seed=5, random_bias=True)
    d.update(pkg.params.init_head_params(cfg.layer_channels(arch, 1)[-1], seed=6))
    return d


def _forward_backward(pkg, arch, tp, pts, boxes, labels):
    xyz, feat = pkg.tf_ops.split_points(pts)
    o = pkg.backbone.train_forward(arch, tp, xyz, feat)
    tg = pkg.loss.assign_targets(o.base_xyz, o.vote_base, boxes, labels)
    losses = pkg.loss.detection_loss(o.base_xyz, *o.head, o.vote_offsets[-1], tg)
    losses["total"].backward()
    return losses


def run_simulated(pkg, cuda, arch, world, per_rank, npoints, steps=3, seed=2):
    """`world` simulated ranks training on shards of one batch: the first step's exchange against the oracle applied to
    the captured pre-exchange gradients and BN records, then `steps` Adam steps after which the replicas must agree."""
    D = pkg.dist
    ctas = sim_ctas(pkg, world)
    d = _params(pkg, arch)
    tps = [pkg.params.TrainableParams(d, cuda) for _ in range(world)]
    nbytes = D.DataParallel.symmetric_bytes(tps[0], world, ctas)
    sym = [torch.zeros((nbytes,), dtype=torch.uint8, device=cuda) for _ in range(world)]
    dps = [D.DataParallel(tp, peers=[t.data_ptr() for t in sym], world=world, rank=r, ctas=ctas) for r, tp in enumerate(tps)]
    opts = [torch.optim.Adam(tp.parameters(), lr=1e-3) for tp in tps]
    streams = [torch.cuda.Stream(device=cuda) for _ in range(world)]
    p, b, l = synth.kitti_like_with_boxes(world * per_rank, npoints, 20, seed=seed)
    pts, boxes, labels = (torch.from_numpy(a).to(cuda) for a in (p, b, l))
    for step in range(steps):
        losses = []
        for r, (tp, dp) in enumerate(zip(tps, dps)):
            dp.zero_grad()
            with dp.recording():
                sh = [D.shard_batch(t, r, world) for t in (pts, boxes, labels)]
                lo = _forward_backward(pkg, arch, tp, *sh)
            losses.append(lo)
            for k, t in tp.named_parameters():                      # gradients landed in the flat buffer
                o = tp.grad_offsets[k]
                assert t.grad.data_ptr() == tp.grad_flat.data_ptr() + 4 * o, k
        torch.cuda.synchronize()
        if step == 0:
            grads = [N(dp.grad).copy() for dp in dps]
            records = [N(dp.record).copy() for dp in dps]
            stats0 = N(tps[0].stats_flat).copy()
            loss_vals = [[float(lo[k].detach()) for k in pkg.loss.LOSS_NAMES + ("total",)] for lo in losses]
        means = [None] * world
        for r in reversed(range(world)):                                # launch order != rank order
            with torch.cuda.stream(streams[r]):
                means[r] = dps[r].exchange(losses[r])
        torch.cuda.synchronize()
        if step == 0:
            want_g, want_s, norms, _ = O.exchange(grads, records, stats0, 0.9)
            want_l = O.loss_mean(loss_vals)
            for r in range(world):
                same_bits(N(dps[r].grad), want_g, "mean gradient rank %d" % r)
                same_bits(N(tps[r].stats_flat), want_s, "moving statistics rank %d" % r)
                same_bits(N(dps[r].norms()), norms, "norms rank %d" % r)
                same_bits(np.array([float(means[r][k]) for k in pkg.loss.LOSS_NAMES + ("total",)], np.float32), want_l,
                          "losses rank %d" % r)
            assert (norms > 0).all() and np.isfinite(norms).all()
        for opt in opts:
            opt.step()
        torch.cuda.synchronize()
    for r in range(1, world):
        for (k, a), (_, b2) in zip(tps[0].named_parameters(), tps[r].named_parameters()):
            same_bits(N(b2), N(a), "parameter %s rank %d after %d steps" % (k, r, steps))
        same_bits(N(tps[r].stats_flat), N(tps[0].stats_flat), "statistics rank %d" % r)
    assert sum(dp.timeouts() for dp in dps) == 0


def test_shipped_configuration_two_ranks():
    """GPU_NUM 2 x BATCH_SIZE 4 (configs/kitti/3dssd/3dssd.yaml:21-22) at 16384 points with ARCH_3DSSD and the
    detection loss."""
    isolated("run_simulated(pkg, cuda, pkg.config.ARCH_3DSSD, 2, 4, 16384)")


@pytest.mark.parametrize("world", [3, 4])
def test_eighth_scale_more_ranks(world):
    isolated("run_simulated(pkg, cuda, t.scaled_arch(pkg, 8), %d, 2, 2048, seed=%d)" % (world, world))


def test_one_rank_statistics_equal_in_place_path():
    isolated("one_rank_statistics(pkg, cuda)")


def one_rank_statistics(pkg, cuda):
    """world = 1: the recorded statistics applied by the exchange are the in-place update of bn.cu, bit for bit."""
    arch = scaled_arch(pkg, 8)
    d = _params(pkg, arch)
    p, b, l = synth.kitti_like_with_boxes(2, 2048, 20, seed=9)
    pts, boxes, labels = (torch.from_numpy(a).to(cuda) for a in (p, b, l))
    plain = pkg.params.TrainableParams(d, cuda)
    _forward_backward(pkg, arch, plain, pts, boxes, labels)
    tp = pkg.params.TrainableParams(d, cuda)
    nbytes = pkg.dist.DataParallel.symmetric_bytes(tp, 1)
    sym = torch.zeros((nbytes,), dtype=torch.uint8, device=cuda)
    dp = pkg.dist.DataParallel(tp, peers=[sym.data_ptr()], world=1, rank=0)
    dp.zero_grad()
    with dp.recording():
        losses = _forward_backward(pkg, arch, tp, pts, boxes, labels)
    before = N(tp.stats_flat).copy()
    dp.exchange(losses)
    torch.cuda.synchronize()
    assert not np.array_equal(N(tp.stats_flat), before)
    for s in tp.bn_offsets:
        for k in ("/bn/moving_mean", "/bn/moving_variance"):
            same_bits(N(tp.tensors[s + k]), N(plain.tensors[s + k]), s + k)
    assert dp.timeouts() == 0


# ---- two processes: torchrun's path (NCCL process group + PeerArena symmetric memory) --------------------------------

def two_process_rank(outdir):
    """One rank of test_two_process_step, started with torchrun's environment variables."""
    pkg = pkg_mod()
    D = pkg.dist
    rank, world, local = D.init_from_env(backend="nccl")
    dev = torch.device("cuda", local)
    arch = scaled_arch(pkg, 8)
    d = pkg.params.init_params(arch, 1, seed=5 + 10 * rank, random_bias=True)       # rank 1 starts elsewhere: the
    d.update(pkg.params.init_head_params(pkg.config.layer_channels(arch, 1)[-1], seed=6 + 10 * rank))   # broadcast matters
    tp = pkg.params.TrainableParams(d, dev)
    dp = D.DataParallel(tp, D.PeerArena(D.DataParallel.symmetric_bytes(tp, world), dev))
    p, b, l = synth.kitti_like_with_boxes(2 * world, 2048, 20, seed=7)
    pts, boxes, labels = (D.shard_batch(torch.from_numpy(a), rank, world).to(dev) for a in (p, b, l))
    out = {"params": np.concatenate([N(t).reshape(-1) for t in tp.parameters()]), "stats0": N(tp.stats_flat).copy()}
    dp.zero_grad()
    with dp.recording():
        losses = _forward_backward(pkg, arch, tp, pts, boxes, labels)
    torch.cuda.synchronize()
    out.update(grad0=N(dp.grad).copy(), record=N(dp.record).copy(),
               losses=np.array([float(losses[k].detach()) for k in pkg.loss.LOSS_NAMES + ("total",)], np.float32))
    mean = dp.exchange(losses)
    torch.cuda.synchronize()
    out.update(grad=N(dp.grad).copy(), stats=N(tp.stats_flat).copy(), norms=N(dp.norms()).copy(),
               mean=np.array([float(mean[k]) for k in pkg.loss.LOSS_NAMES + ("total",)], np.float32),
               timeouts=np.array([dp.timeouts()]))
    np.savez(os.path.join(outdir, "rank%d.npz" % rank), **out)
    torch.distributed.barrier()
    torch.distributed.destroy_process_group()


def pkg_mod():
    return importlib.import_module("3dssd_b200")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_process_step(tmp_path):
    """DataParallel(tp, PeerArena) in two processes with an NCCL process group, as torchrun starts it: rank 0's weights
    and statistics are broadcast, and the exchange of the real kernels over the symmetric buffers equals the oracle
    applied to both ranks' captured pre-exchange gradients and BN records -- the oracle the simulated ranks are held to.
    Both processes are waited for (killed on a time-out): none is left behind."""
    import socket
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    code = ("import sys; sys.path[:0] = [%r, %r]; import test_data_parallel_gpu as t; t.two_process_rank(%r)"
            % (ROOT, TESTS, str(tmp_path)))
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
    same_bits(b["params"], a["params"], "parameters after the broadcast")
    same_bits(b["stats0"], a["stats0"], "statistics after the broadcast")
    want_g, want_s, norms, _ = O.exchange([a["grad0"], b["grad0"]], [a["record"], b["record"]], a["stats0"], 0.9)
    for r, x in enumerate((a, b)):
        same_bits(x["grad"], want_g, "mean gradient rank %d" % r)
        same_bits(x["stats"], want_s, "moving statistics rank %d" % r)
        same_bits(x["norms"], norms, "norms rank %d" % r)
        same_bits(x["mean"], O.loss_mean([a["losses"], b["losses"]]), "losses rank %d" % r)
        assert int(x["timeouts"][0]) == 0
