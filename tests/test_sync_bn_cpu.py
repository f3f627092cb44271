"""CPU checks of SyncBN (3dssd_b200/csrc/bn.cu ssd3d_bn_train_sync / ssd3d_bn_train_grad_sync, dist.BnSync,
oracle/sync_bn.py; DESIGN.md section 3.18).

* The exchange protocol, explored under every interleaving: every read must hold exactly the triple its peer sent for
  that scope and replay, and no run may deadlock.  Each scope's exchanges run on a stream of their own, so every
  relative order of the two scopes' exchanges -- different on different ranks included -- is among the interleavings.
  The same explorer must find the violation when the protocol is weakened (flag before data; no wait; one set of slots
  for both scopes), and it shows why ranks that issue the scopes on ONE stream must issue them in the same order.
* The oracle: at one rank it is the single-rank restatement of bn.cu bit for bit; on equal shards it agrees with the
  float64 restatement of the reference's sync_batch_norm; its backward agrees with float64 autograd of one BatchNorm
  over the concatenated shards, with grad_gamma / grad_beta the rank's own.
* bn_sync_area_bytes / bn_sync_layout / DataParallel.symmetric_bytes arithmetic.
* Malformed operands rejected before any launch, and the once-per-scope bookkeeping of TrainableParams.start_bn_sync."""
import numpy as np
import pytest
import torch

from oracle import sync_bn as O
from test_tf_ops_abi_cpu import _FakeLib, abi  # noqa: F401  (abi is a fixture)


# ---- the protocol ---------------------------------------------------------------------------------------------------

W_, F_, WAIT_, R_ = range(4)


def explore(world, replays, scopes=2, flag_first=False, wait=True, shared_slots=False, rank_orders=None):
    """Depth-first search over all interleavings.  Threads: by default one per (rank, scope), running that scope's
    exchanges replay after replay (a scope on a stream of its own: any order between scopes); with rank_orders, one per
    rank, running the scopes of every replay in the rank's order (one stream per rank).  One exchange of scope k, replay s
    (the scope's own counter, parity s % 2) on rank me, at the granularity of one CTA:
        W     store my triple into every peer p's data[slot][par][me]      (tag = (k, s))
        F     publish every peer p's flag[slot][par][me] = s               (flag_first: F before W)
        WAIT  until my flag[slot][par][p] >= s for every p                 (wait=False: no wait)
        R     read my data[slot][par][p] for every p: must be tagged (k, s)
    slot = k (shared_slots: 0 for every scope).  A CTA's own slot is written and read by itself only and is left out.
    Returns None when every read is right and every run finishes, else the first violation or deadlock found."""
    nslot = 1 if shared_slots else scopes
    steps = (F_, W_, WAIT_, R_) if flag_first else (W_, F_, WAIT_, R_)
    if not wait:
        steps = tuple(s for s in steps if s != WAIT_)
    if rank_orders is None:
        threads = [(r, [(k, s) for s in range(1, replays + 1)]) for r in range(world) for k in range(scopes)]
    else:
        threads = [(r, [(k, s) for s in range(1, replays + 1) for k in rank_orders[r]]) for r in range(world)]
    plen = [len(p) * len(steps) for _, p in threads]

    def cell(dst, slot, par, src):
        return ((dst * nslot + slot) * 2 + par) * world + src

    size = world * nslot * 2 * world
    start = (tuple([0] * len(threads)), tuple([0] * size), tuple([0] * size))
    seen, stack = set(), [start]
    while stack:
        st = stack.pop()
        if st in seen:
            continue
        seen.add(st)
        pcs, data, flag = st
        moved = False
        for t, (me, prog) in enumerate(threads):
            pc = pcs[t]
            if pc == plen[t]:
                continue
            k, s = prog[pc // len(steps)]
            op, par, slot = steps[pc % len(steps)], s % 2, 0 if shared_slots else k
            peers = [p for p in range(world) if p != me]
            nd, nf = data, flag
            if op == W_:
                nd = list(data)
                for p in peers:
                    nd[cell(p, slot, par, me)] = k * 1000 + s
                nd = tuple(nd)
            elif op == F_:
                nf = list(flag)
                for p in peers:
                    nf[cell(p, slot, par, me)] = s
                nf = tuple(nf)
            elif op == WAIT_:
                if any(flag[cell(me, slot, par, p)] < s for p in peers):
                    continue                                             # still spinning
            else:
                for p in peers:
                    got = data[cell(me, slot, par, p)]
                    if got != k * 1000 + s:
                        return "rank %d scope %d replay %d read peer %d's triple of scope %d replay %d" % (
                            me, k, s, p, got // 1000, got % 1000)
            npcs = list(pcs)
            npcs[t] = pc + 1
            stack.append((tuple(npcs), nd, nf))
            moved = True
        if not moved and any(pcs[t] < plen[t] for t in range(len(threads))):
            return "deadlock at %s" % (pcs,)
    return None


@pytest.mark.parametrize("world,replays", [(2, 5), (3, 4)])
def test_protocol_is_safe_under_every_interleaving_of_two_scopes(world, replays):
    assert explore(world, replays) is None


@pytest.mark.parametrize("world,replays", [(2, 5), (3, 4)])
def test_same_scope_order_on_one_stream_is_safe(world, replays):
    """One stream per rank, both scopes in the same order on every rank (what autograd's one graph gives)."""
    assert explore(world, replays, rank_orders=[(1, 0)] * world) is None


def test_flag_before_data_is_caught():
    assert explore(2, 2, flag_first=True) is not None


def test_missing_wait_is_caught():
    assert explore(2, 2, wait=False) is not None


def test_slots_shared_between_scopes_are_caught():
    """Two scopes with their own counters but one set of slots: a peer's triple of the other scope passes the wait."""
    v = explore(2, 3, shared_slots=True)
    assert v is not None and "deadlock" not in v


def test_crossed_scope_order_on_one_stream_deadlocks():
    """An exchange holds its rank's stream until every peer's exchange of the same scope arrives: ranks that issue the
    scopes on one stream in different orders wait on each other (DESIGN.md section 3.18)."""
    v = explore(2, 1, rank_orders=[(0, 1), (1, 0)])
    assert v is not None and v.startswith("deadlock")


# ---- the oracle -----------------------------------------------------------------------------------------------------

def _shards(rng, sizes, c, spread=1.0):
    return [(rng.standard_normal((n, c)) * spread + rng.standard_normal(c) * 3).astype(np.float32) for n in sizes]


def _bits(a):
    return np.asarray(a, np.float32).view(np.int32)


@pytest.mark.parametrize("rows,c", [(1, 3), (7, 33), (513, 64), (5000, 130)])
def test_oracle_one_rank_is_the_single_rank_restatement(rows, c):
    rng = np.random.default_rng(rows + c)
    x = _shards(rng, [rows], c)[0]
    gamma, beta = (rng.standard_normal(c).astype(np.float32) for _ in range(2))
    for got, want in zip(O.forward([x], gamma, beta), O.bn_train_single(x, gamma, beta)):
        np.testing.assert_array_equal(_bits(got), _bits(want))


def test_oracle_rank_sum_is_rank_ordered():
    """Rank 0's triple first, then the others in order: a reordering that changes the double sum is visible."""
    t = [(np.array([1.0]), np.array([v]), np.array([0.0])) for v in (1.0, -1.0, 2.0 ** -60)]
    assert O.rank_order_sum(t)[1][0] == 2.0 ** -60 and O.rank_order_sum(t[::-1])[1][0] == 0.0


def test_rsqrt_rn_is_correctly_rounded():
    a = np.array([1e-3, 1.0, 2.0, 3.0, 0.25, 1e-30, 7.1e12], np.float32)
    got = O.rsqrt_rn(a)
    for ai, gi in zip(a, got):
        from fractions import Fraction
        t2 = 1 / Fraction(float(ai))                                         # (1/sqrt(a))^2
        cands = [np.nextafter(gi, np.float32(0)), gi, np.nextafter(gi, np.float32(np.inf))]
        errs = [abs(Fraction(float(v)) ** 2 - t2) for v in cands]
        assert errs[1] == min(errs), ai


@pytest.mark.parametrize("world,rows,c", [(2, 300, 17), (3, 128, 64), (4, 1000, 9)])
def test_oracle_equals_reference_formula_on_equal_shards(world, rows, c):
    rng = np.random.default_rng(world * 7 + c)
    xs = _shards(rng, [rows] * world, c)
    gamma, beta = (rng.standard_normal(c).astype(np.float32) for _ in range(2))
    mm, mv = rng.standard_normal(c).astype(np.float32), rng.random(c).astype(np.float32) + 0.5
    scale, shift, mean, var = O.forward(xs, gamma, beta)
    outs, rmean, rvar, rmm, rmv = O.reference_sync_batch_norm(xs, gamma, beta, mm, mv, 0.9)
    np.testing.assert_allclose(mean, rmean, rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(var, rvar, rtol=1e-5, atol=1e-6)
    for x, o in zip(xs, outs):
        np.testing.assert_allclose(O.apply(x, scale, shift, relu=False), o, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(O.moving_update(mm, mean, 0.9), rmm, rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(O.moving_update(mv, var, 0.9), rmv, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("sizes,relu", [((40, 40), True), ((17, 60, 5), True), ((33, 1, 90, 12), False)])
def test_oracle_backward_equals_autograd_of_the_whole_batch(sizes, relu):
    """grad_x of every rank = float64 autograd of ONE BatchNorm (+ ReLU) over the concatenated shards; grad_gamma and
    grad_beta are each rank's own share of the whole-batch gradient (they sum to it)."""
    rng = np.random.default_rng(sum(sizes))
    c, eps = 11, 1e-3
    xs = _shards(rng, sizes, c)
    gouts = [rng.standard_normal(x.shape).astype(np.float32) for x in xs]
    gamma, beta = rng.standard_normal(c).astype(np.float32), rng.standard_normal(c).astype(np.float32)
    scale, shift, mean, var = O.forward(xs, gamma, beta, eps)
    got = O.backward(xs, gouts, scale, shift, mean, var, gamma, relu=relu, eps=eps)

    x = torch.from_numpy(np.concatenate(xs)).double().requires_grad_(True)
    gm = torch.from_numpy(gamma).double().requires_grad_(True)
    bt = torch.from_numpy(beta).double().requires_grad_(True)
    mu = x.mean(0)
    vr = (x * x).mean(0) - mu * mu
    y = (x - mu) / torch.sqrt(vr + eps) * gm + bt
    mask = torch.from_numpy(np.concatenate([O.apply(x_, scale, shift, relu=False) > 0 for x_ in xs]))
    if relu:
        y = torch.where(mask, y, torch.zeros_like(y))
    y.backward(torch.from_numpy(np.concatenate(gouts)).double())
    want_gx = np.split(x.grad.numpy(), np.cumsum(sizes)[:-1])
    for (gx, gg, gb), w in zip(got, want_gx):
        np.testing.assert_allclose(gx, w, rtol=1e-4, atol=1e-5 * np.abs(x.grad.numpy()).max())
    np.testing.assert_allclose(sum(g[1].astype(np.float64) for g in got), gm.grad.numpy(), rtol=1e-4, atol=1e-4)
    np.testing.assert_allclose(sum(g[2].astype(np.float64) for g in got), bt.grad.numpy(), rtol=1e-4, atol=1e-4)
    assert not np.allclose(got[0][2], bt.grad.numpy())                   # local, not the whole batch's


# ---- layout ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("world,c", [(1, 1), (1, 128), (2, 129), (3, 64), (4, 1024), (7, 33)])
def test_area_bytes(pkg, world, c):
    ctas = -(-c // 128)
    data = -(-(world * 3 * c * 8) // 16) * 16
    flags = -(-(world * ctas * 4) // 16) * 16
    assert pkg.dist.bn_sync_area_bytes(world, c) == 2 * data + 2 * flags
    assert pkg.dist.bn_sync_area_bytes(world, c) % 16 == 0


def test_layout_gives_every_scope_its_own_areas(pkg):
    D = pkg.dist
    ch = [("a", 64), ("b", 130), ("c", 1)]
    L = D.bn_sync_layout(ch, 3, base=4096)
    off = 4096
    for s, c in ch:
        n = D.bn_sync_area_bytes(3, c)
        assert L.areas[s] == (off, off + n)
        off += 2 * n
    assert L.nbytes == off - 4096
    with pytest.raises(ValueError):
        D.bn_sync_layout(ch, 3, base=8)
    with pytest.raises(ValueError):
        D.bn_sync_layout(ch + [("a", 4)], 3)
    with pytest.raises(ValueError):
        D.bn_sync_area_bytes(0, 4)


def _tp(pkg):
    P = pkg.params
    arch = [[[0], [0], [0.4], [16], [[8, 16]], True, [-1], ['D-FPS'], [64], -1, False, 'SA_Layer', 'l1', False, -1, 24]]
    return P.TrainableParams(P.init_params(arch, 1, seed=1), "cpu")


@pytest.mark.parametrize("world", [1, 2, 4])
def test_symmetric_bytes_include_the_sync_areas(pkg, world):
    D = pkg.dist
    tp = _tp(pkg)
    ch = [(s, tp.tensors[s + "/bn/moving_mean"].numel()) for s in tp.bn_scopes()]
    plain = D.DataParallel.symmetric_bytes(tp, world)
    assert D.DataParallel.symmetric_bytes(tp, world, sync_bn=False) == plain
    extra = D.DataParallel.symmetric_bytes(tp, world, sync_bn=True) - plain
    assert extra == -(-D.bn_sync_layout(ch, world).nbytes // 256) * 256 and extra > 0


def test_handle_slots(pkg):
    D = pkg.dist
    tp = _tp(pkg)
    peers = torch.tensor([0, 1 << 20], dtype=torch.int64)
    calls = []
    h = D.BnSync(tp, peers, 2, 1, base=512, before_exchange=lambda s, d: calls.append((s, d)))
    scopes = tp.bn_scopes()
    assert list(h.layout.areas) == scopes and h.state.shape == (len(scopes), 2, 4)
    for i, s in enumerate(scopes):
        f, b = h.slots(s)
        assert (f.area, b.area) == h.layout.areas[s] and f.world == 2 and f.rank == 1
        assert f.state.data_ptr() == h.state[i, 0].data_ptr() and b.state.data_ptr() == h.state[i, 1].data_ptr()
        f.before(); b.before()
    assert calls == [(s, d) for s in scopes for d in (0, 1)]
    with pytest.raises(ValueError):
        h.slots("nope")
    with pytest.raises(ValueError):
        D.BnSync(tp, peers, 2, 2)
    with pytest.raises(ValueError):
        D.BnSync(tp, peers[:1], 2, 0)


# ---- operands and bookkeeping ---------------------------------------------------------------------------------------

def _bad_cases(T):
    f, i32, i64 = torch.float32, torch.int32, torch.int64
    z = lambda *n, dt=f: torch.zeros(n, dtype=dt)
    S = lambda **kw: T.BnSyncSlot(**dict(dict(peers=z(2, dt=i64), world=2, rank=0, area=256, state=z(4, dt=i32)), **kw))
    x, v = z(6, 24), z(24)
    yield "fw_no_handle", lambda: T.bn_train_sync(x, v, v, None)
    yield "fw_tuple_handle", lambda: T.bn_train_sync(x, v, v, (z(2, dt=i64), 2, 0, 256, z(4, dt=i32)))
    yield "fw_world0", lambda: T.bn_train_sync(x, v, v, S(world=0))
    yield "fw_world65", lambda: T.bn_train_sync(x, v, v, S(world=65, peers=z(65, dt=i64)))
    yield "fw_rank", lambda: T.bn_train_sync(x, v, v, S(rank=2))
    yield "fw_rank_neg", lambda: T.bn_train_sync(x, v, v, S(rank=-1))
    yield "fw_area", lambda: T.bn_train_sync(x, v, v, S(area=8))
    yield "fw_peers_short", lambda: T.bn_train_sync(x, v, v, S(peers=z(1, dt=i64)))
    yield "fw_peers_dtype", lambda: T.bn_train_sync(x, v, v, S(peers=z(2, dt=i32)))
    yield "fw_state_small", lambda: T.bn_train_sync(x, v, v, S(state=z(2, dt=i32)))
    yield "fw_state_dtype", lambda: T.bn_train_sync(x, v, v, S(state=z(4, dt=i64)))
    yield "fw_gamma_shape", lambda: T.bn_train_sync(x, z(23), v, S())
    yield "fw_x_dtype", lambda: T.bn_train_sync(z(6, 24, dt=torch.float64), v, v, S())
    yield "fw_moving_pair", lambda: T.bn_train_sync(x, v, v, S(), moving_mean=z(24))
    g = z(6, 24)
    yield "bw_no_handle", lambda: T.bn_train_grad_sync(x, g, v, v, v, v, v, None)
    yield "bw_shape", lambda: T.bn_train_grad_sync(x, z(6, 23), v, v, v, v, v, S())
    yield "bw_vec", lambda: T.bn_train_grad_sync(x, g, v, v, z(23), v, v, S())
    yield "bw_rank", lambda: T.bn_train_grad_sync(x, g, v, v, v, v, v, S(rank=5))
    yield "bw_state", lambda: T.bn_train_grad_sync(x, g, v, v, v, v, v, S(state=z(1, dt=i32)))
    w, b = z(24, 24), z(24)
    yield "conv_sync_without_bn", lambda: T.conv_train(x, w, b, v, v, bn=False, sync=(S(), S()))
    yield "conv_sync_one_slot", lambda: T.conv_train(x, w, b, v, v, sync=(S(),))


def test_malformed_sync_operands_raise_before_any_launch(abi):  # noqa: F811
    T, fake = abi
    failures = []
    for name, op in _bad_cases(T):
        fake.calls.clear()
        try:
            op()
        except ValueError:
            if fake.calls:
                failures.append("%s: raised after calling %s" % (name, [c[0] for c in fake.calls]))
            continue
        failures.append("%s: accepted" % name)
    assert not failures, "\n".join(failures)


def test_wellformed_sync_calls_reach_the_library(abi):  # noqa: F811
    """The operands as packed for the C ABI, the hook run before the launch, and the plain calls unchanged."""
    T, fake = abi
    order = []
    peers, state = torch.zeros(3, dtype=torch.int64), torch.zeros(4, dtype=torch.int32)
    s = T.BnSyncSlot(peers, 3, 2, 4096, state, lambda: order.append(len(fake.calls)))
    x, v = torch.zeros((6, 24)), torch.zeros(24)
    T.bn_train_sync(x, v, v, s, moving_mean=torch.zeros(24), moving_var=torch.zeros(24), decay=0.5)
    T.bn_train_grad_sync(x, torch.zeros((6, 24)), v, v, v, v, v, s, relu=False)
    T.bn_train(x, v, v)
    T.bn_train_grad(x, torch.zeros((6, 24)), v, v, v, v, v)
    names = [c[0] for c in fake.calls]
    assert names == ["ssd3d_bn_train_workspace", "ssd3d_bn_train_sync", "ssd3d_bn_train_grad_workspace", "ssd3d_bn_train_grad_sync",
                     "ssd3d_bn_train_workspace", "ssd3d_bn_train", "ssd3d_bn_train_grad_workspace", "ssd3d_bn_train_grad"]
    assert order == [1, 3]                                               # after the workspace query, before the launch
    fw, bw, pf, pb = fake.calls[1][1], fake.calls[3][1], fake.calls[5][1], fake.calls[7][1]
    assert len(fw) == 24 and len(bw) == 24 and len(pf) == 19 and len(pb) == 19
    assert fw[0] == 6 and fw[1] == 24 and fw[8] == pytest.approx(0.5) and fw[19:22] == (3, 2, 4096)
    assert fw[18].value == peers.data_ptr() and fw[22].value == state.data_ptr()
    assert bw[12] == 0 and bw[19:22] == (3, 2, 4096)


def test_bn_sync_bookkeeping(pkg):
    tp = _tp(pkg)
    tp.flat_stats()
    scopes = list(tp.bn_offsets)
    h = pkg.dist.BnSync(tp, torch.zeros(1, dtype=torch.int64), 1, 0)
    with pytest.raises(ValueError):
        tp.start_bn_sync(None)                                           # no handle
    with pytest.raises(ValueError):
        tp.finish_bn_sync()                                              # none open
    tp.start_bn_sync(h)
    with pytest.raises(ValueError):
        tp.start_bn_sync(h)                                              # one at a time
    with pytest.raises(ValueError):
        tp.start_bn_record(torch.zeros(tp.stats_flat.numel()))           # not beside a record
    tp._claim(tp._bn_sync, "BN sync", scopes[0], 0.9)
    with pytest.raises(ValueError):
        tp._claim(tp._bn_sync, "BN sync", scopes[0], 0.9)                # synced twice in one step
    with pytest.raises(ValueError):
        tp._claim(tp._bn_sync, "BN sync", scopes[1], 0.5)                # another decay
    with pytest.raises(ValueError):
        tp.finish_bn_sync()                                              # scopes[1:] never synced
    tp.start_bn_record(torch.zeros(tp.stats_flat.numel()))
    with pytest.raises(ValueError):
        tp.start_bn_sync(h)                                              # not beside a record
    tp.finish_bn_record(check=False)
    tp.start_bn_sync(h)
    for s in scopes:
        tp._claim(tp._bn_sync, "BN sync", s, 0.9)
    assert tp.finish_bn_sync() == 0.9


def test_sync_bn_is_off_by_default(pkg):
    """config.SYNC_BN mirrors the reference's MODEL.NETWORK.SYNC_BN, off in the shipped configuration."""
    assert pkg.config.SYNC_BN is False
