"""CPU checks of data-parallel training (3dssd_b200/csrc/grad_exchange.cu, dist.DataParallel, oracle/data_parallel.py).

* The three-phase allreduce protocol, explored under every interleaving at the level of one CTA's sub-slice: each
  copy-out must hold the reduction of exactly that replay's inputs and no run may deadlock.  The same explorer must find
  the violation when the protocol is weakened (flag before data; phase 2 before every F1; copy-out before every F2).
  One parity alone turns out not to be a weakening of this protocol: the explorer proves it safe too.
* The chunk / sub-slice / offset layout of dist.allreduce_layout.
* The oracle against exact (Fraction) arithmetic and the TF 1.4 float32 clip formula, including a zero norm, a norm of
  exactly 5 and NaN / inf propagation.
* Malformed operands rejected before any launch, through the recording stand-in of test_tf_ops_abi_cpu."""
import importlib
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import data_parallel as O
from test_tf_ops_abi_cpu import _FakeLib, abi  # noqa: F401  (abi is a fixture)


# ---- the protocol ---------------------------------------------------------------------------------------------------

def explore(world, replays, parities=2, flag_first=False, wait_f1=True, wait_f2=True):
    """Depth-first search over all interleavings of `world` ranks, one CTA each, running `replays` launches.  A rank's
    program per replay s (parity s % parities), over the peers p != me (a CTA's own slot is written and read by itself
    only, in program order, so it cannot take part in a violation and is left out to keep the search small):
        W1 p: peer p's R1[par][me] = s          F1 p: peer p's F1[par][me] = s        (flag_first: F1 before W1)
        WT1 q: wait my F1[par][q] >= s          RD q: read my R1[par][q]               (wait_f1=False: no WT1)
        W2 p: peer p's R2[par][me] = what I read                F2 p: peer p's F2[par][me] = s
        WT2 q: wait my F2[par][q] >= s          CP q: my R2[par][q] must be the reduction of replay s   (wait_f2=False: no WT2)
    Returns None when every run is correct and terminates, else a description of the first violation."""
    G = world
    progs = []
    for r in range(G):
        peers = [p for p in range(G) if p != r]
        ph1 = [("F1", p) for p in peers] + [("W1", p) for p in peers] if flag_first else \
            [("W1", p) for p in peers] + [("F1", p) for p in peers]
        prog = ph1 + ([("WT1", q) for q in peers] if wait_f1 else []) + [("RD", q) for q in peers] + \
            [("W2", p) for p in peers] + [("F2", p) for p in peers] + ([("WT2", q) for q in peers] if wait_f2 else []) + \
            [("CP", q) for q in peers]
        progs.append(prog)

    def ix(r, par, src):
        return (r * parities + par) * G + src

    size = G * parities * G
    empty_local = tuple(tuple(0 for _ in range(G)) for _ in range(G))
    start = (tuple([1] * G), tuple([0] * G), empty_local, (0,) * size, ((0,) * G,) * size, (0,) * size, (0,) * size)
    seen = set()
    stack = [start]
    while stack:
        st = stack.pop()
        if st in seen:
            continue
        seen.add(st)
        seq, pc, local, r1, r2, f1, f2 = st
        moved = False
        for r in range(G):
            s = seq[r]
            if s > replays:
                continue
            par = s % parities
            op, p = progs[r][pc[r]]
            nr1, nr2, nf1, nf2, nlocal = r1, r2, f1, f2, local
            if op == "W1":
                nr1 = list(r1); nr1[ix(p, par, r)] = s; nr1 = tuple(nr1)
            elif op == "F1":
                nf1 = list(f1); nf1[ix(p, par, r)] = s; nf1 = tuple(nf1)
            elif op == "WT1":
                if f1[ix(r, par, p)] < s:
                    continue
            elif op == "RD":
                row = list(local[r]); row[p] = r1[ix(r, par, p)]; row[r] = s     # own slot: always this replay's
                nlocal = list(local); nlocal[r] = tuple(row); nlocal = tuple(nlocal)
            elif op == "W2":
                nr2 = list(r2); nr2[ix(p, par, r)] = local[r]; nr2 = tuple(nr2)
            elif op == "F2":
                nf2 = list(f2); nf2[ix(p, par, r)] = s; nf2 = tuple(nf2)
            elif op == "WT2":
                if f2[ix(r, par, p)] < s:
                    continue
            else:
                got = r2[ix(r, par, p)]
                if got != (s,) * G:
                    return "rank %d replay %d copied peer %d's reduction of inputs from replays %s" % (r, s, p, got)
            npc, nseq = list(pc), seq
            npc[r] += 1
            if npc[r] == len(progs[r]):                       # launch of replay s done: the next may start (same stream)
                npc[r] = 0
                nseq = list(seq); nseq[r] = s + 1; nseq = tuple(nseq)
            stack.append((nseq, tuple(npc), nlocal, nr1, nr2, nf1, nf2))
            moved = True
        if not moved and not all(s > replays for s in seq):
            return "deadlock at replays %s" % (seq,)
    return None


@pytest.mark.parametrize("world,replays", [(2, 5), (3, 4)])
def test_three_phase_protocol_is_safe_under_every_interleaving(world, replays):
    assert explore(world, replays) is None


def test_single_parity_alone_is_not_a_violation():
    """Unlike the one-phase all-gather, this protocol stays safe with one set of buffers: a rank finishes replay s only
    after every peer's F2 of s, which each peer publishes after its phase-2 reads of R1, and it writes R2 in s+1 only
    after every peer's F1 of s+1.  The kernel keeps two parities anyway, so the reuse argument does not lean on F2
    doubling as an acknowledgement; without the phase-3 wait, one parity is caught (next test)."""
    assert explore(2, 4, parities=1) is None
    assert explore(3, 3, parities=1) is None


def test_copy_before_every_f2_is_caught():
    assert explore(2, 2, wait_f2=False) is not None
    assert explore(2, 3, parities=1, wait_f2=False) is not None


def test_flag_before_data_is_caught():
    assert explore(2, 2, flag_first=True) is not None


def test_phase_two_before_every_f1_is_caught():
    """Reducing without waiting for every peer's F1 reads a peer's clipped sub-slice before it arrived."""
    assert explore(2, 2, wait_f1=False) is not None
    assert explore(3, 2, wait_f1=False) is not None


# ---- the layout -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n,world,ctas", [(1, 1, 64), (1, 3, 64), (7, 2, 64), (11, 4, 3), (37, 3, 64), (1000003, 3, 64),
                                          (2513858, 2, 64), (2513858, 4, 64), (4 * 8 - 1, 8, 5)])
def test_allreduce_layout(pkg, n, world, ctas):
    L = pkg.dist.allreduce_layout(n, world, ctas, base=256)
    assert L.chunk % 4 == 0 and L.sub % 4 == 0 and L.sub > 0
    assert L.chunk * world >= n and (L.chunk - 4) * world < n or L.chunk == 4      # the smallest 16-byte chunk covering n
    assert L.sub * ctas >= L.chunk and (L.sub - 4) * ctas < L.chunk
    covered = np.zeros(world * L.chunk, dtype=np.int32)                          # every float in exactly one sub-slice
    for p in range(world):
        for j in range(ctas):
            lo, hi = min(j * L.sub, L.chunk), min((j + 1) * L.sub, L.chunk)
            covered[p * L.chunk + lo: p * L.chunk + hi] += 1
    assert (covered == 1).all()
    data, flags = world * L.chunk * 4, world * ctas * 4
    regions = sorted([(L.r1[0], data), (L.r1[1], data), (L.r2[0], data), (L.r2[1], data),
                      (L.f1[0], flags), (L.f1[1], flags), (L.f2[0], flags), (L.f2[1], flags)])
    assert regions[0][0] == 256
    for (a, la), (b, _) in zip(regions, regions[1:]):
        assert a + la <= b                                                       # disjoint
    assert regions[-1][0] + regions[-1][1] <= 256 + L.nbytes
    assert all(o % 16 == 0 for o in L.r1 + L.r2) and all(o % 4 == 0 for o in L.f1 + L.f2)
    with pytest.raises(ValueError):
        pkg.dist.allreduce_layout(n, world, ctas, base=8)


def test_allreduce_layout_rejects_empty(pkg):
    for args in ((0, 2), (5, 0), (5, 2, 0)):
        with pytest.raises(ValueError):
            pkg.dist.allreduce_layout(*args)


# ---- the oracle -----------------------------------------------------------------------------------------------------

def rn32(x):
    """Round a Fraction to the nearest float32, ties to even (exactly: no detour through a double)."""
    if x == 0:
        return np.float32(0.0)
    c = np.float32(float(x))
    cands = {c, np.nextafter(c, np.float32(np.inf)), np.nextafter(c, np.float32(-np.inf))}
    best = min(cands, key=lambda f: (abs(Fraction(float(f)) - x), int(np.float32(f).view(np.int32)) & 1))
    return np.float32(best)


def tf_scale(norm, clip=5.0):
    """TF 1.4's float32 clip_by_global_norm scale from a finite positive float32 norm, with exact intermediate values."""
    inv = rn32(1 / Fraction(float(norm)))
    cap = rn32(1 / Fraction(clip))
    return rn32(Fraction(clip) * Fraction(float(min(inv, cap))))


@pytest.mark.parametrize("n,seed,spread", [(1, 0, 1.0), (37, 1, 1.0), (70000, 2, 1.0), (200003, 3, 30.0)])
def test_oracle_norm_and_scale_against_exact_arithmetic(n, seed, spread):
    rng = np.random.default_rng(seed)
    g = (rng.standard_normal(n) * np.exp(rng.uniform(-spread, spread, n)) * 1e-3).astype(np.float32)
    exact = sum(Fraction(float(v)) ** 2 for v in g)
    tree = O.sumsq_tree(g)
    assert abs(Fraction(tree) - exact) <= exact * Fraction(n + 16, 2 ** 52)
    norm, scale = O.clip_scale(g)
    assert norm == np.float32(math.sqrt(float(exact)))
    assert scale == tf_scale(norm)
    c = O.allreduce_mean([g], [scale])
    assert np.array_equal(c, g * scale)                    # G = 1: the clipped gradient itself


def test_oracle_clip_edges():
    z = np.zeros(9, dtype=np.float32)
    assert O.clip_scale(z) == (np.float32(0.0), np.float32(1.0))             # 1/0 = inf, minimum -> 1/5, 5 * 0.2f = 1
    n5, s5 = O.clip_scale(np.array([3.0, 4.0], dtype=np.float32))            # norm exactly 5
    assert n5 == np.float32(5.0) and s5 == np.float32(1.0) == tf_scale(n5)
    n10, s10 = O.clip_scale(np.array([6.0, 0.0, 8.0], dtype=np.float32))
    assert n10 == np.float32(10.0) and s10 == tf_scale(n10) == np.float32(0.5)
    small = np.array([0.3, -0.4], dtype=np.float32)                          # norm < 5: scale rn(5 * 0.2f) = 1
    assert O.clip_scale(small)[1] == np.float32(1.0)
    for bad, want_norm in ((np.array([1.0, np.nan], np.float32), "nan"), (np.array([np.inf, 1.0], np.float32), "inf"),
                           (np.array([1e38, 1e38], np.float32), "finite")):
        norm, scale = O.clip_scale(bad)
        if want_norm == "nan":
            assert np.isnan(norm)
        elif want_norm == "inf":
            assert np.isinf(norm)
        else:
            assert np.isfinite(norm) and np.isfinite(scale)  # (1e38)^2 overflows float32, not the double sum
        if want_norm != "finite":
            assert np.isnan(scale)                         # a non-finite norm poisons the scale (no fminf)
            m = O.allreduce_mean([bad, np.ones(2, np.float32)], [scale, np.float32(1.0)])
            assert np.isnan(m).all()                       # ... and through it every element of the mean


def test_oracle_mean_is_rank_ordered_double_sum():
    """Operands on which a float32 sum, or the sum in another order, gives other bits."""
    big, tiny = np.float32(1.0), np.float32(2.0 ** -30)
    gs = [np.array([big, 1e8], np.float32), np.array([tiny, 1.0], np.float32), np.array([-big, -1e8], np.float32)]
    m = O.allreduce_mean(gs, [np.float32(1.0)] * 3)
    exact = [sum(Fraction(float(g[i])) for g in gs) / 3 for i in range(2)]
    assert m[0] == rn32(exact[0]) and m[0] != np.float32((big + tiny - big) / 3)
    assert m[1] == np.float32(float(Fraction(1, 3)))
    f32 = ((gs[0] + gs[1]) + gs[2]) / np.float32(3)
    assert not np.array_equal(m, f32)
    # exponents spanning more than 53 bits: the double sum depends on the order, and rank order is the one pinned
    hs = [np.array([2.0 ** -60], np.float32), np.array([1.0], np.float32), np.array([-1.0], np.float32)]
    ones = [np.float32(1.0)] * 3
    assert O.allreduce_mean(hs, ones)[0] == 0.0
    assert O.allreduce_mean(hs[::-1], ones)[0] == np.float32(2.0 ** -60 / 3)
    # the scale multiplies in float32 before the double sum
    g = np.array([1.0 + 2.0 ** -23], np.float32)
    assert O.allreduce_mean([g], [np.float32(0.1)])[0] == np.float32(g[0] * np.float32(0.1))


def test_oracle_bn_update_matches_single_rank_update():
    rng = np.random.default_rng(4)
    v, b = rng.standard_normal(50).astype(np.float32), rng.standard_normal((3, 50)).astype(np.float32)
    om = np.float32(1.0) - np.float32(0.9)
    one = v - (v - b[0]) * om
    assert np.array_equal(O.bn_update(v, b[:1], 0.9), one)
    two = O.bn_update(v, b, 0.9)
    want = v
    for r in range(3):
        want = want - (want - b[r]) * om
    assert np.array_equal(two, want)
    assert not np.array_equal(two, O.bn_update(v, b[::-1], 0.9))       # rank order is part of the result
    assert np.array_equal(O.loss_mean([[1.0, 2.0], [2.0, 4.0], [4.0, 8.0]]), np.array([7 / 3, 14 / 3], np.float32))


# ---- malformed operands -----------------------------------------------------------------------------------------------

def _bad_cases(T, D):
    f, i8, i32, i64 = torch.float32, torch.uint8, torch.int32, torch.int64
    z = lambda n, dt=f: torch.zeros(n, dtype=dt)
    L = D.allreduce_layout(37, 2, 4)
    g, sc, peers, st = z(37), z(1), z(2, i64), z(3, i32)
    yield "clip_f64", lambda: T.grad_clip_scale(z(37, torch.float64), z(1), z(1))
    yield "clip_empty", lambda: T.grad_clip_scale(z(0), z(1), z(1))
    yield "clip_norm_dtype", lambda: T.grad_clip_scale(g, z(1, torch.float64), z(1))
    yield "clip_scale_empty", lambda: T.grad_clip_scale(g, z(1), z(0))
    yield "clip_workspace_dtype", lambda: T.grad_clip_scale(g, z(1), z(1), workspace=z(4096, i32))
    yield "clip_strided", lambda: T.grad_clip_scale(z(74)[::2], z(1), z(1))
    yield "ar_layout_n", lambda: T.peer_allreduce_mean(z(36), sc, peers, 2, 0, L, st)
    yield "ar_layout_world", lambda: T.peer_allreduce_mean(g, sc, z(3, i64), 3, 0, L, st)
    yield "ar_misaligned", lambda: T.peer_allreduce_mean(z(38)[1:], sc, peers, 2, 0, L, st)
    yield "ar_state_small", lambda: T.peer_allreduce_mean(g, sc, peers, 2, 0, L, z(2, i32))
    yield "ar_peers_dtype", lambda: T.peer_allreduce_mean(g, sc, z(2, i32), 2, 0, L, st)
    yield "ar_peers_short", lambda: T.peer_allreduce_mean(g, sc, z(1, i64), 2, 0, L, st)
    yield "ar_grad_f64", lambda: T.peer_allreduce_mean(z(37, torch.float64), sc, peers, 2, 0, L, st)
    yield "ar_scale_empty", lambda: T.peer_allreduce_mean(g, z(0), peers, 2, 0, L, st)
    yield "bn_rows", lambda: T.bn_moving_update_ranks(z(10), z((3, 10)), 2, 0.9)
    yield "bn_narrow", lambda: T.bn_moving_update_ranks(z(10), z((2, 9)), 2, 0.9)
    yield "bn_column_stride", lambda: T.bn_moving_update_ranks(z(10), z((2, 20))[:, ::2], 2, 0.9)
    yield "bn_decay", lambda: T.bn_moving_update_ranks(z(10), z((2, 10)), 2, 1.5)
    yield "bn_stats_f64", lambda: T.bn_moving_update_ranks(z(10, torch.float64), z((2, 10)), 2, 0.9)
    yield "bn_batch_vector", lambda: T.bn_moving_update_ranks(z(10), z(20), 2, 0.9)
    yield "bn_empty", lambda: T.bn_moving_update_ranks(z(0), z((2, 4)), 2, 0.9)
    yield "bn_train_stats_out", lambda: T.bn_train(z((6, 24)), z(24), z(24), stats_out=(z(23), z(24)))


def test_malformed_exchange_operands_raise_before_any_launch(abi):  # noqa: F811
    T, fake = abi
    D = importlib.import_module("3dssd_b200.dist")
    failures = []
    for name, op in _bad_cases(T, D):
        fake.calls.clear()
        try:
            op()
        except ValueError:
            if fake.calls:
                failures.append("%s: raised after calling %s" % (name, [c[0] for c in fake.calls]))
            continue
        failures.append("%s: accepted" % name)
    assert not failures, "\n".join(failures)


def test_wellformed_exchange_calls_reach_the_library(abi):  # noqa: F811
    """The three entry points with their operands as packed for the C ABI (the stand-in records them)."""
    T, fake = abi
    D = importlib.import_module("3dssd_b200.dist")
    g = torch.zeros(37)
    T.grad_clip_scale(g, torch.zeros(1), torch.zeros(1), clip_norm=5.0)
    L = D.allreduce_layout(37, 2, 4, base=512)
    T.peer_allreduce_mean(g, torch.zeros(1), torch.zeros(2, dtype=torch.int64), 2, 1, L, torch.zeros(4, dtype=torch.int32))
    T.bn_moving_update_ranks(torch.zeros(10), torch.zeros((2, 16))[:, 2:12], 2, 0.9)
    names = [c[0] for c in fake.calls]
    assert names == ["ssd3d_grad_clip_scale_workspace", "ssd3d_grad_clip_scale", "ssd3d_peer_allreduce_mean",
                     "ssd3d_bn_moving_update_ranks"]
    ar = fake.calls[2][1]
    assert ar[1] == 37 and ar[4:9] == (2, 1, 4, L.chunk, L.sub) and ar[9:17] == L.r1 + L.r2 + L.f1 + L.f2
    bn = fake.calls[3][1]
    assert bn[1] == 10 and bn[3] == 16 and bn[4] == 2 and bn[5] == pytest.approx(0.9)


# ---- TrainableParams: the opt-in flat buffers and the BN record -------------------------------------------------------

def _tp(pkg):
    P = pkg.params
    arch = [[[0], [0], [0.4], [16], [[8, 16]], True, [-1], ['D-FPS'], [64], -1, False, 'SA_Layer', 'l1', False, -1, 24]]
    return P.TrainableParams(P.init_params(arch, 1, seed=1), "cpu")


def test_flat_grads_and_stats_are_views(pkg):
    tp = _tp(pkg)
    before = {k: t.detach().clone() for k, t in tp.tensors.items()}
    flat = tp.flat_grads()
    assert flat.numel() == sum(t.numel() for t in tp.parameters())
    for k, t in tp.named_parameters():
        o = tp.grad_offsets[k]
        assert t.grad.data_ptr() == flat.data_ptr() + 4 * o and t.grad.shape == t.shape
    stats = tp.flat_stats()
    assert stats.numel() == sum(2 * c for _, c in tp.bn_offsets.values())
    for s, (off, c) in tp.bn_offsets.items():
        assert tp.tensors[s + "/bn/moving_mean"].data_ptr() == stats.data_ptr() + 4 * off
        assert tp.tensors[s + "/bn/moving_variance"].data_ptr() == stats.data_ptr() + 4 * (off + c)
    for k, t in tp.tensors.items():
        assert torch.equal(t.detach(), before[k]), k


def test_bn_record_bookkeeping(pkg):
    tp = _tp(pkg)
    tp.flat_stats()
    scopes = list(tp.bn_offsets)
    rec = torch.zeros(tp.stats_flat.numel())
    with pytest.raises(ValueError):
        tp.start_bn_record(torch.zeros(tp.stats_flat.numel() - 1))
    tp.start_bn_record(rec)
    with pytest.raises(ValueError):
        tp.start_bn_record(rec)                                      # one record at a time
    off, c = tp.bn_offsets[scopes[0]]
    m, v = tp._record_slot(scopes[0], 0.9)
    assert m.data_ptr() == rec.data_ptr() + 4 * off and v.data_ptr() == rec.data_ptr() + 4 * (off + c)
    with pytest.raises(ValueError):
        tp._record_slot(scopes[0], 0.9)                              # twice in one step
    with pytest.raises(ValueError):
        tp._record_slot(scopes[1], 0.5)                              # another decay
    with pytest.raises(ValueError):
        tp.finish_bn_record()                                        # scopes[1:] never recorded
    tp.start_bn_record(rec)
    for s in scopes:
        tp._record_slot(s, 0.9)
    assert tp.finish_bn_record() == 0.9


def test_simulated_ctas_leave_an_sm_without_spinners(pkg):
    for world in range(1, 9):
        for sms in (16, 132):
            c = pkg.dist.simulated_ctas(world, sms)
            assert 1 <= c <= pkg.dist.ALLREDUCE_CTAS and (world - 1) * c < sms
    assert pkg.dist.simulated_ctas(4, 132) == 43 and pkg.dist.simulated_ctas(3, 132) == 64
