"""Every FPS kernel instantiation the launch plan can pick, run on the GPU against the CPU oracle.

Each `fn<CL,P>` of csrc/fps.cu (and the F-FPS `<CL,P,CP>` variants, the bucket and the fallback kernel) hands its threads
a different mix of residue classes and slots and leaves a different number of threads and CTAs without points, so an
index or tie-break mistake in one instantiation is invisible to the others.  FPS indices are bit-exact: a wrong
tie-break shows up as a different sample set, not as a tolerance.

The cases come from the pinned plan table, tests/golden/fps_routes.json (tests/test_fps_plan_cpu.py): for every distinct
outcome (kind, CL, P, CP) the route key with the smallest n that reaches it and, when it differs, the one with the
largest n.  The call uses exactly the key's n, c, cluster request, flags and input alignment; only m moves, within the
bucket rule.  test_cases_cover_every_outcome (no GPU) checks that the cases cover the table and that every launch below
plans to the outcome its case names.

Scenes (b = 2, b = 1 for matrices over 256 MiB): random points with planted duplicates, an integer lattice (many
distances exactly equal) and all points identical with m > n; m = 1, 2 and n for the smallest-n key; strided input,
a wider output row and an index offset; and, where the route runs partial ranges of rounds, a cut sequence through temp.
"""
import json
import os
import subprocess
import zlib
from collections import namedtuple
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
with open(os.path.join(HERE, "golden", "fps_routes.json")) as _fh:
    TABLE = json.load(_fh)

M_MAIN = 160                 # rounds of the random and lattice scenes (fewer when n is smaller)
BIG = 256 << 20              # a distance matrix larger than this runs one scene instead of two
HOST_DIST_N = 16385          # largest matrix the oracle reads from a host copy; above it the reference is feature-based
# A case may use another n than the table's key when the same outcome is planned there: dist (16,16) is reached in the
# table only at n = 65536 (a 17 GB matrix), and packet / generic (16,16) only at 65536, which costs the oracle 4x the
# time of 32769 at m = n.  The table's n stays as the largest-n case where its matrix fits (dist: n <= DIST_MAX_N).
OVERRIDE_N = {("dist", 16, 16, 0): 32769, ("packet", 16, 16, 0): 32769, ("generic", 16, 16, 0): 32769}
DIST_MAX_N = 32769
SENTINEL = -7
IOFF = 100000

Case = namedtuple("Case", "id outcome family n c key_m cluster flags aligned rounds smallest")
Launch = namedtuple("Launch", "scene m placed cuts")


def _outcome(o):
    return tuple(o[:4])


def _reach(table):
    """(outcome, family, n, c, key m, cluster request, flags, aligned) for every route entry, in table order; for the
    features family the per-entry argument is the channel count."""
    out = []
    for key, ids in table["routes"].items():
        fam, *kv = key.split()
        kv = dict(p.split("=") for p in kv)
        n = int(kv["n"])
        if fam == "features":
            for c, i in zip((int(v) for v in kv["c"].split(",")), ids):
                out.append((_outcome(table["outcomes"][i]), fam, n, c, 0, 0, 0, 1))
        else:
            for cl, i in zip(table["clusters"], ids):
                o = table["outcomes"][i]
                if fam == "fps":
                    out.append((_outcome(o), fam, n, int(kv["c"]), int(kv["m"]), cl, int(kv["flags"]), int(kv["aligned"])))
                else:
                    out.append((_outcome(o), fam, n, 0, 0, cl, 0, 1))
    return out


def _bucket(n, m, flags):
    """fps_plan.h fps3_bucket_applies: the only place m enters the plan."""
    if flags & 2 or n > 16384 or n < 64 or m < 2:
        return False
    return bool(flags & 4) or (n > 8192 and m >= 256)


def _m_free(r):
    """the plan of this route entry does not depend on m"""
    _, fam, n, c, m, _, flags, _ = r
    return fam != "fps" or c != 3 or len({_bucket(n, mm, flags) for mm in (1, 2, 255, 256, m)}) == 1


def _pick(rs, n):
    """the entry at n: m-free entries first (so m = 1, 2, n and m > n keep the plan), then table order"""
    at = [r for r in rs if r[2] == n]
    return sorted(at, key=lambda r: not _m_free(r))[0]


def _fits(r):
    return r[1] != "dist" or r[2] <= DIST_MAX_N


def _picks(table):
    """(outcome, family, n, c, key m, cluster, flags, aligned, smallest) of every case: per outcome the entry with the
    smallest n and, when it differs, the one with the largest n; F-FPS takes every channel count of the key that plans
    to the outcome (c = 68 / 132 fill the packet exactly)"""
    by = {}
    for r in _reach(table):
        by.setdefault(r[0], []).append(r)
    out = []
    for o, rs in by.items():
        lo_n = min(r[2] for r in rs)
        ns = [r[2] for r in rs if _fits(r)]
        lo = _pick(rs, lo_n)
        hi = _pick(rs, max(ns)) if ns and max(ns) != lo_n else None
        if o in OVERRIDE_N:
            if hi is None and _fits(lo):
                hi = lo                   # the table's n stays as the largest-n case
            lo = lo[:2] + (OVERRIDE_N[o],) + lo[3:]
        for r, smallest in ((lo, True), (hi, False)):
            if r is None:
                continue
            for c in sorted({q[3] for q in rs if q[2] == r[2]}) if r[1] == "features" else [r[3]]:
                out.append(r[:3] + (c,) + r[4:] + (smallest,))
    return out


def _cases(table):
    rounds = {_outcome(o): bool(o[7]) for o in table["outcomes"]}
    out = []
    for p in _picks(table):
        o, fam, n, c, m, cl, flags, aligned, smallest = p
        cid = "%s-%d-%d-%d_%s_n%d_c%d_cl%d_f%d_a%d" % (o + (fam, n, c, cl, flags, aligned))
        out.append(Case(cid, o, fam, n, c, m, cl, flags, aligned, rounds[o], smallest))
    return out


CASES = _cases(TABLE)


def _keeps(case, m):
    return case.family != "fps" or case.c != 3 or _bucket(case.n, m, case.flags) == _bucket(case.n, case.key_m, case.flags)


def _launches(case):
    """every launch a case makes, in order"""
    n = case.n
    mm = min(n, M_MAIN) if _keeps(case, min(n, M_MAIN)) else case.key_m
    out = [Launch("dups", mm, False, None), Launch("lattice", mm, False, None)]
    out.append(Launch("same", n + 3 if _keeps(case, n + 3) else mm, False, None))
    if case.smallest:
        out += [Launch("dups", m, False, None) for m in (1, 2, n) if m != mm and _keeps(case, m)]
    if case.family == "dist" and n <= HOST_DIST_N:
        out.append(Launch("asym", mm, False, None))
    mp = max(mm, 8) if _keeps(case, max(mm, 8)) else mm
    out.append(Launch("lattice", mp, True, None))
    if case.rounds:
        out.append(Launch("lattice", mp, True, tuple(sorted({0, 1, 2, 7, (mp // 2) | 1, mp}))))
    return out


def _plan_query(case, launch):
    if case.family == "fps":
        return "fps %d %d %d %d %d %d" % (case.n, case.c, launch.m, case.cluster, case.flags, case.aligned)
    if case.family == "dist":
        return "dist %d %d" % (case.n, case.cluster)
    return "features %d %d" % (case.n, case.c)


def _coverage_gaps(table, cases):
    """what the case list misses of the table: outcomes without a case, and picks (smallest / largest n of an outcome,
    each F-FPS channel count) without their case"""
    have = {(c.outcome, c.family, c.n, c.c, c.key_m, c.cluster, c.flags, c.aligned, c.smallest) for c in cases}
    gaps = sorted(o for o in {_outcome(o) for o in table["outcomes"]} if o not in {c.outcome for c in cases})
    return gaps + [p for p in _picks(table) if p not in have]


def test_cases_cover_every_outcome(tmp_path):
    """No GPU: the cases reach every outcome of the plan table, at its smallest and largest n, and every launch the GPU
    test makes plans (tests/fps_routes.cpp over csrc/fps_plan.h) to the outcome its case names."""
    assert len({_outcome(o) for o in TABLE["outcomes"]}) == len({c.outcome for c in CASES})
    assert _coverage_gaps(TABLE, CASES) == []
    exe = str(tmp_path / "fps_routes")
    subprocess.check_call(["c++", "-std=c++17", "-O1", "-Wall", "-Werror", "-o", exe, os.path.join(HERE, "fps_routes.cpp")])
    queries = [(c, l, _plan_query(c, l)) for c in CASES for l in _launches(c)]
    lines = subprocess.run([exe], input="".join(q + "\n" for _, _, q in queries), capture_output=True, text=True,
                           check=True).stdout.split("\n")[:-1]
    assert len(lines) == len(queries)
    for (case, launch, q), line in zip(queries, lines):
        kind, cl, p, cp, _, _, _, rounds = line.split()
        assert (kind, int(cl), int(p), int(cp)) == case.outcome, (case.id, launch, q, line)
        assert launch.cuts is None or rounds == "1", (case.id, launch, q, line)


def test_coverage_check_sees_gaps():
    """No GPU: dropping any one case, or an outcome the cases do not know, is reported."""
    for i in range(len(CASES)):
        assert _coverage_gaps(TABLE, CASES[:i] + CASES[i + 1:]), CASES[i].id
    fake = json.loads(json.dumps(TABLE))
    fake["outcomes"].append(["packet", 32, 1, 0, 4096, 0, 1, 0, [-1, 0], None])
    assert _coverage_gaps(fake, CASES)


# ---- scenes -------------------------------------------------------------------------------------------------------

def _batch(case):
    return 1 if case.family == "dist" and case.n * case.n * 4 > BIG else 2


def _host(case, scene):
    """the scene as float32 [b, n, c] (dist: the small-integer features its matrix is built from, c = 4).  c = 3:
    float coordinates (random) or integers (lattice); other c: small integers, so every F-FPS and matrix entry is exact,
    with a nonzero last channel."""
    n, b = case.n, _batch(case)
    c = 4 if case.family == "dist" else case.c
    rng = np.random.default_rng(zlib.crc32(("%s/%s" % (case.id, scene)).encode()))
    quant = c != 3
    if scene == "same":
        x = np.full((b, n, c), 1.5 if not quant else 3.0)
    elif scene == "lattice":
        x = rng.integers(0, 6 if not quant else 3, (b, n, c)).astype(np.float64)
        if quant:
            x[..., -1] += 1
    else:
        hi = 200 if case.family == "dist" else 12
        x = rng.uniform(-20, 20, (b, n, c)) if not quant else rng.integers(-hi, hi + 1, (b, n, c)).astype(np.float64)
        if quant:
            x[..., -1] = np.where(x[..., -1] == 0, 1, x[..., -1])
        if n >= 4:
            # copies n/2 + 3 indices away: another residue class mod 1024, for n > 1024 another CTA's points
            src = rng.choice(n, max(1, n // 8), replace=False)
            x[:, (src + n // 2 + 3) % n] = x[:, src]
    return np.ascontiguousarray(x, dtype=np.float32)


def _reference(oracle_ops, case, scene, m):
    """oracle indices [b, m] of a host-side scene (dist: only where no host copy of the matrix is read)"""
    x = _host(case, scene)
    b, n = x.shape[:2]
    if scene == "same":                 # after round 1 every running distance is 0: point 0 holds the smallest key
        return np.zeros((b, m), np.int32)
    if case.family == "features":       # the oracle's two-step route: calc_square_dist + farthest_point_sample_with_distance
        return oracle_ops.farthest_point_sample_with_distance(m, oracle_ops.calc_square_dist(x))
    if case.family == "dist":
        if m <= M_MAIN:
            return oracle_ops.farthest_point_sample_features(m, x)
        # integer features: every calc_square_dist entry is the exact squared distance, which the generic-c D-FPS
        # computes exactly too (test_quantised_routes_agree)
        return oracle_ops.farthest_point_sample(m, x)
    return oracle_ops.farthest_point_sample(m, x)


@pytest.fixture(scope="module")
def refs(oracle_ops):
    """The host references of every case, computed on a thread pool while the GPU runs (the oracle is single-threaded
    per scene): (case id, scene) -> future of the indices for the largest m the case runs on that scene."""
    jobs = {}
    with ThreadPoolExecutor(max(2, os.cpu_count() or 2)) as pool:
        for case in sorted(CASES, key=lambda c: -c.n):
            ms = {}
            for l in _launches(case):
                ms[l.scene] = max(ms.get(l.scene, 0), l.m)
            if case.family == "dist" and case.n <= HOST_DIST_N:
                continue                # read from the host copy of the matrix in the test
            for scene, m in ms.items():
                jobs[(case.id, scene)] = pool.submit(_reference, oracle_ops, case, scene, m)
        yield jobs
        for f in jobs.values():
            f.cancel()


def _fps_kw(case):
    return dict(cluster=case.cluster, packet_kernel=bool(case.flags & 1),
                bucket_kernel=True if case.flags & 4 else (False if case.flags & 2 else None))


def _device_input(torch, case, x, placed, cuda):
    """x on the device with the key's alignment; placed: a [:, a:a+n] slice of a wider tensor whose scene stride keeps
    the dense one's class mod 4 (what the direct kernel's bulk copy checks)"""
    b, n, c = x.shape
    a, t = (4, 4) if case.aligned else (1, 3)
    if placed:
        wide = torch.zeros((b, n + a + t, c), dtype=torch.float32, device=cuda)
        wide[:, a:a + n] = torch.from_numpy(x).to(cuda)
        d = wide[:, a:a + n]
        assert b == 1 or d.stride(0) % 4 == (n * c) % 4
    else:
        flat = torch.zeros(x.size + (0 if case.aligned else 1), dtype=torch.float32, device=cuda)
        d = flat[flat.numel() - x.size:].view(b, n, c)
        d.copy_(torch.from_numpy(x))
    assert (d.data_ptr() % 16 == 0) == bool(case.aligned) or case.family != "fps", case.id
    return d


def _matrix(torch, pkg, case, scene, x, cuda):
    """the scene's [b, n, n] matrix: calc_square_dist of integer features (exact, symmetric, zero diagonal); asym adds a
    non-negative strictly upper triangle, so row `old` and column `old` differ"""
    g = torch.from_numpy(x).to(cuda)
    if scene == "same":
        return torch.zeros((x.shape[0], case.n, case.n), dtype=torch.float32, device=cuda)
    d = pkg.calc_square_dist(g)
    if scene == "asym":
        k = pkg.calc_square_dist(torch.flip(g, [1]))
        d.add_(torch.triu(k, 1))
        del k
    return d


class _Runner:
    def __init__(self, torch, pkg, case, cuda):
        self.torch, self.pkg, self.case, self.cuda = torch, pkg, case, cuda
        self.kw = _fps_kw(case)

    def inputs(self, x, placed):
        case = self.case
        if case.family == "features":
            xyz, pts = (self.torch.from_numpy(np.ascontiguousarray(v)).to(self.cuda) for v in (x[..., :3], x[..., 3:]))
            if placed:                  # [:, a:a+n] slices of two wider tensors: xyz and features with their own strides
                b, n = x.shape[:2]
                w = self.torch.zeros((b, n + 5, 3), dtype=self.torch.float32, device=self.cuda)
                v = self.torch.zeros((b, n + 4, pts.shape[2]), dtype=self.torch.float32, device=self.cuda)
                w[:, 2:2 + n], v[:, 1:1 + n] = xyz, pts
                xyz, pts = w[:, 2:2 + n], v[:, 1:1 + n]
            return xyz, pts
        return _device_input(self.torch, case, x, placed, self.cuda)

    def run(self, inp, m, out=None, ioff=0, rounds=None, temp=None):
        case, pkg = self.case, self.pkg
        if case.family == "fps":
            return pkg.farthest_point_sample(m, inp, out=out, idx_offset=ioff, rounds=rounds, temp=temp, **self.kw)
        if case.family == "features":
            xyz, pts = inp
            return pkg.farthest_point_sample_features(m, xyz, pts, out=out, idx_offset=ioff, rounds=rounds, temp=temp)
        return pkg.farthest_point_sample_with_distance(m, inp, out=out, idx_offset=ioff, cluster=case.cluster)

    def temp(self, b, m):
        case = self.case
        if case.family == "fps":
            e = self.pkg.tf_ops.fps_temp_elems(case.n, 3, m, self.kw["packet_kernel"], self.kw["bucket_kernel"])
        else:
            e = case.n
        return self.torch.empty((b, e), dtype=self.torch.float32, device=self.cuda)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_instantiation_matches_oracle(pkg, oracle_ops, cuda, refs, case):
    import torch
    run = _Runner(torch, pkg, case, cuda)
    host = {}
    for l in _launches(case):
        inp = None                      # frees the previous matrix before the next one is built
        x = host.setdefault(l.scene, _host(case, l.scene if l.scene != "asym" else "dups"))
        b = x.shape[0]
        if case.family == "dist":
            inp = _matrix(torch, pkg, case, l.scene, x, cuda)
            if case.n <= HOST_DIST_N:
                exp = oracle_ops.farthest_point_sample_with_distance(l.m, inp.cpu().numpy())
            else:
                exp = refs[(case.id, l.scene)].result()[:, :l.m]
        else:
            inp = run.inputs(x, l.placed)
            exp = refs[(case.id, l.scene)].result()[:, :l.m]
        what = "%s scene=%s m=%d placed=%s cuts=%s" % (case.id, l.scene, l.m, l.placed, l.cuts)
        if not l.placed:
            got = run.run(inp, l.m).cpu().numpy()
            assert got.shape == exp.shape and np.array_equal(got, exp), \
                "%s: first difference at %s" % (what, np.argwhere(got != exp)[:1].tolist())
            continue
        # placed: a column block of a wider output with an index offset; the rest of the row must stay untouched
        col, m = 3, l.m
        single = run.run(inp, m).cpu().numpy()
        assert np.array_equal(single, exp), what
        buf = torch.full((b, col + m + 5), SENTINEL, dtype=torch.int32, device=cuda)
        if l.cuts is None:
            run.run(inp, m, out=(buf, col), ioff=IOFF)
            h = buf.cpu().numpy()
            assert np.array_equal(h[:, col:col + m] - IOFF, exp), what
            assert (h[:, :col] == SENTINEL).all() and (h[:, col + m:] == SENTINEL).all(), what
            continue
        temp = run.temp(b, m)
        for j0, j1 in zip(l.cuts[:-1], l.cuts[1:]):
            run.run(inp, m, out=(buf, col), ioff=IOFF, rounds=(j0, j1), temp=temp)
            h = buf.cpu().numpy()
            step = "%s rounds [%d,%d)" % (what, j0, j1)
            assert np.array_equal(h[:, col:col + j1] - IOFF, exp[:, :j1]), step
            assert np.array_equal(h[:, col:col + j1] - IOFF, single[:, :j1]), step
            assert (h[:, col + j1:] == SENTINEL).all() and (h[:, :col] == SENTINEL).all(), step
    inp = None
    if case.family == "dist":
        torch.cuda.empty_cache()


def test_quantised_routes_agree(oracle_ops):
    """No GPU: on integer features the references above agree -- the oracle's two-step F-FPS route, its row-by-row
    restatement and the generic-c D-FPS (every distance is an exact integer) -- and on identical points with m > n every
    pick is point 0."""
    rng = np.random.default_rng(7)
    for n, c, hi in ((700, 4, 200), (300, 132, 12), (1100, 68, 3)):
        x = rng.integers(-hi, hi + 1, (2, n, c)).astype(np.float32)
        src = rng.choice(n, n // 8, replace=False)
        x[:, (src + n // 2 + 3) % n] = x[:, src]
        two = oracle_ops.farthest_point_sample_with_distance(n, oracle_ops.calc_square_dist(x))
        assert np.array_equal(two, oracle_ops.farthest_point_sample(n, x))
        assert np.array_equal(two[:, :64], oracle_ops.farthest_point_sample_features(64, x))
    for c in (3, 5, 68):
        same = np.full((2, 37, c), 3.0, np.float32)
        assert not oracle_ops.farthest_point_sample(41, same).any()
        assert not oracle_ops.farthest_point_sample_with_distance(41, oracle_ops.calc_square_dist(same)).any()
