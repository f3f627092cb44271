"""The FPS launch plan (3dssd_b200/csrc/fps_plan.h), pinned without a GPU.

Every index an FPS route returns is bit-exact, so a routing change keeps the GPU tests green while the speed moves.
This test records which kernel, cluster size, points per thread and shared memory every swept shape gets, what the
query entry points answer, and the return code and message of every call the library rejects before any CUDA call.
The table must equal tests/golden/fps_routes.json; SSD3D_RECORD_FPS_ROUTES=<file> re-records it (the library it reads
is the one SSD3D_LIB names, if set).  The file lists every distinct outcome once, numbered, then one line per swept
shape with the outcome of each cluster request (fps, dist) or, per cluster request, of each channel count (features).
Queries are swept in the order they joined the table, so a new one never renumbers the recorded outcomes."""
import json
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "fps_routes.json")

NS = (1, 64, 300, 512, 1000, 1024, 1025, 2048, 2049, 4095, 4096, 8192, 8193, 12001, 16384, 16385, 20000, 65536, 65537)
CLUSTERS = (0, 1, 2, 4, 8, 16, -1, -2, -4, -8, -16)
ALIGNED, UNALIGNED = 16, 20                                  # never dereferenced: every call below returns before CUDA
OUT = 16
FEATURE_NS = tuple(sorted(NS + (3000, 4097)))
FEATURE_CS = (2, 3, 67, 68, 69, 131, 132, 133)
FEATURE_CLUSTERS = (0, -1, -2, -4, -8, -16)             # the requests ssd3d_farthest_point_sample_features_cl accepts


def _queries():
    q = []
    for n in NS:
        for m in (255, 256):
            for cluster in CLUSTERS:
                for flags in (0, 1, 2, 4):
                    for aligned in (1, 0):
                        q.append(("fps", n, 3, m, cluster, flags, aligned))
        for c in (5, 67, 131, 200):
            for cluster in CLUSTERS:
                q.append(("fps", n, c, 256, cluster, 0, 1))
        for cluster in CLUSTERS:
            q.append(("dist", n, cluster))
        for c in (67, 68, 69, 131, 132, 133):
            q.append(("features", n, c, 0))
    seen = set(q)
    q += [f for n in FEATURE_NS for cl in FEATURE_CLUSTERS for c in FEATURE_CS if (f := ("features", n, c, cl)) not in seen]
    return q


def _plans(tmp_path, queries):
    exe = str(tmp_path / "fps_routes")
    subprocess.check_call(["c++", "-std=c++17", "-O1", "-Wall", "-Werror", "-o", exe, os.path.join(HERE, "fps_routes.cpp")])
    out = subprocess.run([exe], input="".join(" ".join(map(str, q)) + "\n" for q in queries), capture_output=True,
                         text=True, check=True).stdout.split("\n")
    assert len(out) == len(queries) + 1
    return [[int(v) if v.lstrip("-").isdigit() else v for v in line.split()] for line in out[:-1]]


def _abi(L, q, plan, messages):
    """(return code, message number) of the calls the library answers before any CUDA call: a partial range without
    temp, and a full range without temp where the plan has no on-chip kernel."""
    kind = plan[0]

    def call(fn, *a):
        rc = fn(*a)
        msg = L.ssd3d_last_error().decode() if rc != 0 else ""
        return [rc, messages.setdefault(msg, len(messages))]

    if q[0] == "fps":
        _, n, c, m, cluster, flags, aligned = q
        inp = ALIGNED if aligned else UNALIGNED
        part = call(L.ssd3d_farthest_point_sample_ex, 1, n, c, m, inp, n * c, None, OUT, m, 0, 0, 1, cluster, flags, None)
        full = call(L.ssd3d_farthest_point_sample_ex, 1, n, c, m, inp, n * c, None, OUT, m, 0, 0, m, cluster, flags, None) \
            if kind == "fallback" else None
        return [part, full]
    if q[0] == "dist":
        _, n, cluster = q
        return [None, call(L.ssd3d_farthest_point_sample_with_distance_ex, 1, n, 256, ALIGNED, None, OUT, 256, 0, cluster, None)
                if kind == "fallback" else None]
    _, n, c, cluster = q
    ca = min(c, 3)
    args = (1, n, ca, c - ca, 256, ALIGNED, n * ca, ALIGNED, n * (c - ca), None, OUT, 256, 0)
    part = call(L.ssd3d_farthest_point_sample_features_cl, *args, 0, 1, cluster, None)
    full = call(L.ssd3d_farthest_point_sample_features_cl, *args, 0, 256, cluster, None) if kind == "fallback" else None
    return [part, full]


def test_fps_routes_match_recording(pkg, tmp_path):
    L = pkg.lib()
    queries = _queries()
    plans = _plans(tmp_path, queries)
    messages = {}
    abis = [_abi(L, q, p, messages) for q, p in zip(queries, plans)]
    rows = [list(q) + p + a for q, p, a in zip(queries, plans, abis)]
    text = sorted(messages, key=messages.get)
    by_key = {tuple(r[:7]): r[7:] for r in rows if r[0] == "fps"}
    feat = {q[1:]: p + a for q, p, a in zip(queries, plans, abis) if q[0] == "features"}
    answers = []
    for n in NS:
        for c in (3, 5, 67, 131, 200):
            ans = [n, c, L.ssd3d_fps_needs_temp(n, c), L.ssd3d_fps_supports_rounds(n, c),
                   [L.ssd3d_fps_temp_elems(n, c, m, f) for m in (255, 256) for f in (0, 1, 2, 4)]]
            # the queries are reads of the plan at their documented defaults
            m0 = 256
            plan = by_key[("fps", n, c, m0, 0, 0, 1)]
            assert ans[2] == (plan[0] == "fallback"), ans
            assert ans[3] == (c == 3 and by_key[("fps", n, c, m0, 0, 2, 1)][7] == 1), ans
            if c == 3:
                assert ans[4] == [by_key[("fps", n, 3, m, 0, f, 1)][6] for m in (255, 256) for f in (0, 1, 2, 4)], ans
            else:
                assert ans[4] == [n] * 8, ans
            answers.append(ans)
        for c in (67, 68, 69, 131, 132, 133):
            s = L.ssd3d_ffps_supported(n, c)
            assert s == (feat[(n, c, 0)][0] == "features")
            answers.append([n, c, s])
    for q, p, (part, full) in zip(queries, plans, abis):
        kind, rounds = p[0], p[7]
        if part is not None:
            assert part[0] == -1 and text[part[1]], q                 # no temp: never launched
        if q[0] == "fps":
            assert ("resident-scene" in text[part[1]] or "c == 3" in text[part[1]]) == (not rounds), q
        assert (full is not None) == (kind == "fallback"), q
        if full is not None:
            assert full[0] in (-1, -2) and text[full[1]], q
    _check_features_caps(feat)
    outcomes, routes = _table(rows)
    record = os.environ.get("SSD3D_RECORD_FPS_ROUTES")
    if record:
        parts = (_line(CLUSTERS), ",\n".join(map(_line, text)), ",\n".join(map(_line, outcomes)),
                 ",\n".join("%s: %s" % (_line(k), _line(v)) for k, v in routes.items()),
                 ",\n".join('"%d": %s' % (n, _line([a for a in answers if a[0] == n])) for n in NS))
        with open(record, "w") as fh:
            fh.write('{"clusters": %s,\n"messages": [\n%s\n],\n"outcomes": [\n%s\n],\n"routes": {\n%s\n},\n'
                     '"queries": {\n%s\n}}\n' % parts)
        return
    with open(GOLDEN) as fh:
        exp = json.load(fh)
    assert exp["clusters"] == list(CLUSTERS)
    got_routes = {k: [_decode(outcomes[i], text) for i in ids] for k, ids in routes.items()}
    exp_routes = {k: [_decode(exp["outcomes"][i], exp["messages"]) for i in ids] for k, ids in exp["routes"].items()}
    assert list(got_routes) == list(exp_routes)
    for k in exp_routes:
        assert got_routes[k] == exp_routes[k], "route changed for %s\n got: %s\n exp: %s" % (k, got_routes[k], exp_routes[k])
    assert [a for n in NS for a in exp["queries"][str(n)]] == json.loads(json.dumps(answers))


def _check_features_caps(feat):
    """A cap below the 8 CTAs that 2048 < n <= 4096 points of 3 <= c <= 68 channels need runs a full range on the 4-CTA
    bucket kernel (4 slots per thread) and sends partial ranges where cluster 0 sends them; every other request plans
    as cluster 0 does."""
    smem = 2 * 256 * 68 * 4 + 4096 * 8 + 8 * 4 * 72 * 4 + 2 * 8 * 72 * 4 + 2 * 4 * 288
    picked = 0
    for (n, c, cl), got in feat.items():
        base = feat[(n, c, 0)]
        if cl in (-1, -2, -4) and 2048 < n <= 4096 and 3 <= c <= 68:
            picked += 1
            assert got[:8] == ["features_bucket", 4, 4, 68, smem, 0, base[6], 0], (n, c, cl, got)
            assert got[8:13] == base[:5] and got[13:] == base[8:], (n, c, cl, got, base)
        else:
            assert got == base, (n, c, cl, got, base)
    assert picked == 3 * 4 * 3            # cap -1 / -2 / -4, n in (2049, 3000, 4095, 4096), c in (3, 67, 68)


def _line(v):
    return json.dumps(v, separators=(",", ":"))


def _table(rows):
    """Distinct outcomes (plan + the two ABI answers) in order of first appearance, and per swept shape the outcome
    number of each cluster request / channel count."""
    outcomes, index, routes = [], {}, {}
    for r in rows:
        if r[0] == "fps":
            key, arg, res = "fps n=%d c=%d m=%d flags=%d aligned=%d" % (r[1], r[2], r[3], r[5], r[6]), r[4], r[7:]
        elif r[0] == "dist":
            key, arg, res = "dist n=%d" % r[1], r[2], r[3:]
        else:
            key, arg, res = "features n=%d cluster=%d c=%s" % (r[1], r[3], ",".join(map(str, FEATURE_CS))), r[2], r[4:]
        i = index.setdefault(_line(res), len(outcomes))
        if i == len(outcomes):
            outcomes.append(res)
        routes.setdefault(key, {})[arg] = i
    return outcomes, {k: [ids[a] for a in (FEATURE_CS if k.startswith("features") else CLUSTERS)] for k, ids in routes.items()}


def _decode(outcome, messages):
    """An outcome with its message numbers replaced by the messages."""
    return outcome[:-2] + [None if a is None else [a[0], messages[a[1]]] for a in outcome[-2:]]
