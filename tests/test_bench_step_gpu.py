"""The step bench.py measures, tested at its own shape: 8 KITTI-shaped scenes of 16384 points, the full ARCH_3DSSD
layer table with the detection head, the bench's options (fps_cluster=-4, direct F-FPS, tensor-core MLPs, in-kernel
gather, both first convs hoisted, automatic layer-1 FPS kernel) and several CUDA graphs of one net replayed
concurrently.

Every scene of the batch is checked, not only scene 0:
  * scene-position invariance: each scene of the batch-8 forward is bit-identical to the same net on that scene alone,
    and to the fps_cluster=0 and latency-mode nets;
  * concurrent graphs: graphs captured from one net and replayed interleaved on separate streams each reproduce an
    eager forward of their own scenes;
  * a float64 restatement of every inference layer and of the head (raw parameters: conv, bias, BN with the moving
    statistics, ReLU), teacher-forced on the run's own inputs, sampled indices and neighbour lists;
  * decode (boxes bit-exact, scores within 2 ulp of a float64 sigmoid) and the BEV NMS against the oracle;
  * FPS and ball query against float64 distances;
  * the CPU oracle, layer by layer, on scene 7.
The CPU test pins this file's constants to bench.py's, so a change there cannot leave these tests on another workload.
"""
import ast
import importlib
import math
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
synth = importlib.import_module("3dssd_b200.synth")

# bench.py's workload (pinned by test_bench_constants_pinned)
SCENES = 8
NPOINTS = 16384
PARAM_SEED = 0
HEAD_SEED = 1
SCENE_SEED = 1000
PIPELINE = 24
FFPS_MODE = "direct"
MLP_MODE = "tc"
GATHER_IN_KERNEL = 1
HOIST_FIRST = 2
FPS_BUCKET = "auto"
FPS_CLUSTER = -4

BN_EPS = 1e-3             # tf.contrib.layers.batch_norm's default epsilon (tf_util.py does not override it)
FEATURE_TOL = 1e-4


def rel_err(got, exp, rtol=1e-3, atol_frac=2e-5):
    """max|got-exp| / max|exp| (the global norm the tolerances are quoted in), after ALSO asserting the elementwise
    bound |got - exp| <= rtol*|exp| + atol_frac*max|exp|: a small-magnitude feature may not hide behind a large one."""
    g, e = got.astype(np.float64), exp.astype(np.float64)
    scale = max(1e-12, np.abs(e).max())
    excess = np.abs(g - e) - (rtol * np.abs(e) + atol_frac * scale)
    if excess.size and excess.max() > 0:
        k = np.unravel_index(np.argmax(excess), excess.shape)
        raise AssertionError("elementwise bound exceeded at %s: got %r expected %r (max|exp| %g, %d of %d elements over)"
                             % (k, g[k], e[k], scale, int((excess > 0).sum()), excess.size))
    return float(np.abs(g - e).max() / scale)


def assert_close(got, exp, what):
    """got (float32 tensor) against a float64 tensor at the feature tolerance."""
    e = rel_err(got.double().cpu().numpy(), exp.cpu().numpy(), rtol=FEATURE_TOL)
    assert e < FEATURE_TOL, "%s: rel err %g" % (what, e)


# ---------------------------------------------------------------------------------------------------------------------
# 1. bench.py's constants (CPU)
# ---------------------------------------------------------------------------------------------------------------------
def _bench_tree():
    with open(os.path.join(ROOT, "bench.py")) as f:
        return ast.parse(f.read())


def _calls(tree, name):
    out = []
    for node in ast.walk(tree):
        if isinstance(node, ast.Call):
            f = node.func
            if (isinstance(f, ast.Attribute) and f.attr == name) or (isinstance(f, ast.Name) and f.id == name):
                out.append(node)
    return out


def _kw(call, name):
    for k in call.keywords:
        if k.arg == name:
            return k.value
    raise AssertionError("bench.py: %s(...) has no keyword %r" % (ast.unparse(call.func), name))


def _eval(node, env):
    return eval(compile(ast.Expression(node), "bench.py", "eval"), {"max": max}, env)


def test_bench_constants_pinned():
    """This file's workload constants are bench.py's: read from its syntax tree, without importing it."""
    tree = _bench_tree()
    consts = {}
    for node in tree.body:
        if isinstance(node, ast.Assign):
            for t in node.targets:
                if isinstance(t, ast.Name) and t.id in ("SCENES_PER_GPU", "NPOINTS"):
                    consts[t.id] = ast.literal_eval(node.value)
    assert consts == {"SCENES_PER_GPU": SCENES, "NPOINTS": NPOINTS}

    (ip,) = _calls(tree, "init_params")
    assert ast.literal_eval(_kw(ip, "seed")) == PARAM_SEED and ast.literal_eval(ip.args[1]) == 1
    (ih,) = _calls(tree, "init_head_params")
    assert ast.literal_eval(_kw(ih, "seed")) == HEAD_SEED
    (kl,) = _calls(tree, "kitti_like")
    assert [ast.unparse(a) for a in kl.args] == ["SCENES_PER_GPU", "NPOINTS"]
    assert _eval(_kw(kl, "seed"), {"rank": 0, "SCENES_PER_GPU": SCENES}) == SCENE_SEED      # rank 0: the single-GPU run

    defaults = {}
    for call in _calls(tree, "add_argument"):
        flag = ast.literal_eval(call.args[0])
        defaults[flag] = ast.literal_eval(_kw(call, "default")) if any(k.arg == "default" for k in call.keywords) else None
    assert defaults["--pipeline"] == PIPELINE
    assert defaults["--ffps-mode"] == FFPS_MODE
    assert defaults["--mlp-mode"] == MLP_MODE
    assert defaults["--gather-in-kernel"] == GATHER_IN_KERNEL
    assert defaults["--hoist-first"] == HOIST_FIRST
    assert defaults["--fps-bucket"] == FPS_BUCKET
    assert defaults["--fps-cluster"] is None          # None: the pipelined-steps rule below decides

    class Args:
        no_graph, pipeline, fps_bucket = False, PIPELINE, FPS_BUCKET
    rules = {}
    for node in ast.walk(tree):
        if isinstance(node, ast.Assign) and len(node.targets) == 1:
            t = node.targets[0]
            if isinstance(t, ast.Name) and t.id == "P":
                rules["P"] = node.value
            elif isinstance(t, ast.Attribute) and t.attr == "fps_cluster":
                rules["fps_cluster"] = node.value
    P = _eval(rules["P"], {"args": Args})
    assert P == PIPELINE
    assert ast.unparse(rules["fps_cluster"]) == "-4 if P > 1 else 0"
    assert _eval(rules["fps_cluster"], {"P": P}) == FPS_CLUSTER

    # the measured net and the latency-mode net are built with these options
    nets = {}
    for call in _calls(tree, "SABackbone"):
        kws = {k.arg: k.value for k in call.keywords if k.arg}
        nets["latency" if ast.unparse(kws["fps_cluster"]) == "0" else "throughput"] = kws
    thr, lat = nets["throughput"], nets["latency"]
    assert ast.unparse(thr["fps_cluster"]) == "args.fps_cluster"
    assert _eval(thr["fps_bucket"], {"args": Args}) is None
    assert ast.unparse(lat["latency_mode"]) == "True"
    (mk,) = [n for n in ast.walk(tree) if isinstance(n, ast.Assign) and any(isinstance(t, ast.Name) and t.id == "mk"
                                                                             for t in n.targets)]
    mkw = {k.arg: ast.unparse(k.value) for k in mk.value.keywords}
    assert mkw["in_channels"] == "1" and mkw["head"] == "head"
    assert mkw["gather_in_kernel"] == "bool(args.gather_in_kernel)" and mkw["hoist_first"] == "args.hoist_first"
    assert mkw["ffps_mode"] == "args.ffps_mode" and mkw["mlp_mode"] == "args.mlp_mode"


# ---------------------------------------------------------------------------------------------------------------------
# the bench step: net, eager batch-8 forward, raw head outputs
# ---------------------------------------------------------------------------------------------------------------------
class Bench:
    pass


def make_net(pkg, b, **over):
    kw = dict(in_channels=1, device=b.dev, ffps_mode=FFPS_MODE, mlp_mode=MLP_MODE, head=b.head,
              gather_in_kernel=bool(GATHER_IN_KERNEL), hoist_first=HOIST_FIRST, fps_cluster=FPS_CLUSTER,
              fps_bucket={"auto": None, "on": True, "off": False}[FPS_BUCKET])
    kw.update(over)
    return pkg.SABackbone(b.arch, b.params, **kw)


@pytest.fixture(scope="module")
def bench(pkg, cuda):
    b = Bench()
    b.dev = cuda
    b.arch = pkg.config.ARCH_3DSSD
    b.params = pkg.params.init_params(b.arch, 1, seed=PARAM_SEED)
    b.head_params = pkg.params.init_head_params(pkg.config.layer_channels(b.arch, 1)[-1], seed=HEAD_SEED)
    b.head = pkg.DetectionHead(params=b.head_params, device=cuda)
    b.net = make_net(pkg, b)
    b.pts_np = synth.kitti_like(SCENES, NPOINTS, seed=SCENE_SEED)
    b.pts = torch.from_numpy(b.pts_np).to(cuda)
    return b


def run_step(net, pts):
    """Eager forward with the debug lists, then the head with its raw outputs."""
    out = net.forward(pts, return_debug=True)
    blk, cnt, raw = net.head.forward(out[0], out[1], return_raw=True)
    return out, (blk, cnt, raw)


@pytest.fixture(scope="module")
def step(bench):
    r = run_step(bench.net, bench.pts)
    torch.cuda.synchronize()
    return r


def head_reg(raw):
    """The head's raw regression output (b, n, 30) from the views return_raw hands out."""
    return torch.cat([raw["offset"], raw["angle_cls"], raw["angle_res"]], dim=-1)[:, :, 0]


def flatten(arch, out, head_out):
    """Every output of one step by name."""
    xyz_l, feat_l, fps_l, dbg = out
    blk, cnt, raw = head_out
    t = {}
    for li in range(1, len(arch) + 1):
        if fps_l[li] is not None:
            t["layer%d fps_idx" % li] = fps_l[li]
        if xyz_l[li] is not None:
            t["layer%d xyz" % li] = xyz_l[li]
        t["layer%d features" % li] = feat_l[li]
        for sc, (i, c) in enumerate(zip(dbg[li - 1].get("idx", []), dbg[li - 1].get("cnt", []))):
            t["layer%d scale%d idx" % (li, sc)] = i
            t["layer%d scale%d cnt" % (li, sc)] = c
        if "offsets" in dbg[li - 1]:
            t["layer%d vote offsets" % li] = dbg[li - 1]["offsets"]
    t.update({"head feat": raw["feat"], "head cls": raw["cls"], "head reg": head_reg(raw), "boxes": raw["boxes"],
              "scores": raw["score"], "detection block": blk, "detection count": cnt})
    return t


def assert_equal_outputs(got, exp, rows=None, what=""):
    assert got.keys() == exp.keys()
    for k in exp:
        e = exp[k] if rows is None else exp[k][rows]
        assert got[k].shape == e.shape, "%s%s: shape %s vs %s" % (what, k, tuple(got[k].shape), tuple(e.shape))
        assert torch.equal(got[k], e), "%s%s differs" % (what, k)


# ---------------------------------------------------------------------------------------------------------------------
# 2. scene-position invariance, cluster and latency-mode identity (bit-exact)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_every_scene_equals_its_single_scene_run(bench, step):
    """The planners (tensor-core tiles, fused stacks, unit lists, ball-query workspace, bucket-FPS temp) depend on the
    layer shapes, not on the number of rows of a batch: scene s of the batch-8 step is the same bits as scene s alone."""
    exp = flatten(bench.arch, *step)
    for s in range(SCENES):
        got = flatten(bench.arch, *run_step(bench.net, bench.pts[s:s + 1]))
        assert_equal_outputs(got, exp, rows=slice(s, s + 1), what="scene %d alone: " % s)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["fps_cluster=0", "latency_mode"])
def test_bench_step_equals_cluster0_and_latency_nets(pkg, bench, step, variant):
    """The D-FPS cluster cap and the latency schedule (resumable layer-1 FPS, sampling consumed in parts on side
    streams) are execution details: the batch-8 step is bit-identical with fps_cluster=0 and with bench's
    latency-mode net."""
    over = dict(fps_cluster=0) if variant == "fps_cluster=0" else dict(fps_cluster=0, latency_mode=True)
    got = flatten(bench.arch, *run_step(make_net(pkg, bench, **over), bench.pts))
    assert_equal_outputs(got, flatten(bench.arch, *step), what=variant + ": ")


# ---------------------------------------------------------------------------------------------------------------------
# 3. concurrent CUDA graphs of one net
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_concurrent_graphs_of_one_net(pkg, bench):
    """Three graphs captured from the ONE bench net (shared PreparedParams, fused stacks and side streams; graph-private
    workspaces), each with its own gather buffers and scenes, replayed interleaved on separate streams with no
    synchronisation between replays: each reproduces an eager forward of its own scenes."""
    seeds = (SCENE_SEED, 2000, 3000)
    inputs = [torch.from_numpy(synth.kitti_like(SCENES, NPOINTS, seed=sd)).to(bench.dev) for sd in seeds]
    gathers = [pkg.dist.DetectionGather(SCENES, bench.dev) for _ in seeds]
    runners = [bench.net.capture(p, gather=g) for p, g in zip(inputs, gathers)]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(device=bench.dev) for _ in seeds]
    main = torch.cuda.current_stream()
    for st in streams:
        st.wait_stream(main)
    results = [None] * len(seeds)
    for rnd in range(4):
        for j in range(len(seeds)):
            k = (j + rnd) % len(seeds)                   # rotate which graph is enqueued first
            with torch.cuda.stream(streams[k]):
                results[k] = runners[k]()
    for st in streams:
        main.wait_stream(st)
    torch.cuda.synchronize()
    for k, (p, g) in enumerate(zip(inputs, gathers)):
        (xyz_l, feat_l, fps_l), _ = results[k]
        eager = bench.net.forward(p)
        eblk, ecnt = bench.net.detections(eager[0], eager[1])
        torch.cuda.synchronize()
        for li in range(1, len(bench.arch) + 1):
            if eager[2][li] is not None:
                assert torch.equal(fps_l[li], eager[2][li]), "graph %d: fps_idx of layer %d" % (k, li)
            if eager[0][li] is not None:
                assert torch.equal(xyz_l[li], eager[0][li]), "graph %d: xyz of layer %d" % (k, li)
            assert torch.equal(feat_l[li], eager[1][li]), "graph %d: features of layer %d" % (k, li)
        blk, cnt = g.result()
        assert torch.equal(blk, eblk) and torch.equal(cnt, ecnt), "graph %d: detection block" % k
    # the three graphs saw different scenes, so equality above is not the same answer three times
    assert not torch.equal(results[0][0][1][-1], results[1][0][1][-1])


# ---------------------------------------------------------------------------------------------------------------------
# 4. float64 restatement of every inference layer and of the head, teacher-forced
# ---------------------------------------------------------------------------------------------------------------------
def conv64(params, scope, x, bn, relu):
    """tf_util.conv2d / conv1d at inference: x.W + b, BatchNorm with the moving statistics, ReLU -- float64, from the
    raw parameter dict."""
    t = lambda k: torch.from_numpy(np.asarray(params[scope + k], np.float64)).to(x.device)
    y = x @ t("/weights")
    if scope + "/biases" in params:
        y = y + t("/biases")
    if bn:
        y = (y - t("/bn/moving_mean")) / torch.sqrt(t("/bn/moving_variance") + BN_EPS) * t("/bn/gamma") + t("/bn/beta")
    return torch.relu(y) if relu else y


def gather_rows(x, idx):
    """x (b, n, c), idx (b, ...) -> x[s, idx[s, ...]]."""
    b = x.shape[0]
    flat = idx.reshape(b, -1).long()
    return torch.gather(x, 1, flat.unsqueeze(-1).expand(-1, -1, x.shape[-1])).view(*idx.shape, x.shape[-1])


def sa_layer64(params, spec, xyz, feats, fps_idx, src_xyz, idx_list, cnt_list):
    """pointnet_sa_module_msg after the sampling (layers_util.py:116-185) in float64 on the run's own indices."""
    radius, nsample, mlps, bn, scope, agg = spec[2], spec[3], spec[4], spec[5], spec[12], spec[15]
    new_xyz = gather_rows(src_xyz, fps_idx)
    outs = []
    for i in range(len(radius)):
        idx, cnt = idx_list[i], cnt_list[i]
        g_xyz = gather_rows(xyz, idx) - new_xyz.unsqueeze(2)
        g = torch.cat([gather_rows(feats, idx), g_xyz], dim=-1)                  # features first
        for j in range(len(mlps[i])):
            g = conv64(params, "%s/conv%d_%d" % (scope, i, j), g, bn, True)
        outs.append(g.amax(dim=2) * (cnt > 0).unsqueeze(-1).double())
    new_points = torch.cat(outs, dim=-1)
    if agg is not None and agg != -1:
        new_points = conv64(params, scope + "/ensemble", new_points, bn, True)
    return new_xyz, new_points


@pytest.mark.gpu
def test_every_layer_vs_float64(pkg, bench, step):
    every_layer_vs_float64(pkg, bench, step)


def every_layer_vs_float64(pkg, bench, step):
    """Every inference layer and the head of a step against float64, teacher-forced on the step's own indices."""
    (xyz_l, feat_l, fps_l, dbg), (_, _, raw) = step
    d = lambda t: t.double()
    checked = []
    for li, spec in enumerate(bench.arch, start=1):
        xyz_i, feat_i, ltype, vote_idx = spec[0][0], spec[1][0], spec[11], spec[14]
        xin, fin = d(xyz_l[xyz_i]), d(feat_l[feat_i])
        if ltype == "SA_Layer" and len(spec[2]):
            src = xyz_l[vote_idx] if vote_idx != -1 else xyz_l[xyz_i]
            nx, nf = sa_layer64(bench.params, spec, xin, fin, fps_l[li], d(src), dbg[li - 1]["idx"], dbg[li - 1]["cnt"])
            assert torch.equal(nx.float(), xyz_l[li]), "centres of layer %d" % li
            assert_close(feat_l[li], nf, "features of layer %d" % li)
        elif ltype == "SA_Layer":                 # no grouping: the sampled points themselves (:186-187)
            assert torch.equal(xyz_l[li], gather_rows(xyz_l[xyz_i], fps_l[li])), "xyz of layer %d" % li
            assert torch.equal(feat_l[li], gather_rows(feat_l[feat_i], fps_l[li])), "features of layer %d" % li
        elif ltype == "Vote_Layer":
            scope, f = spec[12], fin
            for i in range(len(spec[4])):
                f = conv64(bench.params, "%s/vote_layer_%d" % (scope, i), f, spec[5], True)
            off = conv64(bench.params, scope + "/vote_offsets", f, False, False)
            lo = torch.tensor(pkg.config.MAX_TRANSLATE_RANGE, dtype=torch.float64, device=bench.dev)
            assert_close(feat_l[li], f, "vote features")
            assert_close(dbg[li - 1]["offsets"][..., :3], off, "vote offsets")
            assert_close(xyz_l[li], xin + torch.minimum(torch.maximum(off, lo), -lo), "vote xyz")
            # the translation itself, on the run's own offsets, in float32: xyz + min(max(off, lo), -lo)
            off32, lo32 = dbg[li - 1]["offsets"][..., :3], lo.float()
            assert torch.equal(xyz_l[li], xyz_l[xyz_i] + torch.minimum(torch.maximum(off32, lo32), -lo32)), "vote translate"
        else:
            raise AssertionError("unexpected layer type %r" % ltype)
        checked.append(ltype)
    assert checked.count("SA_Layer") == 5 and checked.count("Vote_Layer") == 1
    # the head (head_builder.py:93-95, head_util.py:26-59) on the run's own CG-layer features
    hp = bench.head_params
    y = conv64(hp, "conv1d_0", d(feat_l[6]), True, True)
    cls = conv64(hp, "pred_cls", conv64(hp, "pred_cls_base", y, True, True), False, False)
    reg = conv64(hp, "pred_reg", conv64(hp, "pred_reg_base", y, True, True), False, False)
    assert_close(raw["feat"], y, "head conv1d_0")
    assert_close(raw["cls"], cls, "head cls")
    assert_close(head_reg(raw), reg, "head reg")


# ---------------------------------------------------------------------------------------------------------------------
# 5. decode and NMS
# ---------------------------------------------------------------------------------------------------------------------
ANGLE_BINS = 12
INTERVAL = torch.tensor(np.float32(2 * math.pi / ANGLE_BINS))     # the kernel's (float)(2*pi/12)


def decode32(ctr, reg):
    """decode_dist_anchor_free + decode_class2angle (anchor_decoder.py:6-14, :86-112) in float32 with the reference's
    operation order: angle = (bin + res[bin]) * interval, ctr = (xyz + d[:3]) + (0, h/2, 0), lhw = max(2*half, 0.1)."""
    bins = torch.argmax(reg[..., 6:6 + ANGLE_BINS], dim=-1)          # first maximum, like tf.argmax
    res = torch.gather(reg[..., 6 + ANGLE_BINS:6 + 2 * ANGLE_BINS], -1, bins.unsqueeze(-1))[..., 0]
    angle = (bins.float() + res) * INTERVAL.to(reg.device)
    x = ctr[..., 0] + reg[..., 0]
    y = (ctr[..., 1] + reg[..., 1]) + reg[..., 4]
    z = ctr[..., 2] + reg[..., 2]
    lhw = torch.maximum(reg[..., 3:6] * 2.0, torch.tensor(np.float32(0.1), device=reg.device))
    return torch.cat([torch.stack([x, y, z], -1), lhw, angle.unsqueeze(-1)], dim=-1), bins


def assert_scores_2ulp(got, cls):
    exp = 1.0 / (1.0 + np.exp(-cls.double().cpu().numpy()))
    g = got.cpu().numpy().astype(np.float64)
    ulp = np.spacing(exp.astype(np.float32)).astype(np.float64)
    over = np.abs(g - exp) > 2 * ulp
    assert not over.any(), "score beyond 2 ulp of the float64 sigmoid at %d of %d candidates (worst %.2f ulp)" % (
        over.sum(), over.size, (np.abs(g - exp) / ulp).max())


@pytest.mark.gpu
def test_decode_and_nms(pkg, bench, step):
    decode_and_nms(pkg, step)


def decode_and_nms(pkg, step):
    """A step's decoded boxes and scores, forced ties on scene 0's outputs, and the BEV NMS of every scene."""
    from oracle import head as ohead
    (xyz_l, feat_l, _, _), (blk, cnt, raw) = step
    ctr, reg, cls = xyz_l[6], head_reg(raw), raw["cls"]
    boxes, _ = decode32(ctr, reg)
    assert torch.equal(raw["boxes"][:, :, 0], boxes), "decoded boxes"
    assert_scores_2ulp(raw["score"][..., 0], cls[..., 0])
    # forced ties between angle bins and sizes at / below the 0.1 floor, on a slice of the run's own outputs
    n = 48
    r = reg[0, :n].clone()
    rows = torch.arange(n, device=r.device)
    a, b = rows % 5, 5 + rows % 7                                     # bins a < b tie at the maximum
    top = r[:, 6:6 + ANGLE_BINS].amax(dim=-1) + 1.0
    r[rows, 6 + a] = top
    r[rows, 6 + b] = top
    r[:16, 3:6] = torch.tensor([[-1.0, 0.0, 0.04], [0.05, 0.0499, 0.051]], device=r.device).repeat(8, 1)
    gb, gs = pkg.tf_ops.decode_dist_anchor_free(ctr[0:1, :n].contiguous(), r[None].contiguous(), cls[0:1, :n].contiguous(),
                                                ANGLE_BINS)
    eb, bins = decode32(ctr[0:1, :n], r[None])
    assert torch.equal(bins[0], a), "tf.argmax takes the first of tied maxima"
    assert torch.equal(gb, eb), "decoded boxes with tied bins and floored sizes"
    assert torch.equal(gb[0, :, 6], (a.float() + r[rows, 6 + ANGLE_BINS + a]) * INTERVAL.to(r.device))
    floor = np.float32(0.1)
    assert (gb[0, :16, 3:6] == floor).sum() >= 16 * 3 - 8 and (gb[0, :16, 3:6] >= floor).all()
    assert (gb[0, :16, 3:6] > floor).any()            # 2 * 0.051 > 0.1 stays unfloored
    assert_scores_2ulp(gs[0], cls[0, :n, 0])
    # the BEV NMS on the GPU's own boxes and scores: the oracle's greedy NMS, bit for bit, every scene
    eblk, ecnt = ohead.bev_nms(raw["boxes"][:, :, 0].cpu().numpy(), raw["score"][..., 0].cpu().numpy(), 0.1, 100)
    np.testing.assert_array_equal(cnt.cpu().numpy(), ecnt)
    np.testing.assert_array_equal(blk.cpu().numpy(), eblk)
    assert int(cnt.min()) >= 1


# ---------------------------------------------------------------------------------------------------------------------
# 6. FPS and ball query against float64 distances
# ---------------------------------------------------------------------------------------------------------------------
def fps_shortfall(p, idx):
    """For sampled indices idx (b, m) of points p (b, n, c) float64: per round j >= 1, how far the float64 running
    min-distance of sample j falls short of the largest one over all points (>= 0), and that largest one."""
    b, n, _ = p.shape
    idx = idx.long()
    rows = torch.arange(b, device=p.device)
    md = torch.full((b, n), float("inf"), dtype=torch.float64, device=p.device)
    short = torch.empty((b, idx.shape[1] - 1), dtype=torch.float64, device=p.device)
    best = torch.empty_like(short)
    for j in range(1, idx.shape[1]):
        prev = p[rows, idx[:, j - 1]]
        md = torch.minimum(md, ((p - prev.unsqueeze(1)) ** 2).sum(-1))
        best[:, j - 1] = md.amax(dim=1)
        short[:, j - 1] = best[:, j - 1] - md[rows, idx[:, j]]
    return short, best


def assert_fps(p, idx, what, feature_space=False):
    """Sample 0 is point 0 and every later sample maximises the running min-distance, within 1e-6 relative.  D-FPS
    evaluates coordinate differences, so 'relative' is to the distance itself.  F-FPS evaluates the reference's norm
    expansion (|a|^2 + |b|^2) - 2 a.b in float32 (model_util.calc_square_dist), which cannot order distances closer than
    a few ulp of |a|^2 + |b|^2, so there it is relative to 2 max|p|^2 of the scene."""
    assert (idx[:, 0] == 0).all(), "%s: first sample" % what
    short, best = fps_shortfall(p, idx)
    scale = 2 * (p ** 2).sum(-1).amax(dim=1, keepdim=True) if feature_space else best
    bad = short > 1e-6 * scale
    if bad.any():
        s, j = [int(v) for v in bad.nonzero()[0]]
        raise AssertionError("%s: scene %d round %d picks a point %g short of the farthest (%g), %d rounds over"
                             % (what, s, j + 1, float(short[s, j]), float(best[s, j]), int(bad.sum())))


@pytest.mark.gpu
def test_fps_farthest_point_property(bench, step):
    fps_farthest_point_property(step)


def fps_farthest_point_property(step):
    """Every D-FPS and F-FPS of a step maximises the running min-distance (assert_fps)."""
    xyz_l, feat_l, fps_l, _ = step[0]
    d = lambda t: t.double()
    assert_fps(d(xyz_l[0]), fps_l[1], "layer-1 D-FPS")
    assert_fps(d(xyz_l[1]), fps_l[2][:, 512:], "layer-2 D-FPS")
    assert_fps(d(xyz_l[2][:, 512:]), fps_l[3][:, 256:] - 512, "layer-3 D-FPS")
    assert_fps(torch.cat([d(xyz_l[1]), d(feat_l[1])], -1), fps_l[2][:, :512], "layer-2 F-FPS (direct)", feature_space=True)
    assert_fps(torch.cat([d(xyz_l[2][:, :512]), d(feat_l[2][:, :512])], -1), fps_l[3][:, :256], "layer-3 F-FPS (matrix)",
               feature_space=True)


def ball_query_check(xyz, new_xyz, radii, nsamples, dilated, idx_list, cnt_list, what, chunk=128):
    """Every centre and scale against float64 squared distances: cnt = min(#in-shell, K) and idx[:cnt] = the first
    in-shell points in index order, the rest padded with the first hit (zeros for an empty shell).  In-shell is
    d == 0 or r_lo <= d < r_hi (dilated), d < r (plain), with the float32 radii.  A centre is left out when a point
    within 1e-6 relative of one of its shell boundaries (in d^2) lies where the scan could reach it."""
    b, m, _ = new_xyz.shape
    x, c = xyz.double(), new_xyz.double()
    r32 = [float(np.float32(r)) for r in radii]
    total = dirty = 0
    for q0 in range(0, m, chunk):
        cq = c[:, q0:q0 + chunk]
        d2 = sum((cq[..., k:k + 1] - x[..., k].unsqueeze(1)) ** 2 for k in range(3))       # (b, mq, n)
        for sc, (r, k) in enumerate(zip(r32, nsamples)):
            r_lo = (r32[sc - 1] if sc > 0 else 0.0) if dilated else 0.0
            hit = d2 < r * r
            amb = (d2 - r * r).abs() <= 1e-6 * r * r
            if r_lo > 0:
                hit &= d2 >= r_lo * r_lo
                amb |= (d2 - r_lo * r_lo).abs() <= 1e-6 * r_lo * r_lo
            if dilated:
                hit |= d2 == 0
            amb &= d2 != 0
            hit &= ~amb
            cum = hit.int().cumsum(-1)
            reach = (cum - hit.int()) < k                    # the scan stops after the k-th hit
            clean = ~(amb & reach).any(-1)
            ecnt = torch.clamp(cum[..., -1], max=k)
            eidx = torch.zeros((b, cq.shape[1], k), dtype=torch.long, device=x.device)
            s_, q_, p_ = (hit & (cum <= k)).nonzero(as_tuple=True)
            eidx[s_, q_, cum[s_, q_, p_].long() - 1] = p_
            slot = torch.arange(k, device=x.device)
            eidx = torch.where(slot < ecnt.unsqueeze(-1), eidx, eidx[..., :1])
            gi = idx_list[sc][:, q0:q0 + chunk].long()
            gc = cnt_list[sc][:, q0:q0 + chunk]
            ok = (gc == ecnt) & (gi == eidx).all(-1)
            bad = clean & ~ok
            if bad.any():
                s, q = [int(v) for v in bad.nonzero()[0]]
                raise AssertionError("%s scale %d, scene %d centre %d: cnt %d idx %s, float64 says cnt %d idx %s"
                                     % (what, sc, s, q0 + q, int(gc[s, q]), gi[s, q, :8].tolist(), int(ecnt[s, q]),
                                        eidx[s, q, :8].tolist()))
            total += clean.numel()
            dirty += int((~clean).sum())
    assert dirty <= 1e-3 * total, "%s: %d of %d centres too close to a shell boundary to judge" % (what, dirty, total)


@pytest.mark.gpu
def test_ball_query_vs_float64(bench, step):
    ball_query_vs_float64(bench, step)


def ball_query_vs_float64(bench, step):
    """Every ball query of a step against float64 squared distances (ball_query_check)."""
    xyz_l, _, _, dbg = step[0]
    for li, spec in enumerate(bench.arch, start=1):
        if spec[11] != "SA_Layer" or not len(spec[2]):
            continue
        ball_query_check(xyz_l[spec[0][0]], xyz_l[li], spec[2], spec[3], spec[13], dbg[li - 1]["idx"], dbg[li - 1]["cnt"],
                         "layer %d ball query" % li)


# ---------------------------------------------------------------------------------------------------------------------
# 7. the CPU oracle, layer by layer, on the batch's last scene
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_last_scene_vs_oracle_layerwise(oracle_ops, bench, step):
    """Teacher-forced: every oracle layer takes scene 7's own GPU outputs of the layers before it, so the indices
    (D-FPS, F-FPS on features, ball query) must match bit for bit by construction of the arithmetic."""
    scene_vs_oracle_layerwise(oracle_ops, bench.arch, bench.params, step, SCENES - 1)


def scene_vs_oracle_layerwise(oracle_ops, arch, params, step, s):
    """Scene s of a step against the CPU oracle, layer by layer on the step's own inputs to each layer: SA, vote and FP
    layers of the table `arch` with the raw parameter dict `params` (an SA layer whose aggregation_channel is -1 has no
    aggregation conv)."""
    from oracle import layers as olayers
    xyz_l, feat_l, fps_l, dbg = step[0]
    npy = lambda t: None if t is None else t[s:s + 1].cpu().numpy()
    for li, spec in enumerate(arch, start=1):
        (xyz_i, feat_i, radius, nsample, mlps, bn, rng, method, npoint, former, attn, ltype, scope, dilated,
         vote_idx, agg) = spec
        xin, fin = npy(xyz_l[xyz_i[0]]), npy(feat_l[feat_i[0]])
        if ltype == "SA_Layer":
            former_idx = npy(fps_l[former]) if former != -1 else None
            vote_ctr = npy(xyz_l[vote_idx]) if vote_idx != -1 else None
            ex, ef, ei, ed = olayers.pointnet_sa_module_msg(xin, fin, radius, nsample, mlps, False, None, bn, rng, method,
                                                            npoint, former_idx, attn, scope, dilated, vote_ctr, agg,
                                                            params=params, ffps_mode="matrix", return_debug=True)
            np.testing.assert_array_equal(npy(fps_l[li]), ei, err_msg="fps_idx of layer %d" % li)
            for sc, (a, b) in enumerate(zip(dbg[li - 1].get("idx", []), ed["idx"])):
                np.testing.assert_array_equal(npy(a), b, err_msg="ball-query idx layer %d scale %d" % (li, sc))
            for sc, (a, b) in enumerate(zip(dbg[li - 1].get("cnt", []), ed["cnt"])):
                np.testing.assert_array_equal(npy(a), b, err_msg="pts_cnt layer %d scale %d" % (li, sc))
            np.testing.assert_array_equal(npy(xyz_l[li]), ex, err_msg="new_xyz of layer %d" % li)
        elif ltype == "Vote_Layer":
            ex, ef, _ = olayers.vote_layer(xin, fin, mlps, False, None, bn, scope, params=params)
            e = rel_err(npy(xyz_l[li]), ex, rtol=FEATURE_TOL)
            assert e < FEATURE_TOL, "vote xyz of layer %d: rel err %g" % (li, e)
        elif ltype == "FP_Layer":                 # unknown points xyz_i[0], known points and features xyz_i[1] / feat_i[1]
            ef = olayers.pointnet_fp_module(xin, npy(xyz_l[xyz_i[1]]), fin, npy(feat_l[feat_i[1]]), mlps, False, None, scope,
                                            bn, params=params)
            np.testing.assert_array_equal(npy(xyz_l[li]), xin, err_msg="xyz of layer %d" % li)
        else:
            raise AssertionError("unexpected layer type %r" % ltype)
        e = rel_err(npy(feat_l[li]), ef, rtol=FEATURE_TOL)
        assert e < FEATURE_TOL, "features of layer %d: rel err %g" % (li, e)
