"""PointRCNN's second stage at the shape tools/time_pointrcnn_rcnn.py times: batches of eight 16 384-point scenes through
the two-stage net of tests/test_pointrcnn_rcnn_gpu.py, eager with the debug outputs.  Three batches:
  * "real":  the eight real-scan scenes S0..S7 of tests/test_realscan_cpu.py;
  * "timed": synth.kitti_like(8, 16384) with time_pointrcnn_rcnn.py's seed;
  * "short": S0..S6 and, in S7's place, 60 distinct points of S7's region filled to 16 384 with the loader's copies, so
             its RPN block stops short of 100 proposals.

Checked on each batch:
  * the pool on the forward's own inputs, every row: the mask from the float64 sigmoid of the RPN's logits, the
    canonical xyz, the info conv in float64, the copied rpn_fp_layer1 features, the stage-2 centres;
  * rcnn_layer1 and rcnn_layer2 against float64 teacher-forced on all B * 100 pooled scenes, padding included;
and: short blocks through the whole forward (padding pools nothing and is never kept, S0..S6 are the real batch's
bits), real proposals with an empty pool, every scene alone equal to its row of the batch, and three concurrent CUDA
graphs of the one net."""
import importlib

import numpy as np
import pytest
import torch

from test_bench_step_gpu import FEATURE_TOL, assert_fps, conv64, rel_err, sa_layer64
from test_pointrcnn_rcnn_cpu import canonical_np, expand, scan_np
from test_realscan_cpu import NAMES, distinct_rows, loader_choice, realscan_scenes, scene_sources

pytestmark = pytest.mark.gpu

synth = importlib.import_module("3dssd_b200.synth")
C = importlib.import_module("3dssd_b200.config")

B, NPOINTS, P, NS = 8, 16384, 100, 512          # scenes, points per scene, proposals per scene, pooled points
TIMED_SEED = 21                                 # tools/time_pointrcnn_rcnn.py --seed
BATCHES = ["real", "timed", "short"]
SHORT = NAMES.index("S7")                       # the short batch's scene of 60 distinct points
CHUNK = 100                                     # pooled scenes per float64 chunk
MASK_AMBIGUOUS = 2.0 ** -24                     # one float32 ulp of 0.5 (above it; two below)
STAGE = C.STAGE_POINTRCNN_RCNN


def short_scene():
    """60 distinct points of S7's region, filled to 16 384 by the loader's choice (tests/test_pointrcnn_step_gpu.py)"""
    src = scene_sources()["S7"][:60]
    pts = src[loader_choice(len(src), np.random.default_rng(7))]
    assert distinct_rows(pts) == 60
    return pts


def batch_points(name):
    if name == "timed":
        return np.ascontiguousarray(synth.kitti_like(B, NPOINTS, seed=TIMED_SEED), np.float32)
    pts = realscan_scenes()[0]
    if name == "short":
        pts[SHORT] = short_scene()
    return np.ascontiguousarray(pts, np.float32)


class Run:
    pass


@pytest.fixture(scope="module")
def net(pkg, cuda):
    return pkg.PointRCNN(device=cuda, seed=0)


@pytest.fixture(scope="module")
def runs(cuda, net):
    """name -> the batch's eager forward with return_debug=True (computed once)"""
    cache = {}

    def get(name):
        if name not in cache:
            r = Run()
            r.pts = torch.from_numpy(batch_points(name)).to(cuda)
            r.block, r.count, r.d = net.forward(r.pts, return_debug=True)
            torch.cuda.synchronize()
            cache[name] = r
        return cache[name]
    return get


def outputs(block, count, d):
    """Every output of one forward from the RPN's proposals to the block, by name."""
    t = {"rpn score": d["rpn_raw"]["score"], "block": block, "count": count}
    for k in ("proposals", "proposal_count", "pool_xyz", "pool_feat", "pool_idx", "pool_cnt", "ctr", "cls", "reg", "boxes",
              "scores"):
        t[k] = d[k]
    for what in ("xyz", "feat", "fps"):
        for li, x in enumerate(d["rcnn_" + what]):
            if x is not None:
                t["rcnn %s %d" % (what, li)] = x
    for li, dbg in enumerate(d["rcnn_dbg"]):
        for sc, (i, c) in enumerate(zip(dbg.get("idx", []), dbg.get("cnt", []))):
            t["rcnn layer %d scale %d idx" % (li + 1, sc)] = i
            t["rcnn layer %d scale %d cnt" % (li + 1, sc)] = c
    return t


def scene_rows(x, s, b):
    """Scene s's rows of a tensor whose leading dimension is b scenes or b * P pooled scenes."""
    per = x.shape[0] // b
    assert per * b == x.shape[0]
    return x[s * per:(s + 1) * per]


def assert_scene_equal(got, gb, gs, exp, eb, es, what):
    """Scene gs of a b = gb run has scene es's bits of a b = eb run at every output."""
    assert got.keys() == exp.keys()
    for k in exp:
        g, e = scene_rows(got[k], gs, gb), scene_rows(exp[k], es, eb)
        assert g.shape == e.shape, "%s: %s shape %s vs %s" % (what, k, tuple(g.shape), tuple(e.shape))
        assert torch.equal(g, e), "%s: %s differs" % (what, k)


def assert_block_is_c_twins(oracle_ops, block, count, d, what):
    """Each scene's block and count are the C twin's BEV NMS over its real proposals only, bit for bit; padding rows
    (at or past the proposal count) have score 0, pool nothing, and no kept box is one of them alone."""
    boxes, scores = d["boxes"].cpu().numpy(), d["scores"].cpu().numpy()
    pcount = d["proposal_count"].cpu().numpy()
    pcnt, pidx = d["pool_cnt"].cpu().numpy(), d["pool_idx"].cpu().numpy()
    blk, cnt = block.cpu().numpy(), count.cpu().numpy()
    for s in range(len(pcount)):
        nv = int(pcount[s])
        assert not pcnt[s, nv:].any() and not pidx[s, nv:].any(), "%s: scene %d pools padding rows" % (what, s)
        assert not scores[s, nv:].any(), "%s: scene %d scores padding rows" % (what, s)
        if nv == 0:
            assert cnt[s] == 0 and not blk[s].any()
            continue
        eblk, ecnt = oracle_ops.bev_nms(boxes[s:s + 1, :nv], scores[s:s + 1, :nv], STAGE["NMS_THRESH"], STAGE["MAX_OUTPUT_NUM"])
        assert cnt[s] == ecnt[0], "%s: scene %d keeps %d boxes, the C twin %d" % (what, s, cnt[s], ecnt[0])
        np.testing.assert_array_equal(blk[s].view(np.uint32), eblk[0].view(np.uint32), err_msg="%s: scene %d" % (what, s))
        for k in range(cnt[s]):
            hit = np.flatnonzero((boxes[s] == blk[s, k, :7]).all(-1))
            assert len(hit) and hit.min() < nv, "%s: scene %d keeps a padding row" % (what, s)


# ---------------------------------------------------------------------------------------------------------------------
# A. the pool on the forward's own inputs
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", BATCHES)
def test_pool_on_the_forward_inputs(pkg, cuda, net, runs, name):
    """region_pool as PointRCNN.forward calls it, every row of the batch, against values computed from the RPN's debug
    outputs alone: the scan of each expanded proposal (the box query kernel and, wherever no point is ambiguous, the
    numpy scan); the mask as the float64 sigmoid of the RPN's per-point logit >= 0.5 (points within an ulp of 0.5 left
    out and counted); the canonical xyz in float32; the info conv in float64; the features of rpn_fp_layer1 (the RPN's
    last layer) copied bit for bit; and the stage-2 centres y - h/2 of the proposals in float32."""
    r = runs(name)
    d = r.d
    xyz, feat = d["rpn_xyz"][-1], d["rpn_feat"][-1]
    assert tuple(xyz.shape) == (B, NPOINTS, 3) and feat.shape[:2] == (B, NPOINTS)
    sig = torch.sigmoid(d["rpn_raw"]["cls"][..., 0].double())
    amb = (sig - 0.5).abs() <= MASK_AMBIGUOUS
    print("\n%s: %d of %d points have a sigmoid within an ulp of 0.5" % (name, int(amb.sum()), amb.numel()))
    assert amb.sum() <= 16
    props, pcount = d["proposals"], d["proposal_count"]
    valid = torch.arange(P, device=cuda)[None] < pcount[:, None].long()
    pidx, pcnt = d["pool_idx"], d["pool_cnt"]
    assert tuple(pidx.shape) == (B, P, NS) and tuple(pcnt.shape) == (B, P)
    # the scan: the box query on the expanded block (the same device function), and the numpy scan
    props_np, xyz_np = props.cpu().numpy(), xyz.cpu().numpy()
    ex = np.stack([np.stack([expand(props_np[s, q]) for q in range(P)]) for s in range(B)])
    qi, qc = pkg.tf_ops.query_boxes_3d_points(NS, xyz, torch.from_numpy(ex).to(cuda))
    assert torch.equal(pcnt, torch.where(valid, qc, 0))
    assert torch.equal(pidx, torch.where(valid[..., None], qi, 0))
    idx_np, cnt_np, vnp = pidx.cpu().numpy(), pcnt.cpu().numpy(), valid.cpu().numpy()
    compared = 0
    for s in range(B):
        for q in np.flatnonzero(vnp[s]):
            i, c, a = scan_np(xyz_np[s], ex[s, q], NS)
            if a == 0:
                compared += 1
                assert c == cnt_np[s, q] and np.array_equal(i, idx_np[s, q]), "%s: scan of scene %d proposal %d" % (name, s, q)
    assert compared >= 0.9 * vnp.sum()
    empty = int((vnp & (cnt_np == 0)).sum())
    print("%s: proposal counts %s, %d real proposals with an empty pool" % (name, pcount.tolist(), empty))
    # canonical xyz, every row (padding rows transform point 0 by their own block row)
    pxyz = d["pool_xyz"].cpu().numpy().reshape(B, P, NS, 3)
    for s in range(B):
        for q in range(P):
            can = canonical_np(xyz_np[s, idx_np[s, q]], props_np[s, q])
            np.testing.assert_allclose(pxyz[s, q], can, rtol=0, atol=4 * np.spacing(np.float32(np.abs(can).max() + 1)),
                                       err_msg="%s: canonical xyz of scene %d proposal %d" % (name, s, q))
    # [info conv | features], in chunks of CHUNK pooled scenes
    prm = net.params.raw
    co = prm["roi_pool/conv0/weights"].shape[1]
    pfeat = d["pool_feat"]
    assert tuple(pfeat.shape) == (B * P, NS, co + feat.shape[2])
    flat_idx = pidx.view(B * P, NS).long()
    scene = torch.arange(B * P, device=cuda) // P
    worst, left_out = 0.0, 0
    for lo in range(0, B * P, CHUNK):
        sl = slice(lo, lo + CHUNK)
        k, sc = flat_idx[sl], scene[sl, None].expand(-1, NS)
        p64 = xyz[sc, k].double()
        info = torch.cat([d["pool_xyz"][sl].double(), (sig[sc, k] >= 0.5).double()[..., None], p64.norm(dim=-1, keepdim=True)], -1)
        exp = conv64(prm, "roi_pool/conv0", info, True, True)
        got = pfeat[sl, :, :co].double()
        a = amb[sc, k]
        left_out += int(a.sum())
        exp[a], got[a] = 0.0, 0.0
        e = rel_err(got.cpu().numpy(), exp.cpu().numpy(), rtol=FEATURE_TOL)
        assert e < FEATURE_TOL, "%s: info conv of pooled scenes %d..%d: rel err %g" % (name, lo, lo + CHUNK - 1, e)
        worst = max(worst, e)
        assert torch.equal(pfeat[sl, :, co:], feat[sc, k]), "%s: copied features of pooled scenes %d.." % (name, lo)
    print("%s: info conv worst rel err %.3g, %d pooled points left out as ambiguous" % (name, worst, left_out))
    # the stage-2 centres and the lists the stage-2 layers start from
    ctr = d["ctr"].cpu().numpy()
    f32 = props_np.astype(np.float32)
    np.testing.assert_array_equal(ctr[..., 1].view(np.uint32), (f32[..., 1] - f32[..., 4] / np.float32(2)).view(np.uint32))
    np.testing.assert_array_equal(ctr[..., [0, 2]].view(np.uint32), f32[..., [0, 2]].view(np.uint32))
    xl, fl = d["rcnn_xyz"], d["rcnn_feat"]
    assert torch.equal(xl[0], d["ctr"]) and torch.equal(xl[1], d["pool_xyz"]) and torch.equal(fl[1], pfeat)


# ---------------------------------------------------------------------------------------------------------------------
# B. every pooled scene against float64
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", BATCHES)
def test_stage2_sa_layers_every_row_vs_float64(net, runs, name):
    """rcnn_layer1 and rcnn_layer2 teacher-forced on their own D-FPS indices and neighbour lists over all B * 100
    pooled scenes, padding rows (512 copies of one point) included: centres bit for bit, features at FEATURE_TOL,
    every D-FPS a farthest-point walk in float64."""
    d = runs(name).d
    prm = net.params.raw
    xl, fl, fps, dbg = d["rcnn_xyz"], d["rcnn_feat"], d["rcnn_fps"], d["rcnn_dbg"]
    rows = xl[1].shape[0]
    assert rows == B * P
    for li, spec in ((2, C.ARCH_POINTRCNN_RCNN[0]), (3, C.ARCH_POINTRCNN_RCNN[1])):
        xi, fi, scope = spec[0][0], spec[1][0], spec[12]
        idx, cnt = dbg[li - 2]["idx"], dbg[li - 2]["cnt"]
        spec64 = list(spec[:15]) + [-1]
        worst = 0.0
        for lo in range(0, rows, CHUNK):
            sl = slice(lo, lo + CHUNK)
            x64 = xl[xi][sl].double()
            nx, nf = sa_layer64(prm, spec64, x64, fl[fi][sl].double(), fps[li][sl], x64, [i[sl] for i in idx], [c[sl] for c in cnt])
            what = "%s: %s on pooled scenes %d..%d" % (name, scope, lo, lo + CHUNK - 1)
            assert torch.equal(nx.float(), xl[li][sl]), what + ": centres"
            e = rel_err(fl[li][sl].double().cpu().numpy(), nf.cpu().numpy(), rtol=FEATURE_TOL)
            assert e < FEATURE_TOL, "%s: features rel err %g" % (what, e)
            worst = max(worst, e)
            assert_fps(x64, fps[li][sl], what + ": D-FPS")
        print("\n%s: %s worst rel err %.3g over %d pooled scenes" % (name, scope, worst, rows))


# ---------------------------------------------------------------------------------------------------------------------
# C. short proposal blocks through the whole forward
# ---------------------------------------------------------------------------------------------------------------------
def test_short_block_through_the_forward(oracle_ops, runs):
    """S7's 60 distinct points give at most 60 proposals: its padding rows pool nothing, score 0 and are never kept,
    and the block is the C twin's over the real rows.  Scenes S0..S6 are the real batch's bits at every output from
    the proposals to the block."""
    r = runs("short")
    pcount = r.d["proposal_count"].cpu().numpy()
    print("\nshort: proposal counts %s" % pcount.tolist())
    assert pcount[SHORT] < P and pcount[SHORT] <= 60
    assert_block_is_c_twins(oracle_ops, r.block, r.count, r.d, "short")
    real = runs("real")
    got, exp = outputs(r.block, r.count, r.d), outputs(real.block, real.count, real.d)
    for s in range(B):
        if s != SHORT:
            assert_scene_equal(got, B, s, exp, B, s, "short batch scene %s" % NAMES[s])


def test_real_proposals_with_an_empty_pool(oracle_ops, monkeypatch, net, runs):
    """Real proposals 500 m from every point (the RPN head's block moved on this net only, its count kept): they pool
    nothing and score 0, yet stay candidates of the NMS, whose block is still the C twin's; every other row pools as
    before."""
    r = runs("short")
    pcount, pcnt = r.d["proposal_count"].cpu().numpy(), r.d["pool_cnt"].cpu().numpy()
    moved = {}
    for s in (0, 3, SHORT):                                      # the first, a middle and the last that hold points
        held = np.flatnonzero(pcnt[s, :pcount[s]] > 0)
        moved[s] = sorted({int(held[0]), int(held[len(held) // 2]), int(held[-1])})
    head_forward = net.rpn_head.forward

    def far_rows(*a, **kw):
        block, count, raw = head_forward(*a, **kw)
        block = block.clone()
        for s, rows in moved.items():
            block[s, rows, 0] += 500.0
            block[s, rows, 2] += 500.0
        return block, count, raw

    monkeypatch.setattr(net.rpn_head, "forward", far_rows)
    block, count, d = net.forward(r.pts, return_debug=True)
    torch.cuda.synchronize()
    monkeypatch.undo()
    assert torch.equal(d["proposal_count"], r.d["proposal_count"])
    far = torch.zeros((B, P), dtype=torch.bool, device=block.device)
    for s, rows in moved.items():
        far[s, rows] = True
    assert not d["pool_cnt"][far].any() and not d["scores"][far].any()
    assert (r.d["pool_cnt"][far] > 0).all()                        # they held points where the RPN put them
    assert torch.equal(d["pool_cnt"][~far], r.d["pool_cnt"][~far]) and torch.equal(d["pool_idx"][~far], r.d["pool_idx"][~far])
    assert_block_is_c_twins(oracle_ops, block, count, d, "moved proposals")


# ---------------------------------------------------------------------------------------------------------------------
# D. batch independence
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["real", "timed"])
def test_every_scene_equals_its_single_scene_run(net, runs, name):
    """The pool indexes scenes by its grid's y, the stage-2 layers run B * 100 pooled scenes, the decode and the NMS
    run per scene: scene s alone (B = 1) is the same bits as its row of the B = 8 forward at every output."""
    r = runs(name)
    exp = outputs(r.block, r.count, r.d)
    for s in range(B):
        block, count, d = net.forward(r.pts[s:s + 1], return_debug=True)
        assert_scene_equal(outputs(block, count, d), 1, 0, exp, B, s, "%s scene %d alone" % (name, s))


# ---------------------------------------------------------------------------------------------------------------------
# F. concurrent CUDA graphs of one net
# ---------------------------------------------------------------------------------------------------------------------
def test_concurrent_graphs_of_one_two_stage_net(cuda, net, runs):
    """Three graphs of the one PointRCNN (the real, timed and short batches) replayed interleaved on three streams with
    no synchronisation between replays: each equals the eager forward of its own scenes, and they differ."""
    inputs = [runs(name).pts for name in BATCHES]
    runners = [net.capture(p) for p in inputs]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(device=cuda) for _ in inputs]
    main = torch.cuda.current_stream()
    for st in streams:
        st.wait_stream(main)
    results = [None] * len(inputs)
    for rnd in range(4):
        for j in range(len(inputs)):
            k = (j + rnd) % len(inputs)                  # rotate which graph is enqueued first
            with torch.cuda.stream(streams[k]):
                results[k] = runners[k]()
    for st in streams:
        main.wait_stream(st)
    torch.cuda.synchronize()
    for k, name in enumerate(BATCHES):
        blk, cnt = results[k]
        r = runs(name)
        assert torch.equal(blk, r.block) and torch.equal(cnt, r.count), "graph of the %s batch" % name
    for a in range(len(inputs)):
        for b in range(a + 1, len(inputs)):
            assert not torch.equal(results[a][0], results[b][0]), "graphs %s and %s" % (BATCHES[a], BATCHES[b])
