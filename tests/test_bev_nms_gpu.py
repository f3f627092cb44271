"""GPU tests (-m gpu) of the BEV NMS kernel (csrc/nms.cu) against both oracles, bit for bit in block and count, on the
boundary pairs and scenes of tests/test_bev_nms_cpu.py (IoU an ulp from the threshold, sort edges, degenerate boxes,
thresholds, output sizes, batches), into views of a larger buffer, and on the greedy property at full size against
the exact IoU of the float32 rectangles."""
import numpy as np
import pytest
import torch

from oracle import head as ohead
from test_bev_nms_cpu import REL_BOUND, boundary_pairs, clustered_boxes, exact_iou, iou64, near_threshold, nms_scenes

pytestmark = pytest.mark.gpu


def kernel(pkg, cuda, boxes, scores, thr, max_out, cls_id=0):
    blk, cnt = pkg.bev_nms(torch.from_numpy(boxes).to(cuda), torch.from_numpy(scores).to(cuda), thr, max_out, cls_id)
    return blk.cpu().numpy(), cnt.cpu().numpy()


def assert_same(got, exp, what):
    """Blocks bit for bit (a -0 score must stay -0), counts equal; on failure, the scenes and rows that differ."""
    (gb, gc), (eb, ec) = got, exp
    bad = np.flatnonzero(gc != ec)
    assert not len(bad), "%s: counts differ in %d of %d scenes, first %s: %s vs %s" % (
        what, len(bad), len(gc), bad[:5].tolist(), gc[bad[:5]].tolist(), ec[bad[:5]].tolist())
    rows = np.argwhere((gb.view(np.uint32) != eb.view(np.uint32)).any(-1))
    assert not len(rows), "%s: %d block rows differ, first (scene, row) %s" % (what, len(rows), rows[:5].tolist())


@pytest.mark.parametrize("thr", [0.1, 0.5])
def test_kernel_boundary_pairs(pkg, oracle_ops, cuda, thr):
    """Every boundary pair as a two-box scene: the last float32 position that suppresses and the first that keeps."""
    a, bs, bk = boundary_pairs(thr)
    boxes = np.ascontiguousarray(np.concatenate([np.stack([a, bs], 1), np.stack([a, bk], 1)]))
    scores = np.ascontiguousarray(np.broadcast_to(np.array([0.9, 0.8], np.float32), (len(boxes), 2)))
    got = kernel(pkg, cuda, boxes, scores, thr, 2)
    assert_same(got, ohead.bev_nms(boxes, scores, thr, 2), "kernel vs numpy oracle")
    assert_same(got, oracle_ops.bev_nms(boxes, scores, thr, 2), "kernel vs C oracle")


@pytest.mark.parametrize("name", list(nms_scenes()))
def test_kernel_scenes(pkg, oracle_ops, cuda, name):
    c = nms_scenes()[name]
    args = (c["thr"], c["max_out"], c["cls_id"])
    got = kernel(pkg, cuda, c["boxes"], c["scores"], *args)
    assert_same(got, ohead.bev_nms(c["boxes"], c["scores"], *args), "kernel vs numpy oracle")
    assert_same(got, oracle_ops.bev_nms(c["boxes"], c["scores"], *args), "kernel vs C oracle")


@pytest.mark.parametrize("b", [0, 1, 33])
def test_kernel_into_buffer_views(pkg, oracle_ops, cuda, b):
    """out= into views of a larger buffer, as the gather send buffer is written; the rows around the views keep their
    sentinels, and b = 0 launches nothing."""
    rng = np.random.default_rng(40 + b)
    n, max_out, cls_id = 100, 50, 5
    boxes = clustered_boxes(rng, b, n, objects=12) if b else np.zeros((0, n, 7), np.float32)
    scores = rng.uniform(0, 1, (b, n)).astype(np.float32)
    blk_buf = torch.full((b + 2, max_out, 9), -7.0, device=cuda)
    cnt_buf = torch.full((b + 2,), -7, dtype=torch.int32, device=cuda)
    out = (blk_buf[1:1 + b], cnt_buf[1:1 + b])
    rb, rc = pkg.bev_nms(torch.from_numpy(boxes).to(cuda), torch.from_numpy(scores).to(cuda), 0.1, max_out, cls_id, out=out)
    assert rb.data_ptr() == out[0].data_ptr() and rc.data_ptr() == out[1].data_ptr()
    blk, cnt = blk_buf.cpu().numpy(), cnt_buf.cpu().numpy()
    assert (blk[0] == -7).all() and (blk[b + 1] == -7).all() and cnt[0] == -7 and cnt[b + 1] == -7
    got = (blk[1:1 + b], cnt[1:1 + b])
    assert_same(got, ohead.bev_nms(boxes, scores, 0.1, max_out, cls_id), "kernel vs numpy oracle")
    assert_same(got, oracle_ops.bev_nms(boxes, scores, 0.1, max_out, cls_id), "kernel vs C oracle")


def _decide(ra, rb, thr):
    """Exact comparison of IoU(ra[i], rb[j]) with float32(thr) for all i, j: +1 above, -1 below, 0 within REL_BOUND
    (either decision is faithful there).  float64 decides where it is far from the threshold, Fraction elsewhere."""
    t = float(np.float32(thr))
    v = iou64(ra[:, None], rb[None])
    out = np.where(v > t, 1, -1)
    for i, j in np.argwhere(np.abs(v - t) <= 4 * float(REL_BOUND) * abs(t)):
        e = exact_iou(ra[i], rb[j])
        out[i, j] = 0 if near_threshold(e, thr) else (1 if e > t else -1)
    return out


def test_kernel_greedy_property_full_size(pkg, oracle_ops, cuda):
    """b = 8, n = 512, KITTI-like clusters, max_output = n (so nothing is cut off): kept boxes pairwise at IoU <= thr,
    every dropped candidate has a higher-ranked kept box at IoU > thr (both exact, within REL_BOUND), kept scores
    non-increasing -- and the same blocks as the C oracle."""
    rng = np.random.default_rng(50)
    b, n, thr = 8, 512, 0.1
    boxes = clustered_boxes(rng, b, n, objects=60, jitter=0.6)
    scores = rng.uniform(0, 1, (b, n)).astype(np.float32)
    blk, cnt = kernel(pkg, cuda, boxes, scores, thr, n)
    assert_same((blk, cnt), oracle_ops.bev_nms(boxes, scores, thr, n), "kernel vs C oracle")
    dropped_total = 0
    for s in range(b):
        k = int(cnt[s])
        assert (np.diff(blk[s, :k, 7]) <= 0).all() and (blk[s, k:] == 0).all()
        where = {row.tobytes(): i for i, row in enumerate(np.concatenate([boxes[s], scores[s][:, None]], 1))}
        kept = np.array([where[blk[s, r, :8].tobytes()] for r in range(k)])
        rank = np.empty(n, np.int64)
        rank[sorted(range(n), key=lambda i: (-float(scores[s, i]), i))] = np.arange(n)
        assert (np.diff(rank[kept]) > 0).all()
        rects = ohead.bev_rects(boxes[s])
        dk = _decide(rects[kept], rects[kept], thr)
        np.fill_diagonal(dk, -1)
        assert not (dk == 1).any(), "scene %d: kept boxes %s overlap above the threshold" % (s, np.argwhere(dk == 1)[:3])
        dropped = np.setdiff1d(np.arange(n), kept)
        dropped_total += len(dropped)
        dd = _decide(rects[dropped], rects[kept], thr)
        earlier = rank[kept][None, :] < rank[dropped][:, None]
        assert ((dd >= 0) & earlier).any(1).all(), "scene %d: a dropped candidate has no earlier kept box above it" % s
    assert dropped_total > b * n // 2
