"""CPU dry run of the layer orchestration (3dssd_b200/layers_util.py, backbone.py): every tf_ops entry point the fp32
route touches is replaced by a few lines on top of the CPU oracle, and torch.cuda's streams / events by inert stand-ins,
so that the PYTHON around the kernels -- segment placement into the shared fps_idx buffer, offsets, scene-strided slices,
resumable rounds, the latency-mode part schedule and its joins -- runs here without a GPU and must reproduce the
oracle's own layer code.  (The kernels themselves are covered by the -m gpu tests.)"""
import copy
import importlib
import inspect
import json
import os

import numpy as np
import pytest
import torch

_SYNC = {}   # state of the stream / event stand-ins: creation counters, the torch.cuda.stream stack, the trace (list or None)


def _reset_sync(trace=None):
    _SYNC.clear()
    _SYNC.update(s=0, e=0, trace=trace)
    main = _Inert(kind="s")
    main.name = "main"
    _SYNC["stack"] = [main]


def _log(line):
    if _SYNC["trace"] is not None:
        _SYNC["trace"].append(line)


class _Inert:
    """Stream / event stand-in with an identity: streams s1, s2, ... and events e1, e2, ... in creation order; the
    stream outside every torch.cuda.stream block is 'main'.  What they are asked to do goes to the trace."""

    def __init__(self, *a, kind="s", **k):
        _SYNC[kind] += 1
        self.name = "%s%d" % (kind, _SYNC[kind])

    def wait_stream(self, s):
        _log("%s.wait_stream(%s)" % (self.name, s.name))

    def wait_event(self, e):
        _log("%s.wait_event(%s)" % (self.name, e.name))

    def record(self, s=None):
        _log("%s.record(%s)" % (self.name, (s or _SYNC["stack"][-1]).name))

    def __enter__(self):
        _SYNC["stack"].append(self)
        return self

    def __exit__(self, *a):
        _SYNC["stack"].pop()
        return False


@pytest.fixture()
def dry(monkeypatch, oracle_ops):
    pkg = importlib.import_module("3dssd_b200")
    T, L = pkg.tf_ops, pkg.layers_util
    o = oracle_ops
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    n = lambda x: x.detach().cpu().numpy()

    def place(res, out, idx_offset, b, npoint, rounds=None):
        res = res.astype(np.int32) + int(idx_offset)
        if out is None:
            return t(res)
        buf, col = out
        j0, j1 = (0, npoint) if rounds is None else rounds
        buf[:, col + j0: col + j1] = t(res[:, j0:j1])
        return buf[:, col: col + npoint]

    def fps(npoint, inp, *, out=None, idx_offset=0, rounds=None, temp=None, cluster=0, packet_kernel=False, bucket_kernel=None):
        if rounds is not None and tuple(rounds) != (0, npoint):
            assert temp is not None and temp.shape == (inp.shape[0], 2 * inp.shape[1])      # fps_temp_elems of the fake
        return place(o.farthest_point_sample(npoint, n(inp)), out, idx_offset, inp.shape[0], npoint, rounds)

    def ffps(npoint, xyz, points=None, *, out=None, idx_offset=0, rounds=None, temp=None, **kw):
        assert set(kw) <= {"cluster"}                                # the real wrapper's CTA cap changes no index
        if rounds is not None and tuple(rounds) != (0, npoint):
            assert temp is not None and temp.shape == xyz.shape[:2]
        f = n(xyz) if points is None else np.concatenate([n(xyz), n(points)], -1)
        return place(o.farthest_point_sample_with_distance(npoint, o.calc_square_dist(f)), out, idx_offset, xyz.shape[0], npoint, rounds)

    def fpsd(npoint, dist, *, out=None, idx_offset=0, cluster=0):
        return place(o.farthest_point_sample_with_distance(npoint, n(dist)), out, idx_offset, dist.shape[0], npoint)

    def iota(b, npoint, device, *, out=None, start=0):
        return place(np.tile(np.arange(npoint, dtype=np.int32)[None], (b, 1)), out, start, b, npoint)

    def bq_multi(lows, highs, ks, xyz1, xyz2, dilated, grid=None, return_units=False):
        res = [(o.query_ball_point_dilated(lo, hi, k, n(xyz1), n(xyz2)) if dilated else o.query_ball_point(hi, k, n(xyz1), n(xyz2)))
               for lo, hi, k in zip(lows, highs, ks)]
        out = [t(r[0]) for r in res], [t(r[1]) for r in res]
        if not return_units:
            return out
        units = []                                                   # the unit lists of include/ssd3d.h, in REVERSED group order
        for r, k in zip(res, ks):                                    # (the order is unspecified: consumers may not rely on it)
            cnt = r[1].reshape(-1)
            lst = [(g << 4) | j for g in range(cnt.size - 1, -1, -1) for j in range((min(int(cnt[g]), k) + 7) // 8)]
            u = np.full(1 + cnt.size * ((k + 7) // 8), -1, np.int32)
            u[0] = len(lst); u[1:1 + len(lst)] = lst
            units.append(t(u))
        return out + (units,)

    def group_concat(xyz, points, new_xyz, idx, ldx=None):
        g = np.concatenate([o.group_point(n(points), n(idx)), o.group_point(n(xyz), n(idx)) - n(new_xyz)[:, :, None]], -1)
        return t(g.astype(np.float32))

    def linear_bn_relu(x, w, scale, shift, relu=True, pool=1, rowmask=None, cin=None):
        y = (n(x).astype(np.float64)[..., : w.shape[0]] @ n(w).astype(np.float64)) * n(scale) + n(shift)
        if relu:
            y = np.maximum(y, 0)
        if pool > 1:
            y = y.max(axis=-2) * (n(rowmask) > 0)[..., None]
        return t(y.astype(np.float32))

    # ---- tensor-core route: split bf16 operands are real (hi + lo), the contraction is float64 on the folded layers
    def split_rows(x, kp=None):
        c = x.shape[-1]
        kp = T.round16(c) if kp is None else int(kp)
        hi = torch.zeros(tuple(x.shape[:-1]) + (kp,), dtype=torch.bfloat16)
        lo = torch.zeros_like(hi)
        hi[..., :c] = x.to(torch.bfloat16)
        lo[..., :c] = (x - hi[..., :c].float()).to(torch.bfloat16)
        return hi, lo

    unsplit = lambda hi, lo: hi.float() + lo.float()

    def emit(y, pool, rowmask, want_f32, want_split, out_f32, out_split):
        if pool > 1:
            y = y.max(dim=-2).values * (rowmask > 0).unsqueeze(-1).to(y.dtype) if rowmask is not None else y.max(dim=-2).values
        nn = y.shape[-1]
        ret = None
        if out_f32 is not None:
            buf, off = out_f32
            buf[..., off: off + nn] = y
            ret = buf
        elif want_f32:
            ret = y
        sp = None
        if out_split is not None:
            hb, lb, off = out_split
            h, l = split_rows(y, nn)
            hb[..., off: off + nn] = h; lb[..., off: off + nn] = l
            sp = (hb, lb)
        elif want_split:
            sp = split_rows(y)
        return ret, sp

    def compact(x, units):
        """Dense grouped rows (b, m, ns, C) -> the compact layout of the *_units kernels: 8 rows per listed unit at the start
        of the buffer, NaN beyond (so that anything consuming rows it should not shows up)."""
        b, m, ns, c = x.shape
        u = n(units); nu = int(u[0])
        flat = x.reshape(b * m, ns, c)
        out = torch.full((b * m * ns, c), float("nan"), dtype=x.dtype)
        for i in range(nu):
            g, j = int(u[1 + i]) >> 4, int(u[1 + i]) & 15
            out[8 * i: 8 * i + 8] = flat[g, 8 * j: 8 * j + 8]
        return out.reshape(b, m, ns, c)

    def unit_pool_into(y, units, out_f32):
        """atomicMax of every unit's column maxima into its group's row of the caller's buffer (no fill of other groups)."""
        buf, off = out_f32
        u = n(units); nu = int(u[0])
        rows = y.reshape(-1, y.shape[-1])
        flat = buf.view(-1, buf.shape[-1])
        assert not torch.isnan(flat[:, off: off + rows.shape[1]]).any()
        for i in range(nu):
            g = int(u[1 + i]) >> 4
            mx = rows[8 * i: 8 * i + 8].max(dim=0).values
            assert not torch.isnan(mx).any() and (mx >= 0).all()
            flat[g, off: off + rows.shape[1]] = torch.maximum(flat[g, off: off + rows.shape[1]], mx)
        return buf, None

    def conv(x, f, relu=True):
        y = (x[..., : f.cin].double() @ f.w.double()) * f.scale.double() + f.shift.double()
        return (torch.relu(y) if relu else y).float()

    def linear_tc(a_hi, a_lo, f, relu=True, pool=1, rowmask=None, want_f32=True, want_split=False, out_f32=None, out_split=None,
                  units=None, unit_pool=False):
        assert a_hi.shape[-1] == f.kp and a_hi.dtype == torch.bfloat16
        y = conv(unsplit(a_hi, a_lo), f, relu)
        if unit_pool:
            assert units is not None and relu and pool == 1 and rowmask is None and out_split is None and not want_split
            return unit_pool_into(y, units, out_f32)
        return emit(y, pool, rowmask, want_f32, want_split, out_f32, out_split)

    def grouped(xyz, points, new_xyz, idx):
        return group_concat(xyz, points, new_xyz, idx)

    def hoisted_operand(xyz, z, zoff, wx, new_xyz, idx):
        n1 = wx.shape[1]
        d = t(o.group_point(n(xyz), n(idx)) - n(new_xyz)[:, :, None])
        zg = t(o.group_point(n(z[..., zoff: zoff + n1].contiguous()), n(idx)))
        return torch.relu(zg + d @ wx)

    def linear_tc_gather(xyz, points, new_xyz, idx, f, relu=True, pool=1, rowmask=None, want_f32=False, want_split=True, out_f32=None, out_split=None):
        return emit(conv(grouped(xyz, points, new_xyz, idx), f, relu), pool, rowmask, want_f32, want_split, out_f32, out_split)

    def linear_tc_hoisted(xyz, z, zoff, wx, new_xyz, idx, f, relu=True, pool=1, rowmask=None, want_f32=False, want_split=True, out_f32=None, out_split=None,
                          units=None, unit_pool=False):
        assert f.cin == wx.shape[1]
        x = hoisted_operand(xyz, z, zoff, wx, new_xyz, idx)
        if units is not None:
            y = conv(compact(x, units), f, relu)
            if unit_pool:
                return unit_pool_into(y, units, out_f32)
            return emit(y, 1, None, want_f32, want_split, out_f32, out_split)
        return emit(conv(x, f, relu), pool, rowmask, want_f32, want_split, out_f32, out_split)

    def fused(x, cnt, stack, out_f32, out_split, ns, units=None):
        if units is not None:
            assert out_split is None
            x = compact(x, units)
        for f in stack.convs:
            x = conv(x, f)
        if units is not None:
            return unit_pool_into(x, units, out_f32)[0]
        y, _ = emit(x, ns, cnt if cnt is not None else None, out_f32 is None and out_split is None, False, out_f32, out_split)
        return y

    def sa_mlp_fused(xyz, points, new_xyz, idx, cnt, stack, out_f32=None, out_split=None, units=None):
        assert points.shape[-1] + 3 == stack.cin
        return fused(grouped(xyz, points, new_xyz, idx), cnt, stack, out_f32, out_split, idx.shape[-1], units)

    def sa_mlp_fused_hoisted(xyz, z, zoff, wx, new_xyz, idx, cnt, stack, out_f32=None, out_split=None, units=None):
        assert wx.shape[1] == stack.cin
        return fused(hoisted_operand(xyz, z, zoff, wx, new_xyz, idx), cnt, stack, out_f32, out_split, idx.shape[-1], units)

    # ---- training mode: float64 batch-statistics BatchNorm and the masked row-group max
    def bn_train(x, gamma, beta, moving_mean=None, moving_var=None, decay=0.9, relu=True, eps=1e-3):
        flat = x.reshape(-1, x.shape[-1]).double()
        mean = flat.mean(0)
        var = ((flat - mean) ** 2).mean(0)
        inv = gamma.double() / torch.sqrt(var + eps)
        y = x.double() * inv + (beta.double() - mean * inv)
        if moving_mean is not None:                                  # in place, like updates_collections=None
            moving_mean.sub_(((moving_mean.double() - mean) * (1.0 - decay)).float())
            moving_var.sub_(((moving_var.double() - var) * (1.0 - decay)).float())
        return (torch.relu(y) if relu else y).float(), inv.float(), (beta.double() - mean * inv).float(), mean.float(), var.float()

    def rowgroup_max(y, pool, rowmask=None):
        out = y.max(dim=-2).values
        return out * (rowmask > 0).unsqueeze(-1).to(out.dtype) if rowmask is not None else out

    # ---- FP layers, decoders, NMS and PointRCNN's region pool
    def fp_interp_split(xyz1, xyz2, points2, points1=None, kp=None):
        d = ((xyz1.double()[:, :, None] - xyz2.double()[:, None]) ** 2).sum(-1)
        dist, idx = d.topk(min(3, xyz2.shape[1]), dim=-1, largest=False)
        inv = 1.0 / dist.clamp_min(1e-10)
        w = inv / inv.sum(-1, keepdim=True)
        x = (points2.double()[torch.arange(points2.shape[0])[:, None, None], idx] * w[..., None]).sum(2)
        if points1 is not None:
            x = torch.cat([x, points1.double()], -1)
        return split_rows(x.float(), kp)

    def decode_dist_anchor_free(center_xyz, pred_reg, pred_cls, angle_bins=12):
        reg, cls = pred_reg.numpy(), pred_cls.numpy()
        off, acls, ares = reg[..., :6], reg[..., 6:6 + angle_bins], reg[..., 6 + angle_bins:]
        bins = np.argmax(acls, -1)
        res = np.take_along_axis(ares, bins[..., None], -1)[..., 0]
        ang = ((bins.astype(np.float32) + res) * np.float32(2 * np.pi / angle_bins)).astype(np.float32)
        ctr = center_xyz.numpy() + off[..., :3]
        ctr[..., 1] += off[..., 4]
        boxes = np.concatenate([ctr, np.maximum(off[..., 3:6] * np.float32(2), np.float32(0.1)), ang[..., None]], -1).astype(np.float32)
        return torch.from_numpy(boxes), torch.from_numpy((1 / (1 + np.exp(-cls[..., 0].astype(np.float64)))).astype(np.float32))

    def decode_bin_anchor(center_xyz, pred_reg, pred_cls, anchor_lhw, half_bin_search_range=3.0, bin_num=12, angle_bins=12):
        b, n, _ = center_xyz.shape
        boxes = torch.cat([center_xyz, torch.tensor(anchor_lhw, dtype=torch.float32).expand(b, n, 3),
                           pred_reg[..., :1]], -1)
        return boxes.contiguous(), torch.sigmoid(pred_cls[..., 0]).contiguous()

    def decode_bin_anchor_rows(anchors, pred_reg, pred_cls, pool_cnt=None, half_bin_search_range=1.5, bin_num=6, angle_bins=12):
        score = torch.softmax(pred_cls[..., :2].double(), -1)[..., 1].float()
        if pool_cnt is not None:
            score = score * (pool_cnt > 0).float()
        return anchors[..., :7].contiguous(), score

    def bev_nms(boxes, scores, iou_threshold, max_output, cls_id=0, out=None):
        blk, cnt = oracle_ops.bev_nms(n(boxes), n(scores), iou_threshold, max_output, cls_id)
        if out is None:
            return t(blk), t(cnt)
        out[0].copy_(t(blk)); out[1].copy_(t(cnt))
        return out

    def bev_nms_counted(boxes, scores, n_valid, iou_threshold, max_output, cls_id=0, out=None):
        m = (torch.arange(scores.shape[1])[None] < n_valid[:, None].long()).float()
        return bev_nms(boxes, scores * m - (1 - m), iou_threshold, max_output, cls_id, out)

    def region_pool(xyz, features, point_score, proposals, count, info_conv, nsample=512, context=1.0, mask_thresh=0.5):
        """Each proposal pools the scene's first nsample points (cyclically), canonical = relative to its centre."""
        b, nn = xyz.shape[:2]
        p = proposals.shape[1]
        idx = (torch.arange(nsample) % nn).to(torch.int32).expand(b, p, nsample).contiguous()
        rows = torch.arange(nsample) % nn
        cxyz = xyz[:, None, rows] - proposals[:, :, None, :3]
        mask = (point_score[:, None, rows] >= mask_thresh).float().expand(b, p, nsample)
        info = torch.cat([cxyz, mask[..., None], cxyz.norm(dim=-1, keepdim=True)], -1)
        feat = torch.cat([conv(info, info_conv), features[:, None, rows].expand(b, p, nsample, -1)], -1)
        cnt = torch.full((b, p), nsample, dtype=torch.int32)
        if count is not None:
            cnt = cnt * (torch.arange(p)[None] < count[:, None].long()).to(torch.int32)
        return (cxyz.reshape(b * p, nsample, 3).contiguous(), feat.reshape(b * p, nsample, -1).contiguous(), idx, cnt)

    fakes = dict(
        fill_zero=lambda x: x.zero_(),
        split_rows=split_rows, linear_tc=linear_tc, linear_tc_gather=linear_tc_gather, linear_tc_hoisted=linear_tc_hoisted,
        sa_mlp_fused=sa_mlp_fused, sa_mlp_fused_hoisted=sa_mlp_fused_hoisted,
        hoist_expand_split=lambda xyz, z, zoff, wx, new_xyz, idx, units=None: split_rows(
            hoisted_operand(xyz, z, zoff, wx, new_xyz, idx) if units is None else compact(hoisted_operand(xyz, z, zoff, wx, new_xyz, idx), units)),
        group_concat_split=lambda xyz, points, new_xyz, idx, kp=None: split_rows(grouped(xyz, points, new_xyz, idx), kp),
        split_points=lambda p: (p[..., :3].contiguous(), p[..., 3:].contiguous()),
        farthest_point_sample=fps, farthest_point_sample_features=ffps, farthest_point_sample_with_distance=fpsd,
        calc_square_dist=lambda a: t(o.calc_square_dist(n(a))), concat_cols=lambda a, b: torch.cat([a, b], -1).contiguous(),
        iota_idx=iota, gather_point=lambda inp, idx: t(o.gather_point(n(inp), n(idx))),
        query_ball_point_multi=bq_multi, group_concat=group_concat, linear_bn_relu=linear_bn_relu,
        concat_rows=lambda parts: torch.cat(list(parts), dim=1).contiguous(),
        fps_supports_rounds=lambda nn, c=3: True, ffps_supported=lambda nn, c: c <= 68,
        fps_temp_elems=lambda nn, c=3, npoint=0, **kw: 2 * nn,
        vote_translate=lambda xyz, off, rng: xyz + torch.minimum(torch.maximum(off[..., :3], torch.tensor(rng)), -torch.tensor(rng)),
        bn_train=bn_train, rowgroup_max=rowgroup_max,
        fp_interp_split=fp_interp_split, decode_dist_anchor_free=decode_dist_anchor_free, decode_bin_anchor=decode_bin_anchor,
        decode_bin_anchor_rows=decode_bin_anchor_rows, bev_nms=bev_nms, bev_nms_counted=bev_nms_counted, region_pool=region_pool,
    )
    for k, v in fakes.items():
        monkeypatch.setattr(T, k, v)
    _reset_sync()
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: _SYNC["stack"][-1])
    monkeypatch.setattr(torch.cuda, "Stream", lambda *a, **k: _Inert(kind="s"))
    monkeypatch.setattr(torch.cuda, "Event", lambda *a, **k: _Inert(kind="e"))
    monkeypatch.setattr(torch.cuda, "stream", lambda s: s)
    monkeypatch.setattr(L, "_SIDE_STREAMS", {})
    return pkg


def _scaled(pkg, div):
    arch = copy.deepcopy(pkg.config.ARCH_3DSSD)
    for spec in arch:
        spec[6] = [r if r == -1 else max(1, r // div) for r in spec[6]]
        spec[8] = [p if p in (-1, 0) else max(1, p // div) for p in spec[8]]
    return arch


_ROUTES = [("fp32", True, 2, True), ("tc", True, 2, True), ("tc", True, 1, True), ("tc", True, 0, True), ("tc", False, 0, False),
           ("tc", True, 2, False)]
_LATENCY = [(False, None), (True, 2), (True, [0.5, 0.25, 0.25])]


@pytest.mark.parametrize("mlp_mode,gather,hoist,fuse", _ROUTES)
@pytest.mark.parametrize("latency,parts", _LATENCY)
def test_backbone_orchestration_dry_run_matches_oracle_layers(dry, oracle_ops, latency, parts, mlp_mode, gather, hoist, fuse):
    kw = dict(fps_parts=parts) if parts is not None else {}
    _backbone_dry_run(dry, _scaled(dry, 16), mlp_mode=mlp_mode, latency_mode=latency, gather_in_kernel=gather,
                      hoist_first=hoist, fuse_scale=fuse, **kw)     # 1024 -> 256 -> 64+.. centres


# two SA layers on the 1024 input points whose F-FPS samples 256 points on 4 channels: in latency mode the matrix-free
# kernel hands over its two halves separately, next to a D-FPS half (fusion sampling) or a D-FPS segment on a side stream
_HALVES = [[[0], [0], [0.4, 0.8], [16, 32], [[16, 16, 32], [16, 32, 48]], True, [-1], ['FS'], [256],
            -1, False, 'SA_Layer', 'fs', True, -1, 64],
           [[0], [0], [0.4, 0.8], [16, 32], [[16, 16, 32], [16, 32, 48]], True, [512, -1], ['F-FPS', 'D-FPS'], [256, 256],
            -1, False, 'SA_Layer', 'fd', True, -1, 64]]


def _backbone_dry_run(pkg, arch, **net_kw):
    """SABackbone(arch, **net_kw).forward on two 1024-point scenes against the oracle's layers: every layer's fps_idx,
    ball-query indices, xyz and features."""
    from oracle import layers as olayers
    synth = importlib.import_module("3dssd_b200.synth")
    params = pkg.params.init_params(arch, 1, seed=4, random_bias=True)
    pts = synth.kitti_like(2, 1024, seed=40)
    pts[..., 0] *= 0.2; pts[..., 2] *= 0.2
    net = pkg.SABackbone(arch, params, in_channels=1, device="cpu", **net_kw)
    got = net.forward(torch.from_numpy(pts), return_debug=True)
    exp = olayers.backbone_forward(arch, pts, params, ffps_mode="matrix", return_debug=True)
    for li in range(1, len(arch) + 1):
        if exp[2][li] is not None:
            np.testing.assert_array_equal(got[2][li].numpy(), exp[2][li], err_msg="fps_idx of layer %d" % li)
        for a, b in zip(got[3][li - 1].get("idx", []), exp[3][li - 1].get("idx", [])):
            np.testing.assert_array_equal(a.numpy(), b)
        if exp[0][li] is not None:
            assert np.abs(got[0][li].numpy() - exp[0][li]).max() < 1e-5
        assert np.abs(got[1][li].numpy() - exp[1][li]).max() <= 1e-4 * max(1.0, np.abs(exp[1][li]).max()), "features of layer %d" % li


def test_head_orchestration_dry_run_writes_into_gather_buffers(dry, oracle_ops):
    """DetectionHead + DetectionGather plumbing on the CPU: conv chain -> one-kernel decode -> NMS writing straight into
    the send buffer of the (single-rank) gather, against the oracle's head."""
    pkg = dry
    from oracle import head as ohead
    rng = np.random.default_rng(3)
    xyz = rng.uniform(-10, 10, (3, 64, 3)).astype(np.float32)
    feat = np.maximum(rng.standard_normal((3, 64, 512)), 0).astype(np.float32)
    prm = pkg.params.init_head_params(512, seed=5)
    head = pkg.DetectionHead(params=prm, device="cpu")
    g = pkg.dist.DetectionGather(3, "cpu")
    blk, cnt = head.forward([None] * 6 + [torch.from_numpy(xyz)], [None] * 6 + [torch.from_numpy(feat)], out=g.out())
    g.gather()
    rb, rc = g.result()
    eboxes, escore, _ = ohead.head_forward(xyz, feat, prm)
    eb, ec = ohead.bev_nms(eboxes, escore, 0.1, 100)
    assert rb.data_ptr() == blk.data_ptr() and torch.equal(rc, cnt)
    np.testing.assert_array_equal(rc.numpy(), ec)
    assert np.abs(rb.numpy() - eb).max() < 2e-3


@pytest.mark.parametrize("decay", [None, 0.5])
def test_training_mode_orchestration_dry_run_matches_oracle(dry, oracle_ops, decay):
    """is_training=True through pointnet_sa_module_msg on the CPU (SURVEY 8f row f3): the literal conv -> batch-norm -> relu
    schedule with ssd3d_bn_train / ssd3d_rowgroup_max replaced by a few float64 lines (the dry fixture), against the
    oracle's restatement of tf_util.py:424-444; the moving statistics are updated in place, commit_bn() writes them back
    and inference then folds the NEW statistics."""
    pkg = dry
    from oracle import layers as olayers
    rng = np.random.default_rng(11)
    synth = importlib.import_module("3dssd_b200.synth")
    pts = synth.kitti_like(2, 512, seed=61)
    pts[..., 0] *= 0.1; pts[..., 2] *= 0.1
    xyz, feats = pts[..., :3].copy(), rng.standard_normal((2, 512, 16)).astype(np.float32)
    arch = [[[0], [0], [0.4, 0.8], [16, 32], [[16, 16, 32], [16, 32, 48]], True, [-1], ['D-FPS'], [64],
             -1, False, 'SA_Layer', 'trn', True, -1, 64]]
    params = dict(pkg.params.init_params(arch, 16, seed=8, random_bias=True))
    args = (arch[0][2], arch[0][3], arch[0][4], True, decay, True, [-1], ['D-FPS'], [64], None, False, 'trn', True)
    params_ref = {k: np.array(v, copy=True) for k, v in params.items()}            # on the CPU torch.from_numpy ALIASES the dict's
    pp = pkg.params.prepare(params, "cpu")                                        # arrays: the oracle gets its own copy
    got = pkg.pointnet_sa_module_msg(torch.from_numpy(xyz), torch.from_numpy(feats), *args, aggregation_channel=64, params=pp,
                                     return_debug=True, fps_parts=2)              # fps_parts is ignored when training
    upd = {}
    exp = olayers.pointnet_sa_module_msg(xyz, feats, *args, aggregation_channel=64, params=params_ref, return_debug=True, bn_updates=upd)
    np.testing.assert_array_equal(got[2].numpy(), exp[2])
    for a, b in zip(got[3]["idx"], exp[3]["idx"]):
        np.testing.assert_array_equal(a.numpy(), b)
    assert np.abs(got[1].numpy() - exp[1]).max() <= 1e-4 * np.abs(exp[1]).max()
    assert set(upd) == {"trn/conv%d_%d" % (i, j) for i in range(2) for j in range(3)} | {"trn/ensemble"}
    for scope, u in upd.items():
        st = pp.bn_state(scope)
        for k in ("moving_mean", "moving_variance"):
            assert np.abs(st[k].numpy() - u[k]).max() <= 1e-4 * max(1e-3, np.abs(u[k]).max()), (scope, k)
    pp.commit_bn()
    assert not np.array_equal(params["trn/conv0_0/bn/moving_mean"], params_ref["trn/conv0_0/bn/moving_mean"])
    for scope, u in upd.items():                                                  # the oracle's view of "after one training step"
        for k in ("moving_mean", "moving_variance"):
            params_ref[scope + "/bn/" + k] = u[k]
    args_inf = args[:3] + (False,) + args[4:]
    got_i = pkg.pointnet_sa_module_msg(torch.from_numpy(xyz), torch.from_numpy(feats), *args_inf, aggregation_channel=64, params=pp)
    exp_i = olayers.pointnet_sa_module_msg(xyz, feats, *args_inf, aggregation_channel=64, params=params_ref)
    assert np.abs(got_i[1].numpy() - exp_i[1]).max() <= 1e-4 * np.abs(exp_i[1]).max()


def _scaled_pointrcnn(pkg, mp):
    """PointRCNN's tables with smaller sample counts and 64 points per proposal, so its dry run is small; mp: a
    monkeypatch context that restores them."""
    cfg = pkg.config
    for name, div in (("ARCH_POINTRCNN_RPN", 16), ("ARCH_POINTRCNN_RCNN", 8)):
        arch = copy.deepcopy(getattr(cfg, name))
        for spec in arch:
            spec[8] = [p if p in (-1, 0) else max(1, p // div) for p in spec[8]]
        mp.setattr(cfg, name, arch)
    pool = list(cfg.POINTS_POOLER_POINTRCNN)
    pool[3] = 64
    mp.setattr(cfg, "POINTS_POOLER_POINTRCNN", pool)


def _rpn_dry_run(pkg, mp, latency):
    """PointRCNN's first stage: the SA and FP layers of its table and its Bin-Anchor DetectionHead."""
    _scaled_pointrcnn(pkg, mp)
    cfg = pkg.config
    synth = importlib.import_module("3dssd_b200.synth")
    params = pkg.rcnn.init_pointrcnn_params(seed=3)
    head = pkg.DetectionHead(cfg.HEAD_POINTRCNN_RPN, params, device="cpu", stage=cfg.STAGE_POINTRCNN_RPN_TEST)
    net = pkg.SABackbone(cfg.ARCH_POINTRCNN_RPN, params, in_channels=1, device="cpu", head=head, aggregation=False,
                         latency_mode=latency)
    xyz_l, feat_l, _ = net.forward(torch.from_numpy(synth.kitti_like(2, 1024, seed=42)))
    blk, cnt = net.detections(xyz_l, feat_l)
    assert blk.shape == (2, 100, 9) and feat_l[-1].shape == (2, 1024, 128)


def _pointrcnn_dry_run(pkg, mp):
    """PointRCNN.forward: RPN, region pool, stage-2 layers, RCNN head, row decode and the counted NMS."""
    _scaled_pointrcnn(pkg, mp)
    synth = importlib.import_module("3dssd_b200.synth")
    net = pkg.PointRCNN(device="cpu", seed=3)
    block, count = net.forward(torch.from_numpy(synth.kitti_like(2, 1024, seed=43)))
    assert block.shape == (2, 100, 9) and count.shape == (2,)


def _train_forward_dry_run(pkg):
    """backbone.train_forward over the (scaled) 3DSSD table with TrainableParams."""
    synth = importlib.import_module("3dssd_b200.synth")
    arch = _scaled(pkg, 16)
    d = dict(pkg.params.init_params(arch, 1, seed=4, random_bias=True))
    d.update(pkg.params.init_head_params(pkg.config.layer_channels(arch, 1)[-1], seed=5))
    pts = torch.from_numpy(synth.kitti_like(2, 1024, seed=44))
    o = pkg.train_forward(arch, pkg.params.TrainableParams(d, "cpu"), pts[..., :3].contiguous(), pts[..., 3:].contiguous(),
                          bn_decay=0.5)
    assert o.head[0].shape == o.base_xyz.shape[:2] + (1,) and len(o.vote_offsets) == 1


TRACE_GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "launch_trace.json")


def _describe(v):
    if isinstance(v, torch.Tensor):
        return "%s%s" % (str(v.dtype).replace("torch.", ""), list(v.shape))
    if isinstance(v, (list, tuple)):
        return "(%s)" % ",".join(_describe(x) for x in v)
    if isinstance(v, dict):
        return "{%s}" % ",".join("%s:%s" % (k, _describe(x)) for k, x in sorted(v.items()))
    if hasattr(v, "w_blob"):                                      # params.FusedStack
        return "stack(%d->%s)" % (v.cin, v.nout)
    if hasattr(v, "b_hi"):                                        # params.FoldedConv
        return "conv(%d->%d)" % (v.cin, v.cout)
    if v is None or isinstance(v, (bool, int, float, str)):
        return repr(v)
    return type(v).__name__


def _traced(name, fn):
    sig = inspect.signature(fn)

    def call(*a, **k):
        b = sig.bind(*a, **k)
        b.apply_defaults()
        # a **kwargs parameter shows only the keywords actually passed
        args = [(p, v) for p, v in b.arguments.items() if sig.parameters[p].kind != inspect.Parameter.VAR_KEYWORD or v]
        _log("%s@%s %s" % (name, _SYNC["stack"][-1].name, " ".join("%s=%s" % (p, _describe(v)) for p, v in args)))
        return fn(*a, **k)
    return call


def test_launch_trace_matches_recording(dry, oracle_ops, monkeypatch):
    """Which kernel serves each scale, where its output goes and on which stream, pinned call by call.  A route that
    falls back (a FusedStack that no longer fits, a scale that loses its unit list) gives the same numbers but a
    different trace.  Every tf_ops stand-in of the dry fixture logs its name, stream, tensor shapes and scalar and
    keyword arguments; the streams and events log their waits and records.  The dry runs are the 18 route / latency
    combinations of the backbone test, the training-mode layer, the 3DSSD head, PointRCNN's RPN in both modes, the whole
    PointRCNN forward, backbone.train_forward, the throughput backbone with fps_cluster=-4, with the packet and with the
    bucket D-FPS kernel, and latency mode on F-FPS segments of 256 samples.  SSD3D_RECORD_TRACE=<file> writes the traces to
    <file> instead of comparing them with tests/golden/launch_trace.json."""
    T = dry.tf_ops
    for k, v in list(vars(T).items()):
        if inspect.isfunction(v) and v.__module__ == __name__:
            monkeypatch.setattr(T, k, _traced(k, v))
    runs = {}
    for latency, parts in _LATENCY:
        for route in _ROUTES:
            runs["backbone-%s-gather%d-hoist%d-fuse%d-latency%d-parts%s" % (route + (latency, parts))] = \
                lambda r=route, lt=latency, p=parts: test_backbone_orchestration_dry_run_matches_oracle_layers(dry, oracle_ops, lt, p, *r)
    for decay in (None, 0.5):
        runs["training-decay%s" % decay] = lambda d=decay: test_training_mode_orchestration_dry_run_matches_oracle(dry, oracle_ops, d)
    runs["head-3dssd"] = lambda: test_head_orchestration_dry_run_writes_into_gather_buffers(dry, oracle_ops)

    def scaled(run, *a):
        with monkeypatch.context() as mp:
            run(dry, mp, *a)
    for latency in (False, True):
        runs["rpn-latency%d" % latency] = lambda lt=latency: scaled(_rpn_dry_run, lt)
    runs["pointrcnn-forward"] = lambda: scaled(_pointrcnn_dry_run)
    runs["train-forward"] = lambda: _train_forward_dry_run(dry)
    # the FPS options of bench.py's throughput step (fps_cluster=-4, automatic layer-1 kernel), the two other lone D-FPS
    # kernels, and the F-FPS halves of latency mode
    runs["backbone-throughput-cluster-4"] = lambda: _backbone_dry_run(dry, _scaled(dry, 16), fps_cluster=-4)
    runs["backbone-fps-packet"] = lambda: _backbone_dry_run(dry, _scaled(dry, 16), fps_packet=True)
    runs["backbone-fps-bucket"] = lambda: _backbone_dry_run(dry, _scaled(dry, 16), fps_bucket=True)
    runs["backbone-ffps-halves-latency1"] = lambda: _backbone_dry_run(dry, _HALVES, latency_mode=True)
    got = {}
    for key, run in runs.items():
        monkeypatch.setattr(dry.layers_util, "_SIDE_STREAMS", {})
        _reset_sync(trace=[])
        run()
        got[key] = _SYNC["trace"]
        _reset_sync()
    record = os.environ.get("SSD3D_RECORD_TRACE")
    if record:
        with open(record, "w") as fh:
            json.dump(got, fh, indent=0)
            fh.write("\n")
        return
    with open(TRACE_GOLDEN) as fh:
        exp = json.load(fh)
    assert sorted(got) == sorted(exp)
    for key in exp:
        g, e = got[key], exp[key]
        first = next((i for i in range(min(len(g), len(e))) if g[i] != e[i]), min(len(g), len(e)))
        assert g == e, "%s: call %d differs\n got: %s\n exp: %s" % (key, first, g[first] if first < len(g) else "<end>",
                                                                   e[first] if first < len(e) else "<end>")
