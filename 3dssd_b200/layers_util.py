"""SA / FP / vote layers with the reference's signatures, on the H100 operators.

Mirrors /root/reference/lib/utils/layers_util.py: vote_layer :12-24, pointnet_sa_module :27-55,
pointnet_sa_module_msg :59-189, pointnet_fp_module :192-225 -- same positional arguments and return values,
torch CUDA tensors instead of TF tensors.  What TF resolved through variable scopes is passed explicitly as
`params` (a dict keyed by the reference's variable names, or a params.PreparedParams).  is_training=True runs the
convs with batch-statistics BatchNorm and updates the moving statistics in place (tf_util.py:424-444); the fused
inference kernels fold BN and therefore serve is_training=False only.  With params a params.TrainableParams,
is_training=True runs the same schedule through the differentiable operators of tf_ops (conv_train, group_max_train,
group_concat_train, vote_translate_train): loss.backward() then reaches every weight, bias, gamma and beta.
"""
from functools import partial
from types import SimpleNamespace

import torch

from . import config as _cfg
from . import tf_ops
from .params import TrainableParams, prepare


def _conv(pp, scope, x, bn=True, relu=True, pool=1, rowmask=None):
    f = pp.conv(scope, bn)
    return tf_ops.linear_bn_relu(x, f.w, f.scale, f.shift, relu=relu, pool=pool, rowmask=rowmask, cin=f.cin)


def _trainable(params, is_training):
    return bool(is_training) and isinstance(params, TrainableParams)


def _conv_train(pp, scope, x, bn, bn_decay, relu=True, debug=None):
    """conv (+bias) -> training-mode BatchNorm -> ReLU, tf_util.conv2d / conv1d with is_training=True
    (/root/reference/lib/utils/tf_util.py:51-124, :127-201, :424-444): tf_ops.linear_bn_train with the cached BN-less
    fold; the batch statistics, the normalisation and the in-place update of the moving statistics are one ssd3d_bn_train
    call.  A TrainableParams takes the differentiable twin (tf_ops.conv_train); debug (a list) then receives the conv's
    (pre-BN, post-activation) tensors."""
    if isinstance(pp, TrainableParams):
        return pp.conv_train(scope, x, bn, bn_decay, relu, debug)
    st = pp.bn_state(scope) if bn else {}
    return tf_ops.linear_bn_train(x, pp.conv(scope, False), st.get("gamma"), st.get("beta"), st.get("moving_mean"),
                                  st.get("moving_variance"), bn=bn, relu=relu,
                                  decay=0.9 if bn_decay is None else float(bn_decay))[1][0]


def _ball_query(xyz, new_xyz, radius_list, nsample_list, dilated_group, want_units=False, unit_rows=None):
    """The ball queries of all scales (:137-145) -> (idx_list, cnt_list, units_list); units_list holds the unit lists of
    query_ball_point_multi(return_units=True) when want_units (up to 4 scales), else None per scale; unit_rows: their
    rows per unit, one per scale (None: 8)."""
    nscale = len(radius_list)
    min_r = [0.0 if (i == 0 or not dilated_group) else radius_list[i - 1] for i in range(nscale)]   # :137-141
    if nscale <= 4:   # one pass over the candidates for all shells
        with tf_ops.unit_rows(unit_rows if want_units else None):
            res = tf_ops.query_ball_point_multi(min_r, radius_list, nsample_list, xyz, new_xyz, dilated_group,
                                                return_units=want_units)
        return res[0], res[1], res[2] if want_units else [None] * nscale
    idx_list, cnt_list = [], []
    for i in range(nscale):
        a, c = (tf_ops.query_ball_point_dilated(min_r[i], radius_list[i], nsample_list[i], xyz, new_xyz) if dilated_group
                else tf_ops.query_ball_point(radius_list[i], nsample_list[i], xyz, new_xyz))
        idx_list.append(a); cnt_list.append(c)
    return idx_list, cnt_list, [None] * nscale


def _group_and_mlp_train(pp, scope, xyz, points, new_xyz, radius_list, nsample_list, mlp_list, bn, bn_decay, dilated_group,
                         use_agg):
    """Training-mode twin of _group_and_mlp: the literal op sequence of layers_util.py:137-185 (grouped tensor
    materialised once, conv -> batch-norm -> relu per layer, reduce_max, mask, concat, aggregation).
    Returns (new_points, idx_list, cnt_list, convs): convs lists every conv's tensors with a TrainableParams, else None."""
    idx_list, cnt_list, _ = _ball_query(xyz, new_xyz, radius_list, nsample_list, dilated_group)
    trainable = isinstance(pp, TrainableParams)
    group_concat = tf_ops.group_concat_train if trainable else tf_ops.group_concat
    group_max = tf_ops.group_max_train if trainable else tf_ops.rowgroup_max
    convs = [] if trainable else None
    outs = []
    for i in range(len(radius_list)):
        g = group_concat(xyz, points, new_xyz, idx_list[i])                                         # :160-165
        for j in range(len(mlp_list[i])):
            g = _conv_train(pp, "%s/conv%d_%d" % (scope, i, j), g, bn, bn_decay, debug=convs)       # :167-176
        outs.append(group_max(g, nsample_list[i], cnt_list[i]))                                     # :178-180
    new_points = outs[0] if len(outs) == 1 else torch.cat(outs, dim=-1)
    if use_agg:
        new_points = _conv_train(pp, scope + "/ensemble", new_points, bn, bn_decay, debug=convs)    # :183-185
    return new_points, idx_list, cnt_list, convs


_SIDE_STREAMS = {}


def _side_stream(device, role):
    """The side stream of `role` on `device` ('hoist', ('fork', i) or ('part', i)), created on first use."""
    key = (str(device), role)
    if key not in _SIDE_STREAMS:
        _SIDE_STREAMS[key] = torch.cuda.Stream(device=device)
    return _SIDE_STREAMS[key]


def _ffps_direct(n, c):
    """Whether F-FPS over n points of c concatenated channels takes the matrix-free kernel.  The 132-channel variant
    walks a 131-long dependent fma chain per round: at layer-3 sizes (512 points) the small matrix is faster, so the
    kernel serves where the matrix is the expensive part (c <= 68, layer 2)."""
    return c <= 68 and tf_ops.ffps_supported(n, c)


def ffps_indices(npoint, xyz, points, mode, out=None, idx_offset=0, cluster=None):
    """F-FPS on concat[xyz, points] (layers_util.py:94-96, :102-104).
    mode 'direct': one kernel, no [B,N,N] tensor, the SAME indices as 'matrix' (each round evaluates the picked point's
                   matrix row on chip with calc_square_dist's arithmetic); falls back to 'matrix' for uncovered shapes;
    mode 'matrix': calc_square_dist + farthest_point_sample_with_distance, the reference's route;
    mode 'fused' : matrix-free -- the generic-c FPS kernel evaluates the feature distance on the fly (no
                   [B,N,N] tensor); identical to the reference's own farthest_point_sample on the features.
    xyz / points may be [:, a:b] slices of dense tensors (read in place); out=(buffer, col) / idx_offset as in
    tf_ops.farthest_point_sample; cluster: the 'direct' kernel's CTA cap (tf_ops.farthest_point_sample_features)."""
    if mode == "direct":
        if _ffps_direct(xyz.shape[1], xyz.shape[2] + points.shape[2]):
            kw = {} if cluster is None else {"cluster": cluster}
            return tf_ops.farthest_point_sample_features(npoint, xyz, points, out=out, idx_offset=idx_offset, **kw)
        mode = "matrix"
    feats = tf_ops.concat_cols(xyz, points) if points.shape[2] else xyz
    if mode == "matrix":
        return tf_ops.farthest_point_sample_with_distance(npoint, tf_ops.calc_square_dist(feats), out=out,
                                                          idx_offset=idx_offset)
    if mode == "fused":
        return tf_ops.farthest_point_sample(npoint, feats, out=out, idx_offset=idx_offset)
    raise ValueError("ffps_mode must be 'direct', 'matrix' or 'fused'")


def _part_bounds(npoint, fps_parts):
    """Round ranges of a D-FPS consumed in parts: fps_parts = number of equal parts or a list of fractions."""
    if isinstance(fps_parts, int):
        fr = [1.0 / fps_parts] * fps_parts
    else:
        fr = [float(f) for f in fps_parts]
    cuts, acc = [0], 0.0
    for f in fr[:-1]:
        acc += f
        c = int(round(acc / sum(fr) * npoint / 128.0)) * 128          # parts are whole 128-row tiles of every scale
        cuts.append(min(max(c, cuts[-1]), npoint))
    cuts.append(npoint)
    return [(cuts[i], cuts[i + 1]) for i in range(len(cuts) - 1) if cuts[i + 1] > cuts[i]]


COMPACT_GROUPS = True      # fused SA scales convolve only the 8-row units that hold distinct neighbours (tf_ops.sa_mlp_fused `units`)
UNIT_ROWS = 4              # rows per unit of those lists where nsample <= 64 (DESIGN.md 3.4); 8 for wider groups
HOIST_EXPAND_MIN_K = 256   # hoisted second convs at least this wide materialise their operand (tf_ops.hoist_expand_split)


def _route_plan(pp, scope, nsample_list, mlp_list, bn, c_feat, use_agg, mlp_mode, fuse_scale, gather_in_kernel, hoist_first):
    """Which kernels serve each scale of one SA layer at inference, decided from parameter shapes and options alone:
      tc         the tensor-core route (nsample among the pooling widths of its epilogue, scale widths multiples of 8
                 for 16-byte aligned column slices of the concat buffers), else the fp32 route;
      hoisted    the scales whose first conv is hoisted (hoist_first: 0 off, 1 layer-by-layer scales only, 2 all): the
                 feature part of those convs runs once per POINT into one table z (_hoist_table);
      scales[i]  route: 'fused' (tf_ops.sa_mlp_fused) or 'fused_hoisted' (sa_mlp_fused_hoisted, the remaining convs in
                 `stack`) run the whole scale in one kernel; layer by layer, the first operand is 'gather'ed in the
                 kernel (linear_tc_gather), materialised by group_concat_split ('split'), built from z by the producer
                 warps of linear_tc_hoisted ('hoisted') or materialised from z by hoist_expand_split ('expand', wide
                 second convs).  zoff: its columns in z.  units: only the units of its unit list are convolved,
                 and pooled into the zero-filled concat buffer; unit_rows: rows per unit of that list (UNIT_ROWS
                 for nsample <= 64, else 8);
      compact    some scale uses its unit list;
      split_out  the aggregation conv's split operand is written by the scales' epilogues (else split once afterwards)."""
    tc = mlp_mode == "tc" and all(k in tf_ops.TC_POOL_WIDTHS for k in nsample_list) and all(m[-1] % 8 == 0 for m in mlp_list)
    scopes = [["%s/conv%d_%d" % (scope, i, j) for j in range(len(m))] for i, m in enumerate(mlp_list)]
    plan = SimpleNamespace(tc=tc, bn=bn, scopes=scopes, agg=scope + "/ensemble" if use_agg else None, hoisted=[], scales=[],
                           compact=False, split_out=False)
    if not tc:
        return plan
    stacks = [pp.fused_stack(names, bn, c_feat + 3) if fuse_scale else None for names in scopes]
    # an xyz-only cloud (c_feat == 0) has no feature part to hoist: its first conv runs in the grouped domain
    if gather_in_kernel and hoist_first and c_feat > 0:
        plan.hoisted = [i for i, m in enumerate(mlp_list) if len(m) >= 2 and (int(hoist_first) >= 2 or stacks[i] is None)]
    n1 = {i: pp.conv(scopes[i][0], bn).cout for i in plan.hoisted}
    ldz = sum(n1.values())
    for i, names in enumerate(scopes):
        sc = SimpleNamespace(stack=stacks[i], zoff=None, units=COMPACT_GROUPS and len(mlp_list) <= 4,
                             unit_rows=UNIT_ROWS if nsample_list[i] <= 16 * UNIT_ROWS and nsample_list[i] % UNIT_ROWS == 0 else 8)
        if i in plan.hoisted:
            sc.zoff = sum(n1[h] for h in plan.hoisted[:plan.hoisted.index(i)])
        if sc.stack is not None:
            hstack = pp.fused_stack(names[1:], bn, n1[i]) if i in n1 else None
            sc.route, sc.stack = ("fused_hoisted", hstack) if hstack is not None else ("fused", sc.stack)
        elif i in n1:
            wide = pp.conv(names[1], bn).kp >= HOIST_EXPAND_MIN_K and sc.zoff % 4 == 0 and ldz % 4 == 0
            sc.route = "expand" if wide else "hoisted"
        else:
            sc.route, sc.units = "gather" if gather_in_kernel else "split", False
        plan.scales.append(sc)
    plan.compact = any(sc.units for sc in plan.scales)
    plan.split_out = use_agg and not plan.compact
    return plan


def _hoist_table(pp, plan, points):
    """The table of the hoisted first convs (plan.hoisted): z = (features . [Wf_1 | Wf_2 | ...]) * s + t once per point,
    and the xyz part wx of each of those convs.  None when nothing is hoisted."""
    if not plan.hoisted:
        return None
    zconv, wxs, _ = pp.hoisted([plan.scopes[i][0] for i in plan.hoisted], plan.bn, points.shape[-1])
    p_hi, p_lo = tf_ops.split_rows(points)
    z, _ = tf_ops.linear_tc(p_hi, p_lo, zconv, relu=False, want_f32=True, want_split=False)
    return z, dict(zip(plan.hoisted, wxs))


def _fused_scale(sc, xyz, points, new_xyz, idx, cnt, hz, out):
    """A whole scale in one kernel (:157-180); hz = (z, zoff, wx) of a hoisted first conv."""
    kw = dict(out_f32=out["out_f32"], out_split=out.get("out_split"), units=out.get("units"))
    if sc.route == "fused_hoisted":
        return tf_ops.sa_mlp_fused_hoisted(xyz, *hz, new_xyz, idx, cnt, sc.stack, **kw)
    return tf_ops.sa_mlp_fused(xyz, points, new_xyz, idx, cnt, sc.stack, **kw)


def _layer_scale(sc, convs, xyz, points, new_xyz, idx, hz, units, out):
    """A scale conv by conv (:160-180): the first kernel builds its operand from the neighbour lists as sc.route says,
    each later conv is a linear_tc on the split activations of the one before, and the last writes as `out` says."""
    mid = {} if units is None else dict(units=units)
    if sc.route == "gather":         # :160-165 inside the kernel's operand load (no [B,M,K,C] tensor)
        op = partial(tf_ops.linear_tc_gather, xyz, points, new_xyz, idx)
    elif sc.route == "split":        # :160-165 fused with the split, materialised once in bf16 hi/lo
        op = partial(tf_ops.linear_tc, *tf_ops.group_concat_split(xyz, points, new_xyz, idx))
    elif sc.route == "hoisted":      # the first conv is in z; the second builds relu(z[idx] + rel-xyz . wx) in its loads
        convs = convs[1:]
        op = partial(tf_ops.linear_tc_hoisted, xyz, *hz, new_xyz, idx)
    else:                            # 'expand', wide layer: materialise that operand once (elementwise, memory speed)
        convs = convs[1:]
        op = partial(tf_ops.linear_tc, *tf_ops.hoist_expand_split(xyz, *hz, new_xyz, idx, **mid))
    for f in convs[:-1]:
        _, (hi, lo) = op(f, want_f32=False, want_split=True, **mid)
        op = partial(tf_ops.linear_tc, hi, lo)
    op(convs[-1], want_split=False, **out)


def _group_and_mlp(pp, plan, table, xyz, points, new_xyz, radius_list, nsample_list, mlp_list, dilated_group):
    """Everything of pointnet_sa_module_msg after the sampling, for one block of query points new_xyz (b, m_q, 3), on
    the routes of `plan`: ball queries (:137-145), grouping + MLP + max-pool + mask per scale (:157-180), concat +
    aggregation (:182-185).  table: _hoist_table's.  Returns (new_points, idx_list, cnt_list)."""
    idx_list, cnt_list, units_list = _ball_query(xyz, new_xyz, radius_list, nsample_list, dilated_group, plan.compact,
                                                 [sc.unit_rows for sc in plan.scales] if plan.compact else None)
    if not plan.tc:
        outs = []
        for i, scopes in enumerate(plan.scopes):
            # rows with cnt == 0 come back zero-filled, which is what idx * (cnt > 0) produces (:157-159)
            g = tf_ops.group_concat(xyz, points, new_xyz, idx_list[i])                # :160-165 fused
            for j, s in enumerate(scopes):
                last = j == len(scopes) - 1
                g = _conv(pp, s, g, bn=plan.bn, pool=nsample_list[i] if last else 1, rowmask=cnt_list[i] if last else None)
            outs.append(g)                                                             # :167-180
        new_points = outs[0] if len(outs) == 1 else torch.cat(outs, dim=-1)
        return (_conv(pp, plan.agg, new_points, bn=plan.bn) if plan.agg else new_points), idx_list, cnt_list   # :183-185
    # every scale pools straight into its columns of the fp32 concat buffer (and, split_out, of the split bf16 copy the
    # aggregation conv reads); activations stay split between layers
    bs, m_q = new_xyz.shape[:2]
    ctot = sum(m[-1] for m in mlp_list)
    concat = torch.empty((bs, m_q, ctot), dtype=torch.float32, device=xyz.device)
    if plan.compact:                 # unit lists combine their units with atomicMax on the ZERO-FILLED buffer
        tf_ops.fill_zero(concat)
    split = None
    if plan.split_out:
        ldc = tf_ops.round16(ctot)
        mk = torch.zeros if ldc != ctot else torch.empty
        split = tuple(mk((bs, m_q, ldc), dtype=torch.bfloat16, device=xyz.device) for _ in range(2))
    off = 0
    for i, sc in enumerate(plan.scales):
        idx, cnt = idx_list[i], cnt_list[i]
        units = units_list[i] if sc.units else None
        if units is not None:        # the last conv pools every unit into its group's row
            out = dict(out_f32=(concat, off), units=units, unit_pool=True)
        else:                        # :167-180 conv + BN + ReLU + max + mask
            out = dict(out_f32=(concat, off), out_split=None if split is None else split + (off,), pool=nsample_list[i], rowmask=cnt)
        hz = None if sc.zoff is None else (table[0], sc.zoff, table[1][i])
        if sc.route.startswith("fused"):
            _fused_scale(sc, xyz, points, new_xyz, idx, cnt, hz, out)
        else:
            _layer_scale(sc, [pp.conv(s, plan.bn) for s in plan.scopes[i]], xyz, points, new_xyz, idx, hz, units, out)
        off += mlp_list[i][-1]
    if not plan.agg:
        return concat, idx_list, cnt_list
    cat_hi, cat_lo = split if split is not None else tf_ops.split_rows(concat)                 # :183-185
    return tf_ops.linear_tc(cat_hi, cat_lo, pp.conv(plan.agg, plan.bn))[0], idx_list, cnt_list


def _sampling_segments(n, fps_sample_range_list, fps_method_list, npoint_list, vote_ctr):
    """The sampling table (:84-111) as segments in launch order, each (kind, lo, hi, npoint, col): kind 'iota', 'F'
    (F-FPS) or 'D' (D-FPS) picks npoint indices among the rows [lo, hi) into the columns [col, col + npoint) of fps_idx.
    A fusion-sampling entry is two segments over the same rows: its D-FPS half in the upper columns, listed first so that
    it is forked before the F-FPS half in the lower columns starts."""
    segs, last = [], 0
    for rng, method, npoint in zip(fps_sample_range_list, fps_method_list, npoint_list):
        lo, hi = last, n if rng == -1 else last + rng             # tf.slice size -1 (:86-87)
        col = sum(sg[3] for sg in segs)
        last += rng
        if npoint == 0:                                           # :88-90
            continue
        if vote_ctr is not None:                                  # :91-93
            segs.append(("iota", lo, hi, vote_ctr.shape[1], col))
        elif method == "FS":                                      # :94-99 fusion sampling
            segs += [("D", lo, hi, npoint, col + npoint), ("F", lo, hi, npoint, col)]
        elif npoint == hi - lo:                                   # :100-101
            segs.append(("iota", lo, hi, npoint, col))
        else:                                                     # F-FPS :102-105, D-FPS :106-107
            segs.append(("F" if method == "F-FPS" else "D", lo, hi, npoint, col))
    return segs


def pointnet_sa_module_msg(xyz, points, radius_list, nsample_list, mlp_list, is_training, bn_decay, bn,
                           fps_sample_range_list, fps_method_list, npoint_list, former_fps_idx, use_attention, scope,
                           dilated_group, vote_ctr=None, aggregation_channel=None, debugging=False, epsilon=1e-5, *,
                           params, ffps_mode="direct", aggregation=None, return_debug=False, mlp_mode="tc",
                           fuse_scale=True, gather_in_kernel=True, hoist_first=2, fps_cluster=0, fps_parts=None,
                           fps_packet=False, fps_bucket=None):
    """PointNet++ SA module with multi-scale grouping; returns (new_xyz, new_points, fps_idx).

    Keyword extensions (none changes a result):
      fps_cluster  CTAs per scene of the D-FPS kernels (tf_ops.farthest_point_sample `cluster`);
      fps_bucket   lone D-FPS kernel choice (tf_ops.farthest_point_sample `bucket_kernel`: None automatic, False = cluster kernel);
      fps_packet   D-FPS with the coordinates-in-packet kernel (64 KiB of shared memory per CTA instead of the whole
                   scene: other kernels can share its SMs);
      fps_parts    latency mode (inference only).  FPS emits its samples in order, and a sample is final once its round
                   is done, so the layer consumes the sampling IN PARTS: a lone D-FPS runs as resumable launches of
                   rounds (an int = that many equal parts, or a list of fractions), an F-FPS of at least 256 samples on
                   the matrix-free kernel as two, and every other segment is a part of its own; ball query + grouped
                   MLP + aggregation of a part run on a side stream while the sampling of the next part continues, and
                   the per-part results are joined at the end.
                   Captured in a CUDA graph this is a plain dependency graph -- nothing polls."""
    if use_attention:
        raise NotImplementedError("query_ball_point_withidx (use_attention) is unused by the shipped 3DSSD configs")
    if mlp_mode not in ("tc", "fp32"):
        raise ValueError("mlp_mode must be 'tc' or 'fp32'")
    trainable = _trainable(params, is_training)
    pp = params if trainable else prepare(params, xyz.device)
    aggregation = _cfg.AGGREGATION_SA_FEATURE if aggregation is None else aggregation
    bs, n, _ = xyz.shape
    dev = xyz.device
    nscale = len(radius_list)
    main = torch.cuda.current_stream()
    in_parts = bool(fps_parts) and nscale > 0 and former_fps_idx is None and not is_training
    keep = []                                  # temporaries shared between streams stay alive until the final join
    use_agg = bool(aggregation and aggregation_channel is not None and aggregation_channel != -1)

    # ---- inference: the kernels of every scale, and the hoisted first convs (the feature part of conv0 of every
    # scale, once per POINT, independent of the sampling)
    plan = table = None
    if nscale and not is_training:
        plan = _route_plan(pp, scope, nsample_list, mlp_list, bn, points.shape[-1], use_agg, mlp_mode, fuse_scale,
                           gather_in_kernel, hoist_first)
        if in_parts and plan.hoisted:          # overlaps the first rounds of the sampling
            zs = _side_stream(dev, "hoist")
            zs.wait_stream(main)
            with torch.cuda.stream(zs):
                table = _hoist_table(pp, plan, points)
            z_ready = torch.cuda.Event()
            z_ready.record(zs)

    # ---- sampling (:84-111): every segment writes its indices, segment offset included, straight into its columns of
    # fps_idx, in one launch or in resumable launches of rounds, on the main stream or forked onto a side stream
    segs = _sampling_segments(n, fps_sample_range_list, fps_method_list, npoint_list, vote_ctr)
    fps_idx = torch.empty((bs, sum(sg[3] for sg in segs)), dtype=torch.int32, device=dev)
    parts, forks = [], []                      # (col0, col1, event): fps_idx[:, col0:col1] is complete at `event`
    for kind, lo, hi, npoint, col in segs:
        seg_xyz, seg_points = xyz[:, lo:hi], points[:, lo:hi]      # read in place (scene-strided)
        st, temp, rounds = main, None, [(0, npoint)]
        if kind == "D" and len(segs) > 1:
            # D-FPS next to other segments: independent latency-bound chains on a handful of SMs each, run concurrently
            st = _side_stream(dev, ("fork", len(forks)))
            forks.append(st)
            st.wait_stream(main)
        # latency mode: the lone D-FPS, and an F-FPS of at least 256 samples on the matrix-free kernel, run as resumable
        # launches of rounds that carry their state in `temp`, so that earlier samples are consumed while later ones are
        # still being picked
        elif kind == "F" and in_parts and ffps_mode == "direct" and npoint >= 256 and \
                _ffps_direct(seg_xyz.shape[1], seg_xyz.shape[2] + seg_points.shape[2]):
            temp = torch.empty(seg_xyz.shape[:2], dtype=torch.float32, device=dev)
            rounds = _part_bounds(npoint, 2)
        elif kind == "D" and in_parts and not isinstance(fps_parts, bool) and tf_ops.fps_supports_rounds(hi - lo, 3):
            temp = torch.empty((bs, tf_ops.fps_temp_elems(hi - lo, 3, npoint, bucket_kernel=fps_bucket)),
                               dtype=torch.float32, device=dev)
            rounds = _part_bounds(npoint, fps_parts)
        if temp is not None:
            keep.append(temp)
        out = (fps_idx, col)
        with torch.cuda.stream(st):
            for j0, j1 in rounds:
                if kind == "iota":
                    tf_ops.iota_idx(bs, npoint, dev, out=out, start=lo)
                elif kind == "F" and temp is not None:
                    tf_ops.farthest_point_sample_features(npoint, seg_xyz, seg_points, out=out, idx_offset=lo,
                                                          rounds=(j0, j1), temp=temp)
                elif kind == "F":
                    ffps_indices(npoint, seg_xyz, seg_points, ffps_mode, out=out, idx_offset=lo,
                                 cluster=fps_cluster if fps_cluster < 0 else None)
                elif st is not main:
                    tf_ops.farthest_point_sample(npoint, seg_xyz, out=out, idx_offset=lo, cluster=fps_cluster)
                elif temp is not None:
                    tf_ops.farthest_point_sample(npoint, seg_xyz, out=out, idx_offset=lo, rounds=(j0, j1), temp=temp,
                                                 cluster=fps_cluster, bucket_kernel=fps_bucket)
                else:
                    tf_ops.farthest_point_sample(npoint, seg_xyz, out=out, idx_offset=lo, cluster=fps_cluster,
                                                 packet_kernel=fps_packet, bucket_kernel=fps_bucket)
                # final at an event recorded after the launch, or at once in main-stream order
                ev = None
                if in_parts or st is not main:
                    ev = torch.cuda.Event()
                    ev.record(st)
                parts.append((col + j0, col + j1, ev))
    parts.sort(key=lambda p: p[0])             # column order, in which the consumers' results are joined

    # ---- the consumers (:113-187).  Latency mode: one per part of the sampling, each on its own stream as soon as its
    # samples are final, joined at the end; otherwise one over every sample on the main stream once the sampling is done
    src_xyz = vote_ctr if vote_ctr is not None else xyz
    if not in_parts:
        for _, _, ev in parts:
            if ev is not None:
                main.wait_event(ev)
        if former_fps_idx is not None:
            fps_idx = torch.cat([fps_idx, former_fps_idx], dim=-1).contiguous()    # :113-114
        parts = [(0, fps_idx.shape[1], None)]
    if not nscale:
        new_xyz = tf_ops.gather_point(src_xyz, fps_idx)                            # :116-119
        new_points, debug = tf_ops.gather_point(points.contiguous(), fps_idx), {"idx": [], "cnt": []}   # :186-187
    elif is_training:
        new_xyz = tf_ops.gather_point(src_xyz, fps_idx)
        new_points, idx, cnt, convs = _group_and_mlp_train(pp, scope, xyz, points, new_xyz, radius_list, nsample_list,
                                                           mlp_list, bn, bn_decay, dilated_group, use_agg)
        debug = {"idx": idx, "cnt": cnt} if convs is None else {"idx": idx, "cnt": cnt, "convs": convs}
    else:
        xyz_parts, pts_parts, found, done = [], [], [], []
        for pi, (c0, c1, ev) in enumerate(parts):
            st = main
            if in_parts:
                st = _side_stream(dev, ("part", pi))
                st.wait_event(ev)
                if plan.hoisted:
                    st.wait_event(z_ready)
            with torch.cuda.stream(st):
                nx = tf_ops.gather_point(src_xyz, fps_idx[:, c0:c1])
                if not in_parts:
                    table = _hoist_table(pp, plan, points)
                npnts, idx, cnt = _group_and_mlp(pp, plan, table, xyz, points, nx, radius_list, nsample_list, mlp_list,
                                                 dilated_group)
                if in_parts:
                    done.append(torch.cuda.Event())
                    done[-1].record(st)
            xyz_parts.append(nx); pts_parts.append(npnts); found.append({"idx": idx, "cnt": cnt})
        if not in_parts:
            new_xyz, new_points, debug = xyz_parts[0], pts_parts[0], found[0]
        else:
            for e in done:
                main.wait_event(e)
            for s in forks:
                main.wait_stream(s)
            new_xyz = tf_ops.concat_rows(xyz_parts)
            new_points = tf_ops.concat_rows(pts_parts)
            keep.extend(xyz_parts + pts_parts)
            if return_debug:
                debug = {k: [torch.cat([f[k][i] for f in found], dim=1) for i in range(nscale)] for k in ("idx", "cnt")}
            _KEEPALIVE.append((keep, found if not return_debug else None, table))
            del _KEEPALIVE[:-8]
    if return_debug:
        return new_xyz, new_points, fps_idx, debug
    return new_xyz, new_points, fps_idx


_KEEPALIVE = []   # latency mode: the last layers' cross-stream temporaries (freed a few calls later, long after their use)


def pointnet_sa_module(xyz, points, mlp, is_training, bn_decay, bn, scope, *, params):
    """Global SA layer (layer type SA_Layer_SSG_Last): concat[xyz, points] -> MLP -> max over all points."""
    trainable = _trainable(params, is_training)
    pp = params if trainable else prepare(params, xyz.device)
    g = torch.cat([xyz, points], dim=-1).contiguous()              # xyz FIRST here (:42)
    n = g.shape[1]
    for j in range(len(mlp)):
        g = _conv_train(pp, "%s/conv%d" % (scope, j), g, bn, bn_decay) if is_training else _conv(pp, "%s/conv%d" % (scope, j), g, bn=bn)
    if trainable and n:
        return torch.amax(g, dim=1)                                # gradient split evenly among ties, like tf.reduce_max
    return g.max(dim=1).values if n else g


def pointnet_fp_module(xyz1, xyz2, points1, points2, mlp, is_training, bn_decay, scope, bn=True, *, params,
                       want_split=False):
    """Feature propagation: inverse-distance interpolation from (xyz2, points2) onto xyz1, then an MLP.
    At inference one kernel (tf_ops.fp_interp_split) writes the first conv's split operand [interpolated | points1] and
    the convs chain on the tensor cores; there want_split=True returns (features, (hi, lo)), the split features being the
    operand of whatever conv follows (the detection head).  The training route is the reference's op sequence."""
    pp = params if _trainable(params, is_training) else prepare(params, xyz1.device)
    if not is_training and len(mlp):
        hi, lo = tf_ops.fp_interp_split(xyz1, xyz2, points2, points1)                        # :206-214
        for i in range(len(mlp)):
            last = i == len(mlp) - 1
            x, sp = tf_ops.linear_tc(hi, lo, pp.conv("%s/conv_%d" % (scope, i), bn), want_f32=last,
                                     want_split=want_split or not last)
            if sp is not None:
                hi, lo = sp
        return (x, (hi, lo)) if want_split else x
    dist, idx = tf_ops.three_nn(xyz1, xyz2)
    dist = torch.clamp_min(dist, 1e-10)                            # :207
    inv = 1.0 / dist
    weight = inv / inv.sum(dim=2, keepdim=True)                    # :208-210
    x = tf_ops.three_interpolate(points2, idx, weight.contiguous())
    if points1 is not None:
        x = torch.cat([x, points1], dim=2).contiguous()            # :213-214
    for i in range(len(mlp)):
        x = _conv_train(pp, "%s/conv_%d" % (scope, i), x, bn, bn_decay) if is_training else _conv(pp, "%s/conv_%d" % (scope, i), x, bn=bn)
    return x


def vote_layer(xyz, points, mlp_list, is_training, bn_decay, bn, scope, *, params,
               max_translate_range=_cfg.MAX_TRANSLATE_RANGE, mlp_mode="tc"):
    """Vote layer: per-point MLP -> 3 offsets, clamped to +-max_translate_range (layers_util.py:12-24)."""
    trainable = _trainable(params, is_training)
    pp = params if trainable else prepare(params, xyz.device)
    if is_training:
        for i in range(len(mlp_list)):
            points = _conv_train(pp, "%s/vote_layer_%d" % (scope, i), points, bn, bn_decay)
        off = _conv_train(pp, scope + "/vote_offsets", points, False, bn_decay, relu=False)
    elif mlp_mode == "tc":
        hi, lo = tf_ops.split_rows(points)
        for i in range(len(mlp_list)):
            points, (hi, lo) = tf_ops.linear_tc(hi, lo, pp.conv("%s/vote_layer_%d" % (scope, i), bn), want_split=True)
        off, _ = tf_ops.linear_tc(hi, lo, pp.conv(scope + "/vote_offsets", False), relu=False)
    else:
        for i in range(len(mlp_list)):
            points = _conv(pp, "%s/vote_layer_%d" % (scope, i), points, bn=bn)
        off = _conv(pp, scope + "/vote_offsets", points, bn=False, relu=False)
    translate = tf_ops.vote_translate_train if trainable else tf_ops.vote_translate
    return translate(xyz, off, max_translate_range), points, off                                    # :20-23
