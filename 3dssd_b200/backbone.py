"""The 3DSSD set-abstraction backbone as a driver over a 16-field layer table.

Follows SingleStageDetector.network_forward's backbone loop
(/root/reference/lib/modeling/single_stage_detector.py:115-125) and LayerBuilder.build_layer
(/root/reference/lib/builder/layer_builder.py:45-101): xyz_list / feature_list / fps_idx_list grow by one
entry per layer, layers address their inputs by index.
"""
from typing import NamedTuple

import torch

from . import config as _cfg
from . import layers_util as L
from . import tf_ops
from .params import init_params, prepare


class SABackbone:
    """Inference driver.  `forward(points)` takes [B, N, 3+C] float32 CUDA points and returns the three lists.

    capture(points) records the whole forward into a CUDA graph (no allocation or host sync happens inside
    the kernels, include/ssd3d.h) and returns a callable that replays it on new data copied into the static
    input buffer.
    """

    def __init__(self, arch=None, params=None, in_channels=_cfg.INPUT_CHANNELS - 3, device="cuda", ffps_mode="direct",
                 seed=0, mlp_mode="tc", fuse_scale=True, head=None, gather_in_kernel=True, hoist_first=2, fps_cluster=0,
                 latency_mode=False, fps_parts=(0.34, 0.28, 0.22, 0.16), fps_packet=False, fps_bucket=None):
        """fps_cluster: CTAs per scene of the D-FPS kernels (0 heuristic, < 0 cap; see tf_ops.farthest_point_sample).
        latency_mode: minimise the time of ONE step instead of the throughput of many in flight -- every SA layer
        consumes its sampling in parts (pointnet_sa_module_msg `fps_parts`): a lone D-FPS (layer 1) is cut into
        resumable launches with the given round fractions, fusion-sampling layers hand over their halves separately.
        fps_bucket: layer-1 D-FPS kernel (tf_ops.farthest_point_sample `bucket_kernel`): the single-CTA kernel with spatial
        pruning occupies one SM per scene but its round is longer than the 8-CTA cluster kernel's, so the default takes it
        for throughput (many steps in flight share the SMs) and the cluster kernel in latency mode.  Same indices."""
        self.arch = _cfg.ARCH_3DSSD if arch is None else arch
        self.in_channels = in_channels
        self.device = torch.device(device)
        if params is None:
            params = init_params(self.arch, in_channels, seed=seed)
        self.params = prepare(params, self.device).prepare_all()
        self.ffps_mode = ffps_mode
        self.mlp_mode = mlp_mode
        self.gather_in_kernel = gather_in_kernel
        self.hoist_first = hoist_first
        self.fuse_scale = fuse_scale
        self.fps_cluster = fps_cluster
        self.fps_packet = fps_packet
        self.fps_bucket = (False if latency_mode else None) if fps_bucket is None else bool(fps_bucket)
        self.latency_mode = latency_mode
        self.fps_parts = fps_parts if isinstance(fps_parts, int) else list(fps_parts)
        self.head = head                      # optional head.DetectionHead: real detections instead of the stand-in block
        self._graph = None

    def forward(self, points, return_debug=False):
        if points.dim() != 3 or points.shape[-1] != 3 + self.in_channels:
            raise ValueError("points must be [B, N, %d], got %s" % (3 + self.in_channels, tuple(points.shape)))
        xyz0, feat0 = tf_ops.split_points(points)                  # single_stage_detector.py:116-117
        xyz_list, feat_list = [xyz0], [feat0]
        fps_list = [None]
        dbg = []
        for spec in self.arch:
            (xyz_i, feat_i, radius, nsample, mlps, bn, rng, method, npoint, former, attn, ltype, scope, dilated,
             vote_idx, agg) = spec
            former_idx = fps_list[former] if former != -1 else None
            vote_ctr = xyz_list[vote_idx] if vote_idx != -1 else None
            if ltype == "SA_Layer":
                parts = None
                if self.latency_mode and len(radius) and vote_ctr is None:
                    parts = self.fps_parts if (len(npoint) == 1 and method[0] == "D-FPS") else True
                r = L.pointnet_sa_module_msg(xyz_list[xyz_i[0]], feat_list[feat_i[0]], radius, nsample, mlps, False,
                                             None, bn, rng, method, npoint, former_idx, attn, scope, dilated, vote_ctr,
                                             agg, params=self.params, ffps_mode=self.ffps_mode, return_debug=True,
                                             mlp_mode=self.mlp_mode, fuse_scale=self.fuse_scale,
                                             gather_in_kernel=self.gather_in_kernel, hoist_first=self.hoist_first,
                                             fps_cluster=self.fps_cluster, fps_parts=parts, fps_packet=self.fps_packet,
                                             fps_bucket=self.fps_bucket)
                xyz_list.append(r[0]); feat_list.append(r[1]); fps_list.append(r[2]); dbg.append(r[3])
            elif ltype == "Vote_Layer":
                nx, nf, off = L.vote_layer(xyz_list[xyz_i[0]], feat_list[feat_i[0]], mlps, False, None, bn, scope,
                                           params=self.params, mlp_mode=self.mlp_mode)
                xyz_list.append(nx); feat_list.append(nf); fps_list.append(None); dbg.append({"offsets": off})
            elif ltype == "SA_Layer_SSG_Last":
                xyz_list.append(None)
                feat_list.append(L.pointnet_sa_module(xyz_list[xyz_i[0]], feat_list[feat_i[0]], mlps, False, None, bn,
                                                      scope, params=self.params))
                fps_list.append(None); dbg.append({})
            elif ltype == "FP_Layer":
                xyz_list.append(xyz_list[xyz_i[0]])
                feat_list.append(L.pointnet_fp_module(xyz_list[xyz_i[0]], xyz_list[xyz_i[1]], feat_list[feat_i[0]],
                                                      feat_list[feat_i[1]], mlps, False, None, scope, bn,
                                                      params=self.params))
                fps_list.append(None); dbg.append({})
            else:
                raise ValueError("unknown layer type %r" % (ltype,))
        if return_debug:
            return xyz_list, feat_list, fps_list, dbg
        return xyz_list, feat_list, fps_list

    __call__ = forward

    # ---- per-scene detection block ---------------------------------------------------------------------------
    def detections(self, xyz_list, feat_list, out=None):
        """Per-scene detection block [B,100,9] + count [B]: the detection head + decode + BEV NMS when a head is
        attached, otherwise the stand-in derived from the CG layer.  out=(block, count) preallocated outputs."""
        if self.head is not None:
            return self.head(xyz_list, feat_list, out=out)
        blk, cnt = self.detection_block(xyz_list, feat_list)
        if out is not None:
            out[0].copy_(blk); out[1].copy_(cnt)
            return out
        return blk, cnt

    @staticmethod
    def detection_block(xyz_list, feat_list, max_output=100):
        """[B, 100, 9] fp32 + [B] int32, the shape of the reference's per-scene output (MAX_OUTPUT_NUM: 100,
        3dssd.yaml:70; 7 box parameters + score + class).  Until the detection head exists the block holds
        the first 100 candidate centres and feature statistics of the CG layer, so that the multi-GPU gather
        moves the real message shape (SURVEY.md section 8e)."""
        ctr, feat = xyz_list[-1], feat_list[-1]
        b = ctr.shape[0]
        k = min(max_output, ctr.shape[1])
        blk = torch.zeros((b, max_output, 9), dtype=torch.float32, device=ctr.device)
        blk[:, :k, 0:3] = ctr[:, :k]
        f = feat[:, :k]
        blk[:, :k, 3] = f.mean(dim=-1)
        blk[:, :k, 4] = f.amax(dim=-1)
        blk[:, :k, 5] = f.amin(dim=-1)
        blk[:, :k, 6] = (f * f).mean(dim=-1)
        blk[:, :k, 7] = (f > 0).float().mean(dim=-1)
        cnt = torch.full((b,), k, dtype=torch.int32, device=ctr.device)
        return blk, cnt

    # ---- CUDA graph ---------------------------------------------------------------------------------------
    def capture(self, example_points, warmup=2, gather=None):
        """Record forward + detections (+ the multi-GPU all-gather when `gather`, a dist.DetectionGather, is given: the
        NMS writes into its send buffer and ncclAllGather is captured with the kernels) into one CUDA graph.  Returns
        replay(points=None) -> (forward outputs, (block, count)); with `gather` the pair holds this rank's views of the
        send buffer and gather.result() / gather.raw hold all ranks' detections after the replay."""
        static_in = example_points.clone()
        out_buf = gather.out() if gather is not None else None
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(warmup):
                out = self.forward(static_in)
                blk = self.detections(out[0], out[1], out=out_buf)
                if gather is not None:
                    gather.gather()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        # thread_local: NCCL's watchdog thread polls its events while this thread captures
        kw = {"capture_error_mode": "thread_local"} if (gather is not None and gather.world > 1) else {}
        with torch.cuda.graph(g, **kw):
            out = self.forward(static_in)
            blk = self.detections(out[0], out[1], out=out_buf)
            if gather is not None:
                gather.gather()
        self._graph = (g, static_in, out, blk)

        def replay(points=None):
            if points is not None:
                static_in.copy_(points, non_blocking=True)
            g.replay()
            return out, blk

        return replay


class TrainOutputs(NamedTuple):
    """What the loss of a training step needs: head = (pred_cls, pred_offset, pred_angle_cls, pred_angle_res) of
    head.box_regression_head; vote_offsets = the raw offsets of each vote layer; base_xyz = the centres of the last SA
    layer (the candidate points of the head); vote_base = the input points of the last vote layer."""
    head: tuple
    vote_offsets: list
    base_xyz: torch.Tensor
    vote_base: torch.Tensor


def train_forward(arch, tp, xyz, feat, *, bn_decay=None):
    """The backbone loop of SABackbone.forward in training mode (SA and vote layers, batch-statistics BatchNorm) with
    params.TrainableParams, then conv1d_0 and the box-regression head of the 3DSSD head on the last layer's features
    (single_stage_detector.py:115-125, head_builder.py:81-114).  Everything is differentiable w.r.t. tp's parameters.
    bn_decay: the decay of every BatchNorm's moving statistics in this forward (model_forward(bn_decay),
    trainer.py:130; solver.Solver.bn_decay gives the scheduled value); None keeps the layers' default of 0.9."""
    from . import head as _head
    xyz_l, feat_l, fps_l, offs, vote_base = [xyz], [feat], [None], [], None
    for spec in arch:
        (xyz_i, feat_i, radius, nsample, mlps, bn, rng, method, npoint, former, attn, ltype, scope, dilated, vote_idx, agg) = spec
        if ltype == "SA_Layer":
            r = L.pointnet_sa_module_msg(xyz_l[xyz_i[0]], feat_l[feat_i[0]], radius, nsample, mlps, True, bn_decay, bn, rng, method,
                                         npoint, fps_l[former] if former != -1 else None, attn, scope, dilated,
                                         xyz_l[vote_idx] if vote_idx != -1 else None, agg, params=tp)
            xyz_l.append(r[0]); feat_l.append(r[1]); fps_l.append(r[2])
        elif ltype == "Vote_Layer":
            vote_base = xyz_l[xyz_i[0]]                                 # PRED_VOTE_BASE (layer_builder.py:96)
            nx, nf, off = L.vote_layer(vote_base, feat_l[feat_i[0]], mlps, True, bn_decay, bn, scope, params=tp)
            xyz_l.append(nx); feat_l.append(nf); fps_l.append(None); offs.append(off)
        else:
            raise ValueError("layer type %r has no training driver here" % (ltype,))
    f = tp.conv_train("conv1d_0", feat_l[-1], True, bn_decay)
    return TrainOutputs(_head.box_regression_head(f, 1, 1, 6, True, True, params=tp, bn_decay=bn_decay), offs, xyz_l[-1], vote_base)
