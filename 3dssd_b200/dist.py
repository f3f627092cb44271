"""Batch sharding over the GPUs of one node (SURVEY.md section 8e).

Every operator of the SA path is independent per scene and inference BatchNorm uses moving statistics, so
the path shards by scene with no activation exchange: rank r of G processes scenes [r*B/G, (r+1)*B/G).  The
only collective is ONE all-gather per step of the fixed-size per-scene detection block ([100, 9] fp32 + a
count word); at <= 64 scenes x 3.6 KB it is latency-bound, so a single NCCL call is the right tool.
The reference has no inference sharding (evaluation is single-GPU bs=1, lib/core/evaluator.py:145-147).

DetectionGather keeps the whole exchange inside the captured step: the NMS kernel writes its block and count
straight into a preallocated send buffer, ncclAllGather on that buffer is captured into the step's CUDA graph, and the
gathered result is read through views of the receive buffer -- no pack / unpack kernels and no host work per step
beyond graph.replay().
"""
import contextlib
import functools
import os
from typing import NamedTuple

import torch
import torch.distributed as dist

MAX_OUTPUT_NUM = 100
BLOCK_COLS = 9


def init_from_env(backend=None):
    """Initialise torch.distributed from torchrun's environment; returns (rank, world, local_rank)."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        if backend == "nccl":
            torch.cuda.set_device(local)
        dist.init_process_group(backend=backend, rank=rank, world_size=world)
    return rank, world, local


def shard_bounds(total, rank, world):
    """Contiguous scene range of `rank`; the first total % world ranks take one extra scene."""
    base, extra = divmod(total, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def shard_batch(batch, rank, world):
    lo, hi = shard_bounds(batch.shape[0], rank, world)
    return batch[lo:hi]


def _world(group=None):
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size(group), dist.get_rank(group)
    return 1, 0


class DetectionGather:
    """Send / receive buffers of the per-step all-gather, owned by one step pipeline.

    total_scenes scenes are sharded with shard_bounds; every rank sends b_max = ceil(total / world) slots (unused
    slots stay zero).  Layout of a rank's slice (bytes): [b_max * 100 * 9 fp32 block | b_max int32 count].
      out()      -> (block [b_local,100,9] fp32, count [b_local] int32) views of the SEND buffer: hand them to the NMS
      gather()   -> enqueue the all-gather on the current stream (CUDA-graph capturable; a no-op for one rank)
      result()   -> (blocks [total,100,9], counts [total]) of all scenes, assembled from views of the RECEIVE buffer
      raw        -> the receive buffer itself (uint8), what a host reads back in one copy
    group: the process group (= NCCL communicator) to use.  Step pipelines that run concurrently on different streams
    must not share one -- collectives of one communicator may not overlap -- so each pipeline passes its own group."""

    def __init__(self, total_scenes, device, group=None, max_output=MAX_OUTPUT_NUM):
        self.world, self.rank = _world(group)
        self.group = group
        self.total = int(total_scenes)
        self.max_output = int(max_output)
        lo, hi = shard_bounds(self.total, self.rank, self.world)
        self.b_local = hi - lo
        self.b_max = (self.total + self.world - 1) // self.world
        self.block_bytes = self.b_max * self.max_output * BLOCK_COLS * 4
        self.slice_bytes = (self.block_bytes + self.b_max * 4 + 15) // 16 * 16      # 16-byte multiple (vector copies)
        self._alloc(device)

    def _alloc(self, device):
        self.send = torch.zeros((self.slice_bytes,), dtype=torch.uint8, device=device)
        self.raw = self.send if self.world == 1 else torch.zeros((self.world * self.slice_bytes,), dtype=torch.uint8,
                                                                 device=device)

    def _views(self, buf):
        blk = buf[: self.block_bytes].view(torch.float32).view(self.b_max, self.max_output, BLOCK_COLS)
        cnt = buf[self.block_bytes: self.block_bytes + self.b_max * 4].view(torch.int32)
        return blk, cnt

    def out(self):
        blk, cnt = self._views(self.send)
        return blk[: self.b_local], cnt[: self.b_local]

    def gather(self):
        if self.world > 1:
            dist.all_gather_into_tensor(self.raw, self.send, group=self.group)

    def result(self):
        blocks, counts = [], []
        for r in range(self.world):
            lo, hi = shard_bounds(self.total, r, self.world)
            blk, cnt = self._views(self.raw[r * self.slice_bytes: (r + 1) * self.slice_bytes])
            blocks.append(blk[: hi - lo]); counts.append(cnt[: hi - lo])
        if self.world == 1:
            return blocks[0], counts[0]
        return torch.cat(blocks, dim=0), torch.cat(counts, dim=0)


def peer_layout(world, slice_bytes):
    """Byte offsets inside one pipeline's share of the symmetric allocation (csrc/peer_gather.cu):
    ((recv_off parity 0, parity 1), (flag_off parity 0, parity 1), total bytes)."""
    recv = world * slice_bytes
    flags = (world * 4 + 15) // 16 * 16
    return (0, recv), (2 * recv, 2 * recv + flags), 2 * recv + 2 * flags


class PeerArena:
    """ONE symmetric allocation (mapped into every rank of `group`) shared by all step pipelines of a process: a single
    rendezvous instead of one per pipeline.  take(nbytes) hands out 256-byte aligned shares, in the same order on every rank."""

    def __init__(self, nbytes, device, group=None):
        import torch.distributed._symmetric_memory as symm
        self.group = dist.group.WORLD if group is None else group
        self.buf = symm.empty((int(nbytes),), dtype=torch.uint8, device=device)
        self.handle = symm.rendezvous(self.buf, self.group)
        self.buf.zero_()                                  # flags start at 0, before any peer can write
        torch.cuda.synchronize(device)
        dist.barrier(self.group)
        self.peer_bases = [int(p) for p in self.handle.buffer_ptrs]
        self.used = 0

    @staticmethod
    def share_bytes(world, slice_bytes):
        return (peer_layout(world, slice_bytes)[2] + 255) // 256 * 256

    def take(self, nbytes):
        off = self.used
        self.used += (int(nbytes) + 255) // 256 * 256
        if self.used > self.buf.numel():
            raise ValueError("PeerArena exhausted")
        return off


class PeerGather(DetectionGather):
    """DetectionGather with the exchange done by ONE kernel of this library over NVLink peer memory
    (tf_ops.peer_allgather, csrc/peer_gather.cu) instead of ncclAllGather: every rank stores its slice straight into
    the peers' symmetric buffers, publishes a flag and waits for theirs.  Same interface and the same `raw` layout;
    capturable; pipelines need no process group of their own (nothing here is a communicator).  Every rank must call
    gather() the same number of times."""

    def __init__(self, total_scenes, device, arena, max_output=MAX_OUTPUT_NUM):
        self.arena = arena
        super().__init__(total_scenes, device, group=arena.group, max_output=max_output)

    def _alloc(self, device):
        from . import tf_ops                                   # (tf_ops does not import this module)
        self._tf_ops = tf_ops
        super()._alloc(device)
        self.raw = torch.zeros((self.world * self.slice_bytes,), dtype=torch.uint8, device=device)
        self.recv_off, self.flag_off, total = peer_layout(self.world, self.slice_bytes)
        base = self.arena.take(total)
        self.peers = torch.tensor([b + base for b in self.arena.peer_bases], dtype=torch.int64, device=device)
        self.state = torch.zeros((4,), dtype=torch.int32, device=device)   # replay count, CTA count, time-outs

    def timeouts(self):
        """Waits that gave up (a peer that never delivered): 0 in a healthy run.  Synchronises."""
        return int(self.state[2].item())

    def gather(self):
        self._tf_ops.peer_allgather(self.send, self.peers, self.world, self.rank, self.slice_bytes, self.recv_off, self.flag_off,
                                    self.state, self.raw)


def gather_detections(block, count, total_scenes, group=None):
    """One-shot form: all-gather per-scene detection blocks block [b_local, 100, 9] fp32 / count [b_local] int32 of a
    batch of `total_scenes` scenes sharded with shard_bounds -> ([total, 100, 9], [total]) on every rank.
    total_scenes is required: with uneven shards the ranks cannot derive a common slot count from their own b_local."""
    world, rank = _world(group)
    if world == 1:
        return block, count
    lo, hi = shard_bounds(int(total_scenes), rank, world)
    if block.shape[0] != hi - lo or count.shape[0] != hi - lo:
        raise ValueError("rank %d holds %d scenes but shard_bounds(%d, %d, %d) assigns it %d"
                         % (rank, block.shape[0], total_scenes, rank, world, hi - lo))
    g = DetectionGather(total_scenes, block.device, group=group, max_output=block.shape[1])
    b, c = g.out()
    b.copy_(block); c.copy_(count)
    g.gather()
    return g.result()


# ---- SyncBN (DESIGN.md section 3.18) --------------------------------------------------------------------------------

BN_SYNC_THREADS = 128         # channels per exchange CTA of csrc/bn.cu's SyncBN finalize


def bn_sync_area_bytes(world, c):
    """Bytes of one (BN scope, direction) area of csrc/bn.cu's SyncBN (ssd3d_bn_sync_area_bytes): per parity a data block
    [world][3][c] of doubles and a flag block [world][ceil(c / 128)] of int32, each rounded up to 16 bytes."""
    world, c = int(world), int(c)
    if world < 1 or c < 1:
        raise ValueError("bn_sync_area_bytes: world=%d c=%d" % (world, c))
    data = _round(world * 3 * c * 8, 16)
    flags = _round(world * (-(-c // BN_SYNC_THREADS)) * 4, 16)
    return 2 * data + 2 * flags


class BnSyncLayout(NamedTuple):
    """areas[scope] = (forward area offset, backward area offset) in bytes inside every rank's symmetric buffer;
    nbytes: the share's size."""
    areas: dict
    nbytes: int


def bn_sync_layout(channels, world, base=0):
    """BnSyncLayout of the BN scopes `channels` = [(scope, c), ...] over `world` ranks from byte offset `base` (a 16-byte
    multiple): every scope gets its own forward area, then its own backward area, in the order given."""
    base = int(base)
    if base % 16:
        raise ValueError("bn_sync_layout: base=%d must be a 16-byte multiple" % base)
    areas, off = {}, base
    for scope, c in channels:
        if scope in areas:
            raise ValueError("bn_sync_layout: scope %s listed twice" % scope)
        n = bn_sync_area_bytes(world, c)
        areas[scope] = (off, off + n)
        off += 2 * n
    return BnSyncLayout(areas, off - base)


def _bn_channels(tp):
    return [(s, tp.tensors[s + "/bn/moving_mean"].numel()) for s in tp.bn_scopes()]


class BnSync:
    """The SyncBN handle of one rank (TrainableParams.start_bn_sync): which ranks (peers, world, rank), where each BN
    scope's forward and backward exchange live in the symmetric buffers (bn_sync_layout from byte `base`), and their
    replay counters and time-out counts (state [scopes, 2, 4] int32 on the device).  Every scope has its own areas,
    flags and counters, so the order in which scopes exchange does not matter.  Each scope exchanges once per step in the
    forward on every rank.  In the backward it exchanges once per step on every rank, or, when nothing below its
    BatchNorm needs a gradient (a frozen layer below the lowest trained one, TrainableParams(trainable=...)), on no rank:
    every rank freezes the same set, so the ranks skip the same scopes and each scope's counter stays in step across them.
    before_exchange(scope, direction): optional host callable run just before each launch
    (direction 0 forward, 1 backward): tests that simulate ranks on one device bring the ranks together with it."""

    def __init__(self, tp, peers, world, rank, base=0, before_exchange=None):
        from .tf_ops import BnSyncSlot
        self.world, self.rank = int(world), int(rank)
        if not 0 <= self.rank < self.world:
            raise ValueError("BnSync: rank=%d outside world=%d" % (rank, world))
        if not isinstance(peers, torch.Tensor) or peers.dtype != torch.int64 or peers.numel() != self.world:
            raise ValueError("BnSync: peers must be an int64 tensor of world=%d bases" % self.world)
        self.layout = bn_sync_layout(_bn_channels(tp), self.world, base)
        self.state = torch.zeros((len(self.layout.areas), 2, 4), dtype=torch.int32, device=tp.device)
        self._slots = {}
        for i, (scope, offs) in enumerate(self.layout.areas.items()):
            self._slots[scope] = tuple(
                BnSyncSlot(peers, self.world, self.rank, off, self.state[i, d],
                           None if before_exchange is None else functools.partial(before_exchange, scope, d))
                for d, off in enumerate(offs))

    @staticmethod
    def symmetric_bytes(tp, world):
        return bn_sync_layout(_bn_channels(tp), world).nbytes

    def slots(self, scope):
        """(forward, backward) tf_ops.BnSyncSlot of `scope`."""
        if scope not in self._slots:
            raise ValueError("BnSync: %s has no BatchNorm" % scope)
        return self._slots[scope]

    def replays(self):
        """[scopes, 2] exchanges completed per scope and direction (a view of the device state)."""
        return self.state[:, :, 0]

    def timeouts(self):
        """Waits that gave up (a peer that never arrived): 0 in a healthy run.  Synchronises."""
        return int(self.state[:, :, 2].sum().item())


# ---- data-parallel training (DESIGN.md section 3.9) -----------------------------------------------------------------

ALLREDUCE_CTAS = 64           # CTAs per rank of one allreduce launch; all must be co-resident on the device
CLIP_NORM = 5.0               # trainer.py:143-145, tf.clip_by_global_norm(grads, 5.0)
_HEAD_FLOATS = 8              # gathered slice: 7 losses, the rank's gradient norm, then the BN record


class AllreduceLayout(NamedTuple):
    """Where csrc/grad_exchange.cu's allreduce keeps its buffers: n floats cut into `world` chunks of `chunk` floats
    (rank p owns [p*chunk, (p+1)*chunk), zero past n), each cut into `ctas` sub-slices of `sub` floats (both multiples
    of 4).  r1 / r2 / f1 / f2: byte offsets per parity inside every rank's symmetric buffer; nbytes: the share's size."""
    n: int
    world: int
    ctas: int
    chunk: int
    sub: int
    r1: tuple
    r2: tuple
    f1: tuple
    f2: tuple
    nbytes: int


def allreduce_layout(n, world, ctas=ALLREDUCE_CTAS, base=0):
    """AllreduceLayout of an n-float gradient over `world` ranks, placed at byte offset `base` (a 16-byte multiple)."""
    n, world, ctas, base = int(n), int(world), int(ctas), int(base)
    if n <= 0 or world < 1 or ctas < 1 or base % 16:
        raise ValueError("allreduce_layout: n=%d world=%d ctas=%d base=%d" % (n, world, ctas, base))
    chunk = ((n + world - 1) // world + 3) // 4 * 4
    sub = ((chunk + ctas - 1) // ctas + 3) // 4 * 4
    data = world * chunk * 4
    flags = (world * ctas * 4 + 15) // 16 * 16
    r1 = (base, base + data)
    r2 = (base + 2 * data, base + 3 * data)
    f1 = (base + 4 * data, base + 4 * data + flags)
    f2 = (base + 4 * data + 2 * flags, base + 4 * data + 3 * flags)
    return AllreduceLayout(n, world, ctas, chunk, sub, r1, r2, f1, f2, 4 * data + 4 * flags)


def simulated_ctas(world, sms, ctas=ALLREDUCE_CTAS):
    """CTAs per rank when `world` ranks are simulated on ONE device of `sms` SMs.  A rank's kernels before its allreduce
    (clip scale, loss copy) must still find an SM while the other ranks' allreduce CTAs already spin.  Spinning CTAs are
    spread one per SM first, and once they cover every SM those kernels were seen not to be placed until the spinners
    gave up.  So (world - 1) * ctas must stay below the SM count.  Between GPUs this does not arise."""
    return max(1, min(int(ctas), (int(sms) - 1) // max(1, int(world) - 1)))


def _round(x, m):
    return (int(x) + m - 1) // m * m


class DataParallel:
    """Data-parallel training with the semantics of the reference's towers (trainer.py:143-154, trainer_utils.py:23-46,
    tf_util.py:438-443): each rank clips its own gradient to global norm 5, the clipped gradients are averaged in rank
    order, and every rank's batch statistics update the moving averages, in rank order.  Every rank ends a step with the
    same gradient bits and the same statistics; with the same elementwise optimizer the replicas stay identical.
    sync_bn=True (the reference's MODEL.NETWORK.SYNC_BN) normalises every BatchNorm with the statistics of all ranks'
    rows instead (BnSync, DESIGN.md section 3.18); the moving statistics are then updated once per step, in the forward,
    with those statistics, and exchange() leaves them alone.

        dp = DataParallel(tp, arena)                # arena: PeerArena of >= DataParallel.symmetric_bytes(tp, world)
        for step ...:
            dp.zero_grad()
            with dp.recording():
                losses = <forward on shard_batch(batch, rank, world)>
            losses["total"].backward()
            mean_losses = dp.exchange(losses)       # clip -> allreduce mean -> gather -> BN update
            optimizer.step()                        # e.g. torch.optim.Adam(tp.parameters())

    DataParallel(tp, arena) serves torchrun ranks (world and rank from arena.group) and broadcasts rank 0's parameters
    and moving statistics at construction.  DataParallel(tp, peers=[base of every rank's symmetric buffer], world=G,
    rank=r) runs ranks simulated on one device (tests); nothing is broadcast.  Every rank must call exchange() the same
    number of times; nothing in a step synchronises the host."""

    def __init__(self, tp, arena=None, *, peers=None, world=None, rank=None, ctas=ALLREDUCE_CTAS, clip_norm=CLIP_NORM,
                 sync_bn=False, before_exchange=None):
        from . import tf_ops
        self._tf_ops = tf_ops
        self.tp, self.clip_norm = tp, float(clip_norm)
        dev = tp.device
        if arena is not None:
            self.world, self.rank = _world(arena.group)
            bases = arena.peer_bases
        else:
            if peers is None or world is None or rank is None:
                raise ValueError("DataParallel: pass a PeerArena, or peers, world and rank for simulated ranks")
            self.world, self.rank, bases = int(world), int(rank), [int(b) for b in peers]
            sms = torch.cuda.get_device_properties(dev).multi_processor_count
            if (self.world - 1) * int(ctas) >= sms:
                raise ValueError("DataParallel: %d simulated ranks x %d CTAs need (world - 1) * ctas < %d SMs (simulated_ctas)"
                                 % (self.world, ctas, sms))
        if len(bases) != self.world or not 0 <= self.rank < self.world:
            raise ValueError("DataParallel: %d peer bases for world=%d rank=%d" % (len(bases), self.world, self.rank))
        self.grad, stats = tp.flat_grads(), tp.flat_stats()
        if arena is not None and self.world > 1:
            self._broadcast(arena.group)
        self.nstats = stats.numel()
        self.slice_floats = _round(_HEAD_FLOATS + self.nstats, 4)
        self.slice_bytes = 4 * self.slice_floats
        ar_bytes, ga_bytes = self._share_bytes(self.grad.numel(), self.slice_bytes, self.world, ctas)
        sb_bytes = BnSync.symmetric_bytes(tp, self.world) if sync_bn else 0
        if arena is not None:
            ar_base, ga_base = arena.take(ar_bytes), arena.take(ga_bytes)
            sb_base = arena.take(sb_bytes) if sync_bn else 0
        else:
            ar_base, ga_base = 0, _round(ar_bytes, 256)
            sb_base = ga_base + _round(ga_bytes, 256)
        self.layout = allreduce_layout(self.grad.numel(), self.world, ctas, base=ar_base)
        recv, flag, _ = peer_layout(self.world, self.slice_bytes)
        self.recv_off = (ga_base + recv[0], ga_base + recv[1])
        self.flag_off = (ga_base + flag[0], ga_base + flag[1])
        self.peers = torch.tensor(bases, dtype=torch.int64, device=dev)
        self.send = torch.zeros((self.slice_floats,), dtype=torch.float32, device=dev)
        self.gathered = torch.zeros((self.world, self.slice_floats), dtype=torch.float32, device=dev)
        self.record = self.send[_HEAD_FLOATS:_HEAD_FLOATS + self.nstats]   # the forward writes straight into the slice
        self.scale = torch.zeros((1,), dtype=torch.float32, device=dev)
        self.workspace = torch.empty((int(tf_ops.lib().ssd3d_grad_clip_scale_workspace(self.grad.numel())),), dtype=torch.uint8,
                                     device=dev)
        self.state_allreduce = torch.zeros((4,), dtype=torch.int32, device=dev)
        self.state_gather = torch.zeros((4,), dtype=torch.int32, device=dev)
        self.bn_sync = BnSync(tp, self.peers, self.world, self.rank, sb_base, before_exchange) if sync_bn else None
        self.decay = None

    @staticmethod
    def _share_bytes(n, slice_bytes, world, ctas):
        return allreduce_layout(n, world, ctas).nbytes, peer_layout(world, slice_bytes)[2]

    @staticmethod
    def symmetric_bytes(tp, world, ctas=ALLREDUCE_CTAS, sync_bn=False):
        """Bytes of symmetric memory one DataParallel over `world` ranks takes (size a PeerArena with at least this)."""
        n = sum(t.numel() for t in tp.parameters())
        nstats = sum(tp.tensors[s + suffix].numel() for s in tp.bn_scopes() for suffix in tp._STATS)
        ar, ga = DataParallel._share_bytes(n, 4 * _round(_HEAD_FLOATS + nstats, 4), world, ctas)
        sb = BnSync.symmetric_bytes(tp, world) if sync_bn else 0
        return _round(ar, 256) + _round(ga, 256) + _round(sb, 256)

    def _broadcast(self, group):
        src = dist.get_global_rank(group, 0)
        with torch.no_grad():
            for k, t in self.tp.tensors.items():                # frozen tensors too: no step ever makes them agree
                if not k.endswith(self.tp._STATS):
                    dist.broadcast(t.data, src=src, group=group)
            dist.broadcast(self.tp.stats_flat, src=src, group=group)

    def zero_grad(self):
        self.tp.zero_flat_grads()

    @contextlib.contextmanager
    def recording(self):
        """The forward of a step: every training BatchNorm records its batch statistics (exactly once per scope, one decay)
        into this rank's slice of the per-step gather instead of updating the moving statistics in place.  With sync_bn
        every training BatchNorm is synchronised over the ranks instead (exactly once per scope, one decay)."""
        sync = self.bn_sync is not None
        if sync:
            self.tp.start_bn_sync(self.bn_sync)
        else:
            self.tp.start_bn_record(self.record)
        ok = False
        try:
            yield self
            ok = True
        finally:
            decay = self.tp.finish_bn_sync(check=ok) if sync else self.tp.finish_bn_record(check=ok)
        self.decay = decay

    def exchange(self, losses):
        """After backward(): clip scale -> allreduce mean of the clipped gradients (in place in every .grad) -> gather of
        losses, norms and batch statistics -> BN moving-statistics update of every rank.  losses: dict with
        loss.LOSS_NAMES and "total" (0-d tensors).  Returns the rank-averaged losses (summed in double in rank order).
        With sync_bn the forward has already updated the moving statistics, so the BN update is skipped."""
        from .loss import LOSS_NAMES
        keys = LOSS_NAMES + ("total",)
        if self.decay is None:
            raise ValueError("exchange: no recorded forward since the last exchange (use recording())")
        T, W = self._tf_ops, self.world
        with torch.no_grad():
            self.send[:len(keys)].copy_(torch.stack([losses[k].detach().reshape(()).float() for k in keys]))
        T.grad_clip_scale(self.grad, self.send[len(keys):len(keys) + 1], self.scale, self.clip_norm, self.workspace)
        T.peer_allreduce_mean(self.grad, self.scale, self.peers, W, self.rank, self.layout, self.state_allreduce)
        T.peer_allgather(self.send.view(torch.uint8), self.peers, W, self.rank, self.slice_bytes, self.recv_off, self.flag_off,
                         self.state_gather, self.gathered.view(-1).view(torch.uint8))
        if self.bn_sync is None:
            T.bn_moving_update_ranks(self.tp.stats_flat, self.gathered[:, _HEAD_FLOATS:_HEAD_FLOATS + self.nstats], W, self.decay)
        self.decay = None
        g = self.gathered[:, :len(keys)].double()
        acc = g[0].clone()
        for r in range(1, W):
            acc += g[r]
        mean = (acc / W).float()
        return {k: mean[i] for i, k in enumerate(keys)}

    def norms(self):
        """Every rank's gradient norm of the last exchange, [world] (a view of the gathered buffer)."""
        return self.gathered[:, _HEAD_FLOATS - 1]

    def timeouts(self):
        """Waits that gave up (a peer that never arrived): 0 in a healthy run.  Synchronises."""
        n = int(self.state_allreduce[2].item()) + int(self.state_gather[2].item())
        return n + (self.bn_sync.timeouts() if self.bn_sync is not None else 0)
