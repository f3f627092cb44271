"""numpy restatement of the data-parallel exchange (3dssd_b200/csrc/grad_exchange.cu, DESIGN.md section 3.9).

The reference averages its towers' clipped gradients and lets every tower update the BatchNorm moving statistics
(lib/core/trainer.py:143-154, lib/utils/trainer_utils.py:23-46, lib/utils/tf_util.py:438-443).  Here each step of that
is one pinned float32 / float64 recipe, so the kernels must reproduce this module bit for bit:
  norm_r  = float32(sqrt(sum g_r^2)), the double sum over the kernel's fixed tree (sumsq_tree)
  scale_r = rn(clip * minimum(rn(1 / use_norm), rn(1 / clip))), use_norm = norm_r if finite else NaN
  c_r     = rn(g_r * scale_r)
  mean    = float32((sum_r (double) c_r, rank order) / G)
  stats   = for r in rank order: v = rn(v - rn(rn(v - b_r) * rn(1 - decay)))
  losses  = float32((sum_r (double) loss_r, rank order) / G)
"""
import numpy as np

CLIP_BLOCKS = CLIP_THREADS = 256        # the norm's reduction tree (ssd3d_grad_clip_scale)


def _tree(s):
    """Halving tree over the last axis (width 256): s[:, t] += s[:, t + w] for w = 128, 64, ..., 1."""
    s = np.array(s, dtype=np.float64, copy=True)
    w = s.shape[-1] // 2
    while w:
        s[..., :w] = s[..., :w] + s[..., w:2 * w]
        w //= 2
    return s[..., 0]


def sumsq_tree(g):
    """sum g^2 in double in the order of the kernel: thread t of block b adds g[i]^2 for i = b*256 + t + k*65536 in
    index order, then a halving tree inside each block, then the same tree over the 256 block partials."""
    g = np.asarray(g, dtype=np.float32).reshape(-1).astype(np.float64)
    span = CLIP_BLOCKS * CLIP_THREADS
    rows = max(1, -(-g.size // span))
    sq = np.zeros(rows * span, dtype=np.float64)
    sq[: g.size] = g * g
    sq = sq.reshape(rows, span)
    acc = np.zeros(span, dtype=np.float64)
    for r in range(rows):
        acc = acc + sq[r]
    return float(_tree(_tree(acc.reshape(CLIP_BLOCKS, CLIP_THREADS))[None, :])[0])


def clip_scale(g, clip=5.0):
    """(norm, scale) of one rank's flat gradient as float32 scalars, TF 1.4's float32 clip_by_global_norm."""
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        norm = np.float32(np.sqrt(sumsq_tree(g)))
        use = norm if np.isfinite(norm) else np.float32(np.nan)
        inv = np.float32(1.0) / use
        cap = np.float32(1.0) / np.float32(clip)
        scale = np.float32(clip) * np.minimum(inv, cap)          # np.minimum propagates NaN, like tf.minimum
    return np.float32(norm), np.float32(scale)


def allreduce_mean(grads, scales):
    """float32 mean over the ranks of rn(g_r * scale_r), summed in double in rank order, one division, one rounding."""
    with np.errstate(over="ignore", invalid="ignore"):
        acc = None
        for g, s in zip(grads, scales):
            c = (np.asarray(g, dtype=np.float32) * np.float32(s)).astype(np.float64)
            acc = c if acc is None else acc + c
        return (acc / float(len(grads))).astype(np.float32)


def bn_update(stats, batches, decay):
    """The moving-statistics update of bn.cu applied for every rank's batch statistics, in rank order."""
    om = np.float32(1.0) - np.float32(decay)
    v = np.array(stats, dtype=np.float32, copy=True)
    for b in batches:
        v = v - (v - np.asarray(b, dtype=np.float32)) * om
    return v.astype(np.float32)


def loss_mean(losses):
    """Per-name mean over ranks: losses [G, k] -> [k], summed in double in rank order."""
    losses = np.asarray(losses, dtype=np.float32)
    acc = losses[0].astype(np.float64)
    for r in range(1, losses.shape[0]):
        acc = acc + losses[r].astype(np.float64)
    return (acc / float(losses.shape[0])).astype(np.float32)


def exchange(grads, records, stats, decay, clip=5.0):
    """One step's exchange: per-rank gradients and BN records -> (mean gradient, new moving statistics, norms, scales)."""
    ns = [clip_scale(g, clip) for g in grads]
    norms = np.array([n for n, _ in ns], dtype=np.float32)
    scales = np.array([s for _, s in ns], dtype=np.float32)
    return allreduce_mean(grads, scales), bn_update(stats, records, decay), norms, scales
