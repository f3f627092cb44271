"""Training-scene augmentation of 3dssd.yaml on the GPU (DESIGN.md sections 3.12 and 3.13).

DataAugmentor.kitti_forward (lib/builder/data_augmentor.py:62-100) -- the mixup paste when a Mixup is given
(mixup.py), then flip, per-object noise, global rotation, global scale, the context filter -- followed by the choice
of the points the network sees (kitti_dataloader.py:137-147), on ragged scenes.  The kernels (csrc/augment.cu,
csrc/mixup.cu) are pure functions of the scenes, the drawn objects and a draw block, so the same draws give the same
bits; draw() fills one from a seeded torch.Generator on the device.  With mixup the draw block is sized for the pasted
layout (mixup.layout: rows and total).
"""
import collections

import numpy as np
import torch

from . import mixup as _mixup
from . import tf_ops

# configs/kitti/3dssd/3dssd.yaml over lib/core/config.py:82-109
FLIP = True
FLIP_PROB = 0.5
PROB = (0.5, 0.5, 0.5)                       # per-object noise, global rotation, global scale
EXPAND_DIMS_LENGTH = 0.1
ROTATION_PERTURB = (-np.pi / 3, np.pi / 3)
CENTER_NOISE_STD = (1.0, 1.0, 0.0)           # (x, z, y): no vertical noise
RANDOM_SCALE_RANGE_PER_OBJECT = (1.0, 1.0)
RANDOM_ROTATION_RANGE = 45 / 180 * np.pi
RANDOM_SCALE_RANGE = 0.1
FILTER_ENLARGE = (0.5, 2.0, 0.5)             # (l, h, w) of filter_points_boxes_3d
NUM_TRY = tf_ops.AUG_TRIES
POINTS_NUM_FOR_TRAINING = 16384

Draws = collections.namedtuple("Draws", "scene_u loc_noise rot_u keys refill")
Draws.__doc__ = """The randomness of one augmented batch, all on the device:
scene_u [B, 6] float64 uniforms (flip, c0, c1, c2, rotation, scale); loc_noise [B, G, 100, 2] float64 standard normals
(x, z) and rot_u [B, G, 100] float64 uniforms per box and try; keys [T] int32 (uint32 bits) per input point; refill
[B, num_points] int32 (uint32 bits) per output slot."""


def draw_seed(seed, step, rank=0):
    """The generator seed of one rank's batch at one step: every (seed, step, rank) gets its own stream."""
    return int(np.random.SeedSequence([int(seed), int(step), int(rank)]).generate_state(1, np.uint64)[0] >> 1)


def _u32(shape, gen, dev):
    return torch.randint(0, 1 << 32, shape, generator=gen, device=dev, dtype=torch.int64).to(torch.int32)


def draw(b, g, total_points, num_points=POINTS_NUM_FOR_TRAINING, generator=None, device="cuda"):
    """The draw block of b scenes with g GT rows, total_points input points and num_points output slots per scene."""
    dev = torch.device(device)
    if generator is None:
        generator = torch.Generator(device=dev)
        generator.seed()
    f64 = dict(generator=generator, device=dev, dtype=torch.float64)
    return Draws(torch.rand((b, 6), **f64), torch.randn((b, g, NUM_TRY, 2), **f64), torch.rand((b, g, NUM_TRY), **f64),
                 _u32((int(total_points),), generator, dev), _u32((b, int(num_points)), generator, dev))


def check_scenes(offsets, sem_labels=None, g=0):
    """Host checks before any launch: offsets [B + 1] (host) of scenes holding 1 .. 131072 points, at most 256 GT rows,
    non-negative semantic labels (host).  Returns the largest scene's point count."""
    off = np.asarray(offsets.cpu() if isinstance(offsets, torch.Tensor) else offsets, np.int64).reshape(-1)
    if off.size < 2 or off[0] != 0:
        raise ValueError("offsets must start at 0 and hold B + 1 >= 2 entries")
    n = np.diff(off)
    if n.min() < 1 or n.max() > tf_ops.AUG_MAX_POINTS:
        raise ValueError("every scene must hold 1 .. %d points, got %d .. %d" % (tf_ops.AUG_MAX_POINTS, n.min(), n.max()))
    if g > tf_ops.AUG_MAX_BOXES:
        raise ValueError("at most %d GT rows per scene, got %d" % (tf_ops.AUG_MAX_BOXES, g))
    if sem_labels is not None:
        if isinstance(sem_labels, torch.Tensor) and sem_labels.is_cuda:
            raise ValueError("sem_labels must be a host array (they are checked before the launch)")
        sem = np.asarray(sem_labels).reshape(-1)
        if sem.size != off[-1]:
            raise ValueError("sem_labels holds %d labels for %d points" % (sem.size, off[-1]))
        if sem.size and sem.min() < 0:
            raise ValueError("semantic labels must be >= 0")
    return int(n.max())


class Augmentor:
    """Augmentor(num_points)(points_packed [T, 4], offsets [B + 1], sem_labels [T] | None, gt_boxes [B, G, 7],
    gt_labels [B, G], draws) -> (block [B, num_points, 4], gt_boxes [B, G, 7], gt_labels [B, G]) on the device.

    offsets and sem_labels are host arrays (they are checked there); the rest may be host or device tensors.  Without
    sem_labels they are computed on the device from the boxes, as the reference's preprocessing does.  Padded GT rows
    (all zero) stay zero; boxes are never removed, so the shapes are kept.

    mixup (mixup.Mixup: database on the device, ids and planes on the host) pastes the drawn objects first, on the
    semantic labels of the original boxes; the stages after it run on the pasted layout, so the boxes and labels come
    back as [B, G + S, ...] and the draws must be sized for mixup.layout's rows and total slots."""

    def __init__(self, num_points=POINTS_NUM_FOR_TRAINING, device="cuda"):
        if not 1 <= int(num_points) <= tf_ops.AUG_MAX_CHOOSE:
            raise ValueError("num_points must be 1 .. %d, got %d" % (tf_ops.AUG_MAX_CHOOSE, num_points))
        self.num_points = int(num_points)
        self.device = torch.device(device)

    def _dev(self, t, dtype):
        return torch.as_tensor(t).to(self.device, dtype, non_blocking=True).contiguous()

    def __call__(self, points, offsets, sem_labels, gt_boxes, gt_labels, draws, debug=None, mixup=None):
        max_n = check_scenes(offsets, sem_labels, gt_boxes.shape[1])
        gt_boxes, gt_labels = self._dev(gt_boxes, torch.float32), self._dev(gt_labels, torch.int32)
        if draws.refill.shape[1] != self.num_points:
            raise ValueError("the draws are for %d points per scene, not %d" % (draws.refill.shape[1], self.num_points))
        pts, off = self._dev(points, torch.float32), self._dev(offsets, torch.int32)
        if sem_labels is None:
            sem = tf_ops.augment_sem_labels(pts, off, gt_boxes, gt_labels, max_n)
        else:
            sem = self._dev(sem_labels, torch.int32)
        if mixup is not None:
            m = _mixup.paste(mixup, pts, offsets, off, sem, gt_boxes, gt_labels)
            if debug is not None:
                debug.update(input_sem_labels=sem, pasted_points=m.points, pasted_boxes=m.boxes, accepted=m.accepted,
                             layout=m.layout)
            pts, off, sem, gt_boxes, gt_labels, max_n = m.points, m.offsets, m.sem_labels, m.boxes, m.labels, m.layout.max_slots
        boxes, chosen, ws = tf_ops.augment_boxes(gt_boxes, draws.scene_u, draws.loc_noise, draws.rot_u)
        moved_pts, keys, survivors, moved = tf_ops.augment_points(pts, off, max_n, sem, draws.keys, ws, gt_boxes.shape[1],
                                                                  want_moved=debug is not None)
        block = tf_ops.augment_choose(moved_pts, off, keys, survivors, draws.refill)
        if debug is not None:
            debug.update(sem_labels=sem, chosen_try=chosen, points=moved_pts, sort_keys=keys, survivors=survivors, moved_by=moved)
        return block, boxes, gt_labels
