"""The mixup paste of 3dssd.yaml on the GPU (DESIGN.md section 3.13).

MIXUP.OPEN pastes objects of other frames into each training scene before any other augmentation
(DataAugmentor.kitti_mixup_sampling, lib/builder/data_augmentor.py:104-119): 15 Car objects are drawn from an object
database, every drawn object whose enlarged BEV box collides with a box already in the scene is dropped
(box_3d_collision_test, voxelnet_aug.py:197-248), and each object kept is put on the frame's ground plane and appended
with its points.

  ObjectDatabase  the objects of a set of frames (generate_mixup_sample, kitti_dataloader.py:258-287), built on the GPU
  Sampler         which objects each scene draws at a step (MixupSampler._sample / _reset), stateless
  layout          the host plan of the pasted clouds: every scene's output slots, sized before any launch
  paste           the two paste kernels (csrc/mixup.cu) on a batch of ragged scenes
Augmentor (augment.py) takes a Mixup(db, ids, planes) and runs the paste before its own stages.
"""
import collections
import math

import numpy as np
import torch

from . import tf_ops

# configs/kitti/3dssd/3dssd.yaml:14-19 over lib/core/config.py
CLASSES = ("Car",)                   # MIXUP.CLASS
NUMBER = (15,)                       # MIXUP.NUMBER
CLASS_INDEX = (1,)                   # cls2idx_dict: index in cls_list + 1
EXPAND_DIMS_LENGTH = 0.1             # the grown box whose points an object keeps
MIN_POINTS_NUM = 5                   # DATASET.MIN_POINTS_NUM
COLLISION_ENLARGE = (0.5, 2.0, 0.5)  # (l, h, w) of box_3d_collision_test
FLAT_PLANE = (0.0, -1.0, 0.0, 1.65)  # the ground plane of synth.kitti_like scenes (y = 1.65)

Mixup = collections.namedtuple("Mixup", "db ids planes")
Mixup.__doc__ = """The mixup input of Augmentor: db an ObjectDatabase on the device, ids [B, S] int32 (host) database rows
drawn per scene (-1: none), planes [B, 4] float64 (host) ground plane (a, b, c, d) of each scene."""

Layout = collections.namedtuple("Layout", "offsets slot_start rows total max_slots")
Layout.__doc__ = """The pasted clouds, known on the host before any launch: offsets [B + 1] int32 of the output slots,
slot_start [B, S + 1] int32 (scene b's drawn object i owns slots slot_start[b, i] .. slot_start[b, i+1]-1 within the scene,
slot_start[b, 0] = its own point count), rows = G + S boxes per scene, total = the slots of the batch, max_slots = the
largest scene.  Size the augmentation's draw block with rows and total."""


def _host(a, dtype=None):
    if isinstance(a, torch.Tensor):
        if a.is_cuda:
            raise ValueError("expected a host array, got a CUDA tensor")
        a = a.numpy()
    return np.asarray(a) if dtype is None else np.asarray(a, dtype)


class ObjectDatabase:
    """The mixup objects: points [P, 4] float32, offsets [O + 1] int64 (object o holds points offsets[o] .. offsets[o+1]-1;
    host_offsets is its host copy), boxes [O, 7] float32, classes [O] int32, frames [O] and rows [O] int32 (where each
    object comes from).  Objects are ordered by frame, then by row."""

    FIELDS = ("points", "offsets", "boxes", "classes", "frames", "rows")

    def __init__(self, points, offsets, boxes, classes, frames, rows):
        self.points, self.offsets, self.boxes, self.classes, self.frames, self.rows = points, offsets, boxes, classes, frames, rows
        self.host_offsets = _host(offsets.cpu() if isinstance(offsets, torch.Tensor) else offsets, np.int64)

    def __len__(self):
        return int(self.boxes.shape[0])

    @property
    def device(self):
        return self.points.device

    def to(self, device):
        dev = torch.device(device)
        db = ObjectDatabase(*(getattr(self, k).to(dev) for k in self.FIELDS))
        db.host_offsets = self.host_offsets
        return db

    def class_ids(self, cls):
        """The database rows of class index cls, in database order."""
        return np.flatnonzero(_host(self.classes.cpu()) == int(cls)).astype(np.int64)

    def save(self, path):
        np.savez(path, **{k: getattr(self, k).cpu().numpy() for k in self.FIELDS})

    @classmethod
    def load(cls, path, device="cpu"):
        with np.load(path) as z:
            return cls(*(torch.from_numpy(np.ascontiguousarray(z[k])) for k in cls.FIELDS)).to(device)

    @classmethod
    def empty(cls, device="cpu"):
        i32 = lambda *s: torch.zeros(s, dtype=torch.int32)
        return cls(torch.zeros((0, 4)), torch.zeros(1, dtype=torch.int64), torch.zeros((0, 7)), i32(0), i32(0), i32(0)).to(device)

    @classmethod
    def concat(cls, dbs):
        """One database of several (in the given order)."""
        dbs = [d.to("cpu") for d in dbs]
        if not dbs:
            return cls.empty()
        off = [np.zeros(1, np.int64)]
        base = 0
        for d in dbs:
            off.append(d.host_offsets[1:] + base)
            base += int(d.host_offsets[-1])
        cat = lambda k: torch.cat([getattr(d, k) for d in dbs])
        return cls(cat("points"), torch.from_numpy(np.concatenate(off)), cat("boxes"), cat("classes"), cat("frames"), cat("rows"))

    @classmethod
    def build(cls, points, offsets, gt_boxes, gt_labels, classes=CLASS_INDEX, min_points=MIN_POINTS_NUM, frame_base=0,
              device="cuda"):
        """generate_mixup_sample over a batch of ragged frames (points [T, 4], offsets [B + 1] host, gt_boxes [B, G, 7],
        gt_labels [B, G]): every valid row of a class in `classes` holding at least min_points points of its frame inside
        the row grown by 0.1 on (l, h, w) becomes an object with those points, in frame order.  The frames are numbered
        from frame_base.  One host synchronisation between the counting and the writing pass."""
        from . import augment
        dev = torch.device(device)
        off = _host(offsets, np.int64).reshape(-1)
        max_n = augment.check_scenes(off, None, gt_boxes.shape[1])
        boxes = _host(gt_boxes, np.float32)
        labels = _host(gt_labels, np.int32)
        b, g = boxes.shape[:2]
        if g == 0:
            return cls.empty(dev)
        pts = torch.as_tensor(points).to(dev, torch.float32).contiguous()
        doff = torch.from_numpy(off.astype(np.int32)).to(dev)
        dboxes = torch.from_numpy(np.ascontiguousarray(boxes)).to(dev)
        counts = tf_ops.mixup_db_count(pts, doff, max_n, dboxes).cpu().numpy()
        keep = np.any(boxes != 0, -1) & np.isin(labels, np.asarray(classes, np.int32)) & (counts >= int(min_points))
        frames, rows = np.nonzero(keep)                                   # row-major: by frame, then by row
        if frames.size == 0:
            return cls.empty(dev)
        obj_off = np.concatenate([[0], np.cumsum(counts[frames, rows])]).astype(np.int64)
        objects = torch.from_numpy(np.stack([frames, rows], 1).astype(np.int32)).to(dev)
        dpts = tf_ops.mixup_db_write(pts, doff, dboxes, objects, torch.from_numpy(obj_off).to(dev), int(obj_off[-1]))
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        db = cls(dpts, t(obj_off), t(boxes[frames, rows]), t(labels[frames, rows]), t((frames + frame_base).astype(np.int32)),
                 t(rows.astype(np.int32)))
        db.host_offsets = obj_off
        return db


class Sampler:
    """MixupSampler._sample / _reset without state.  Each class walks a shuffled permutation of its objects `num` at a
    time; a call whose cursor + num reaches the count returns the tail and the next call starts a new permutation, so an
    epoch is E = ceil(count / num) calls and the last returns fewer.  Call k of a stream is epoch k // E at position
    k % E, and epoch e's permutation is seeded from (seed, rank, slot, class, e), slot being the scene's place in the
    rank's batch (the reference keeps one sampler per loader worker).  The step is the call index, so a resumed run
    draws the same objects without any saved state."""

    def __init__(self, db, seed=0, classes=CLASS_INDEX, numbers=NUMBER):
        self.seed, self.classes, self.numbers = int(seed), tuple(int(c) for c in classes), tuple(int(n) for n in numbers)
        self.members = [db.class_ids(c) for c in self.classes]

    @property
    def width(self):
        return sum(self.numbers)

    @staticmethod
    def cursor(count, num, k):
        """(epoch, start, stop) of call k over a class of `count` objects drawn `num` at a time."""
        e = int(math.ceil(count / num))
        epoch, pos = divmod(int(k), e)
        start = pos * num
        return epoch, start, min(start + num, count)

    def permutation(self, rank, slot, cls_pos, epoch):
        n = len(self.members[cls_pos])
        ss = np.random.SeedSequence([self.seed, int(rank), int(slot), self.classes[cls_pos], int(epoch)])
        return np.random.default_rng(ss).permutation(n)

    def ids(self, step, batch, rank=0):
        """[batch, S] int32 database rows drawn at `step` by each scene of the rank's batch, -1 past a class's draw."""
        out = np.full((int(batch), self.width), -1, np.int32)
        for slot in range(int(batch)):
            col = 0
            for c, num in enumerate(self.numbers):
                count = len(self.members[c])
                if count:
                    epoch, a, b = self.cursor(count, num, step)
                    out[slot, col:col + b - a] = self.members[c][self.permutation(rank, slot, c, epoch)[a:b]]
                col += num
        return out


def check_planes(planes, b):
    """[b, 4] float64 host planes with finite values and b != 0 (the height solves for y)."""
    pl = _host(planes, np.float64)
    if pl.shape != (b, 4):
        raise ValueError("planes must be [%d, 4], got %s" % (b, pl.shape))
    if not np.isfinite(pl).all() or (pl[:, 1] == 0).any():
        raise ValueError("every plane must be finite with b != 0")
    return pl


def layout(offsets, ids, db_offsets, g):
    """The host plan of the pasted clouds (Layout) from the scenes' offsets [B + 1], the ids [B, S] and the database's host
    offsets, with the checks made before any launch: ids in -1 .. O-1, G + S <= 256, at most 131072 slots per scene."""
    off = _host(offsets, np.int64).reshape(-1)
    ids = _host(ids)
    dbo = _host(db_offsets, np.int64).reshape(-1)
    b = off.size - 1
    if ids.ndim != 2 or ids.shape[0] != b or ids.shape[1] < 1:
        raise ValueError("ids must be [%d, S >= 1], got %s" % (b, ids.shape))
    s = ids.shape[1]
    if g + s > tf_ops.MIXUP_MAX_ROWS:
        raise ValueError("GT rows plus drawn objects must be at most %d, got %d + %d" % (tf_ops.MIXUP_MAX_ROWS, g, s))
    if ids.size and (ids.min() < -1 or ids.max() >= dbo.size - 1):
        raise ValueError("ids must lie in -1 .. %d, got %d .. %d" % (dbo.size - 2, ids.min(), ids.max()))
    ids = ids.astype(np.int64)
    sizes = np.where(ids >= 0, dbo[np.maximum(ids, 0) + 1] - dbo[np.maximum(ids, 0)], 0)
    start = np.concatenate([np.diff(off)[:, None], sizes], 1).cumsum(1)
    slots = start[:, -1]
    if slots.max() > tf_ops.MIXUP_MAX_SLOTS:
        raise ValueError("a pasted scene holds %d slots, more than %d" % (slots.max(), tf_ops.MIXUP_MAX_SLOTS))
    out = np.concatenate([[0], np.cumsum(slots)]).astype(np.int32)
    return Layout(out, start.astype(np.int32), g + s, int(out[-1]), int(slots.max()))


def _upload(a, dev):
    t = torch.from_numpy(np.ascontiguousarray(a))
    if dev.type == "cuda":
        t = t.pin_memory()
    return t.to(dev, non_blocking=True)


Pasted = collections.namedtuple("Pasted", "points offsets sem_labels boxes labels accepted layout")


def paste(mix, points, offsets, dev_offsets, sem_labels, gt_boxes, gt_labels):
    """The paste of mix (Mixup) into device scenes: points [T, 4], offsets [B + 1] host and dev_offsets on the device,
    sem_labels [T] int32, gt_boxes [B, G, 7], gt_labels [B, G] -> Pasted (device tensors; offsets on the device, the
    layout on the host).  Nothing here synchronises the host."""
    lay = layout(offsets, mix.ids, mix.db.host_offsets, gt_boxes.shape[1])
    dev = points.device
    planes = _upload(check_planes(mix.planes, lay.offsets.size - 1), dev)
    ids = _upload(_host(mix.ids, np.int32), dev)
    db = mix.db
    if len(db) == 0:                                                      # every id is -1: a stand-in row nobody reads
        db = ObjectDatabase(torch.zeros((1, 4), device=dev), torch.zeros(2, dtype=torch.int64, device=dev),
                            torch.zeros((1, 7), device=dev), *(torch.zeros(1, dtype=torch.int32, device=dev) for _ in range(3)))
        db.host_offsets = np.zeros(2, np.int64)
    boxes, labels, accepted = tf_ops.mixup_paste_boxes(gt_boxes, gt_labels, ids, db.boxes, db.classes, planes)
    out_off = _upload(lay.offsets, dev)
    pts, sem = tf_ops.mixup_paste_points(points, dev_offsets, sem_labels, ids, db.points, db.offsets, db.boxes, db.classes, planes,
                                         accepted, out_off, _upload(lay.slot_start, dev), lay.max_slots, lay.total)
    return Pasted(pts, out_off, sem, boxes, labels, accepted, lay)
