"""The reference's KITTI preprocessing pass on the GPU (DESIGN.md section 3.14).

KittiDataset.preprocess_batch (kitti_dataloader.py:173-323) turns a raw KITTI tree (velodyne/, calib/, label_2/,
image_2/) and a list file into one sample dict per frame, the files every data path here reads (kitti_io.read_sample).
Per batch of frames:
  read      velodyne, calibration, labels and the PNG size of each frame on the host, into pinned buffers
  kernel    tf_ops.prepare_points: velo -> rect, the image-FOV and extents filters, the ordered compaction (float64)
  labels    tf_ops.augment_sem_labels on the float32 cast, with the boxes padded as kitti_io.make_label_batch pads them
  sync      one host read per batch: the kept offsets and labels, for the two skip rules (no object of the class list;
            no point with a positive semantic label)
  write     '%06d.npy' % (position in the list) and its line of train_list.txt; with a database, the mixup objects of
            the written frames (mixup.ObjectDatabase.build on the device-resident kept points)
"""
import collections
import os

import numpy as np
import torch

from . import kitti_io as io
from . import mixup as _mixup
from . import tf_ops

BATCH = 32
Frame = collections.namedtuple("Frame", "position name points calib hw boxes classes")
Frame.__doc__ = """One raw frame as read: its position in the list, KITTI id, points [N, 4] float32, calibration block [33]
float64 (kitti_io.calib_block), image (H, W), boxes [G, 7] float64 and classes [G] int64 (None without GT)."""
Stats = collections.namedtuple("Stats", "read kept no_objects no_points points_read points_kept")


def read_list(path):
    """The KITTI ids of a list file (train.txt / val.txt / test.txt), one per line, in order."""
    with open(path) as fh:
        ids = [ln.strip() for ln in fh]
    ids = [s for s in ids if s]
    try:
        return [int(s) for s in ids]
    except ValueError:
        raise ValueError("%s: every line of a list file is a KITTI id" % path) from None


def read_frame(split_dir, position, name, cls_list=None):
    """Frame `name` of a split directory (training/ or testing/); labels only when cls_list is given."""
    f = "%06d" % int(name)
    pts = io.read_velodyne(os.path.join(split_dir, "velodyne", f + ".bin"))
    calib = io.calib_block(io.read_calib(os.path.join(split_dir, "calib", f + ".txt")))
    hw = io.png_size(os.path.join(split_dir, "image_2", f + ".png"))
    boxes = classes = None
    if cls_list is not None:
        boxes, classes = io.read_label(os.path.join(split_dir, "label_2", f + ".txt"), tuple(cls_list))
    return Frame(position, int(name), pts, calib, hw, boxes, classes)


def _pinned(a, dev):
    t = torch.from_numpy(np.ascontiguousarray(a))
    return t.pin_memory() if dev.type == "cuda" else t


def run_batch(frames, device="cuda", with_db=False, db_classes=_mixup.CLASS_INDEX):
    """Preprocess a batch of read frames -> (list of (position, sample dict) to write, skipped {position: reason},
    ObjectDatabase of the written frames (frames = their positions) or None).  db_classes: the labels whose rows become
    database objects (label k = the k-th class of the frames' class list)."""
    dev = torch.device(device)
    gt = frames[0].boxes is not None
    sizes = [len(f.points) for f in frames]
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    pts = _pinned(np.concatenate([f.points for f in frames]) if off[-1] else np.zeros((0, 4), np.float32), dev)
    calib = _pinned(np.stack([f.calib for f in frames]), dev)
    hw = np.asarray([f.hw for f in frames], np.int64)
    kept, kept_off = tf_ops.prepare_points(pts.to(dev, non_blocking=True), off, calib.to(dev, non_blocking=True), hw)
    sem = boxes = labels = None
    if gt:
        boxes, labels = io.make_label_batch([{io.KEY_LABEL_BOXES_3D: f.boxes, io.KEY_LABEL_CLASSES: f.classes} for f in frames])
        max_n = min(int(max(sizes)), tf_ops.AUG_MAX_POINTS)
        if boxes.shape[1] and max_n:
            sem = tf_ops.augment_sem_labels(kept.float(), kept_off, _pinned(boxes, dev).to(dev, non_blocking=True),
                                            _pinned(labels, dev).to(dev, non_blocking=True), max_n)
    # the one host synchronisation of the batch
    k_off = kept_off.cpu().numpy().astype(np.int64)
    total = int(k_off[-1])
    host_pts = kept[:total].cpu().numpy()
    host_sem = sem[:total].cpu().numpy().astype(np.int64) if sem is not None else None
    n_kept = np.diff(k_off)
    if gt and n_kept.max(initial=0) > tf_ops.AUG_MAX_POINTS:
        raise ValueError("a frame keeps %d points; the semantic labels take at most %d" % (n_kept.max(), tf_ops.AUG_MAX_POINTS))
    out, skipped = [], {}
    for s, f in enumerate(frames):
        a, b = k_off[s], k_off[s + 1]
        if gt and len(f.boxes) == 0:
            skipped[f.position] = "no_objects"
            continue
        lab = host_sem[a:b] if gt else np.ones(b - a, np.int64)
        if lab.sum() == 0:
            skipped[f.position] = "no_points"
            continue
        d = {io.KEY_POINT_CLOUD: host_pts[a:b], io.KEY_LABEL_SEM_SEG: lab, io.KEY_LABEL_DIST: np.ones(b - a, np.float32),
             io.KEY_STEREO_CALIB: f.calib[21:].reshape(3, 4).copy(), io.KEY_SAMPLE_NAME: f.name}
        if gt:
            d.update({io.KEY_LABEL_BOXES_3D: f.boxes, io.KEY_LABEL_CLASSES: f.classes, io.KEY_LABEL_NUM: len(f.boxes)})
        out.append((s, d))
    db = None
    if with_db and gt and out:
        rows = [s for s, _ in out]
        if len(rows) == len(frames):
            dpts, doff, sel = kept[:total].float(), k_off, slice(None)
        else:
            dpts = torch.cat([kept[k_off[s]:k_off[s + 1]] for s in rows]).float()
            doff = np.concatenate([[0], np.cumsum(n_kept[rows])])
            sel = rows
        db = _mixup.ObjectDatabase.build(dpts, doff, boxes[sel], labels[sel], classes=db_classes, device=dev)
        pos = torch.as_tensor(np.asarray([frames[s].position for s in rows], np.int32), device=db.frames.device)
        db.frames = pos[db.frames.long()] if len(db) else db.frames
    return [(frames[s].position, d) for s, d in out], skipped, db


def write_sample(out_dir, position, d):
    path = os.path.join(out_dir, "%06d.npy" % position)
    np.save(path, np.array(d, dtype=object), allow_pickle=True)
    return path
