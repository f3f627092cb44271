"""Preprocess a raw KITTI tree into the per-frame sample files every data path here reads (prepare.py, DESIGN.md section
3.14), as the reference's preprocessing pass does (KittiDataset.preprocess_batch), with the per-point work on the GPU.

    python tools/prepare_kitti.py --root <KITTI/object> --split training|testing --list val.txt --out DIR
                                  [--classes Car] [--no-gt] [--mixup-db DB.npz] [--batch 32]

For the i-th id of --list it writes DIR/%06d.npy % i (the list position; the KITTI id is the sample's sample_name) and
appends that name to DIR/train_list.txt, unless the frame is skipped: with labels, when no object of --classes is in it
or when none of its kept points lies in such an object.  --split testing or --no-gt writes samples without labels.
--mixup-db also writes the mixup object database of the written frames (mixup.ObjectDatabase, read by
tools/train.py --mixup), each object's `frames` entry being the number of its sample file.  The next batch is read on a
worker thread while the GPU works on the current one.  Prints frames read, kept and skipped by reason, points kept and
the time spent reading, on the GPU and writing."""
import argparse
import concurrent.futures
import importlib
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("3dssd_b200")
PR = importlib.import_module("3dssd_b200.prepare")


def run(root, split, list_path, out, classes=("Car",), gt=True, mixup_db=None, batch=PR.BATCH, device="cuda", log=print):
    """The whole pass; returns a dict of counts and seconds (read, gpu, write)."""
    split_dir = os.path.join(root, split)
    ids = PR.read_list(list_path)
    gt = gt and split == "training"
    if mixup_db and not gt:
        raise SystemExit("--mixup-db needs labelled frames (--split training without --no-gt)")
    os.makedirs(out, exist_ok=True)
    cls = tuple(classes) if gt else None
    read = lambda first: [PR.read_frame(split_dir, first + k, ids[first + k], cls) for k in range(min(batch, len(ids) - first))]
    st = dict(read=0, kept=0, no_objects=0, no_points=0, points_read=0, points_kept=0, t_read=0.0, t_gpu=0.0, t_write=0.0)
    dbs = []
    with open(os.path.join(out, "train_list.txt"), "w") as lst, concurrent.futures.ThreadPoolExecutor(1) as pool:
        t0 = time.perf_counter()
        nxt = pool.submit(read, 0) if ids else None
        for first in range(0, len(ids), batch):
            frames = nxt.result()
            t1 = time.perf_counter()
            st["t_read"] += t1 - t0
            nxt = pool.submit(read, first + batch) if first + batch < len(ids) else None
            written, skipped, db = PR.run_batch(frames, device, with_db=bool(mixup_db))
            t2 = time.perf_counter()
            st["t_gpu"] += t2 - t1
            for pos, d in written:
                PR.write_sample(out, pos, d)
                lst.write("%06d.npy\n" % pos)
                st["points_kept"] += len(d[pkg.kitti_io.KEY_POINT_CLOUD])
            if db is not None:
                dbs.append(db)
            st["read"] += len(frames)
            st["points_read"] += sum(len(f.points) for f in frames)
            st["kept"] += len(written)
            for why in skipped.values():
                st[why] += 1
            t0 = time.perf_counter()
            st["t_write"] += t0 - t2
    if mixup_db:
        db = pkg.mixup.ObjectDatabase.concat(dbs)
        db.save(mixup_db)
        st["objects"] = len(db)
        log("mixup database: %d objects, %d points -> %s" % (len(db), int(db.host_offsets[-1]), mixup_db))
    log("frames read %d, kept %d, skipped %d (no object of %s: %d, no point in an object: %d); points read %d, kept %d"
        % (st["read"], st["kept"], st["no_objects"] + st["no_points"], ",".join(classes), st["no_objects"], st["no_points"],
           st["points_read"], st["points_kept"]))
    log("time: read %.3f s (waited for), gpu %.3f s, write %.3f s" % (st["t_read"], st["t_gpu"], st["t_write"]))
    return st


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--root", required=True, help="KITTI object directory holding training/ and testing/")
    ap.add_argument("--split", default="training", choices=("training", "testing"))
    ap.add_argument("--list", required=True, help="list file of KITTI ids (train.txt, val.txt, test.txt)")
    ap.add_argument("--out", required=True, help="output directory of the sample files and train_list.txt")
    ap.add_argument("--classes", default="Car", help="comma-separated class list (CLS_LIST)")
    ap.add_argument("--no-gt", action="store_true", help="write samples without labels (as for the test list)")
    ap.add_argument("--mixup-db", default=None, help="also write the mixup object database of the written frames (.npz)")
    ap.add_argument("--batch", type=int, default=PR.BATCH, help="frames per GPU batch")
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("prepare_kitti.py runs the filters on a CUDA device; none is available (there is no CPU path)")
    if a.batch < 1:
        raise SystemExit("--batch must be at least 1")
    run(a.root, a.split, a.list, a.out, tuple(c.strip() for c in a.classes.split(",")), not a.no_gt, a.mixup_db, a.batch,
        torch.device("cuda", 0))
    return 0


if __name__ == "__main__":
    sys.exit(main())
