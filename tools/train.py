"""Train the 3DSSD backbone + head with the reference's solver (solver.Trainer: scheduled BatchNorm decay, detection
loss, per-rank clip, rank-ordered gradient mean, TF-style Adam under the step-driven learning rate; DESIGN.md 3.11).

    python tools/train.py --steps N [--batch 4] [--gpus G] [--ckpt DIR] [--resume FILE] [--data DIR] [--augment]
    torchrun --nproc_per_node G tools/train.py --gpus G ...

Scenes are synth.kitti_like_with_boxes draws (a fresh seed every step) or, with --data, the reference's per-frame sample
dicts (*.npy, kitti_io.read_sample) taken in order, --batch per rank.  The losses are logged every --log-interval steps
(reading them synchronises; the steps in between do not), a checkpoint named model-<global_step>.npz is written to --ckpt
every Solver.checkpoint_interval steps and after the last one (rank 0), and --resume continues from such a file at its
step, learning rate and BatchNorm decay.

With --augment the scenes go through the reference's training augmentation on the GPU (augment.Augmentor: flip,
per-object noise, global rotation and scale, the context filter, then the choice of --points points), with draws seeded
from (--seed, step, rank); without it the points are chosen on the host and nothing is augmented.  --mixup DB.npz (an
object database of tools/build_mixup_db.py) adds the mixup paste before those stages: each scene draws 15 Car objects at
each step (mixup.Sampler, seeded from --seed, rank and the scene's place in the batch) and keeps those that collide with
nothing, standing on the frame's ground plane -- read from --planes DIR (<DIR>/%06d.txt per sample name) with --data,
the flat y = 1.65 plane of the synthetic scenes without it."""
import argparse
import glob
import importlib
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("3dssd_b200")
S = importlib.import_module("3dssd_b200.solver")
synth = importlib.import_module("3dssd_b200.synth")


def synthetic_batch(step, rank, world, batch, points, max_boxes):
    p, b, l = synth.kitti_like_with_boxes(world * batch, points, max_boxes, seed=1000 + step)
    return tuple(pkg.dist.shard_batch(torch.from_numpy(x), rank, world) for x in (p, b, l))


def file_batch(files, step, rank, world, batch, points):
    io = pkg.kitti_io
    first = (step * world + rank) * batch
    samples = [io.read_sample(files[(first + i) % len(files)]) for i in range(batch)]
    block, _, _ = io.make_batch(samples, num_points=points, seed=step)
    boxes, labels = io.make_label_batch(samples)
    return block, torch.from_numpy(boxes), torch.from_numpy(labels)


def synthetic_ragged(step, rank, world, batch, points, max_boxes):
    p, b, l = synthetic_batch(step, rank, world, batch, points, max_boxes)
    n = p.shape[0]
    offsets = torch.arange(0, (n + 1) * points, points, dtype=torch.int32)
    return p.reshape(-1, 4), offsets, None, b, l


def file_ragged(files, step, rank, world, batch):
    first = (step * world + rank) * batch
    samples = [pkg.kitti_io.read_sample(files[(first + i) % len(files)]) for i in range(batch)]
    return pkg.kitti_io.make_ragged_batch(samples), [s.get(pkg.kitti_io.KEY_SAMPLE_NAME, (first + i) % len(files))
                                                     for i, s in enumerate(samples)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, required=True, help="training steps to run in this invocation")
    ap.add_argument("--batch", type=int, default=4, help="scenes per rank (BATCH_SIZE of 3dssd.yaml)")
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--points", type=int, default=16384)
    ap.add_argument("--max-boxes", type=int, default=40, help="GT rows per synthetic scene")
    ap.add_argument("--ckpt", default=None, help="directory for checkpoints (none are written without it)")
    ap.add_argument("--resume", default=None, help="checkpoint to continue from (optimizer state and step included)")
    ap.add_argument("--warm-start", default=None, help="pre-trained variables to start from (model only, step 0)")
    ap.add_argument("--data", default=None, help="directory of the reference's per-frame sample dicts (*.npy)")
    ap.add_argument("--log-interval", type=int, default=10)
    ap.add_argument("--augment", action="store_true", help="augment the scenes on the GPU as the reference's training does")
    ap.add_argument("--seed", type=int, default=0, help="seed of the augmentation draws")
    ap.add_argument("--mixup", default=None, help="object database (.npz of tools/build_mixup_db.py): paste objects first")
    ap.add_argument("--planes", default=None, help="directory of the KITTI ground planes of --data (with --mixup)")
    a = ap.parse_args()
    if a.mixup and not a.augment:
        raise SystemExit("--mixup works with --augment")
    if a.mixup and a.data and not a.planes:
        raise SystemExit("--mixup with --data needs --planes DIR (the ground plane of every sample)")
    if not torch.cuda.is_available():
        raise SystemExit("train.py trains on CUDA devices; none is available (there is no CPU path)")
    D = pkg.dist
    rank, world, local = D.init_from_env()
    if world != a.gpus:
        raise SystemExit("--gpus %d but WORLD_SIZE is %d (launch G > 1 ranks with torchrun)" % (a.gpus, world))
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    arch, solver = pkg.config.ARCH_3DSSD, S.Solver()
    d = pkg.params.init_params(arch, 1, seed=0)
    d.update(pkg.params.init_head_params(pkg.config.layer_channels(arch, 1)[-1], seed=1))
    tp = pkg.params.TrainableParams(d, dev)
    dp = None
    if world > 1:
        dp = D.DataParallel(tp, D.PeerArena(D.DataParallel.symmetric_bytes(tp, world), dev), clip_norm=solver.clip_norm)
    tr = S.Trainer(arch, tp, solver, dp)
    if a.resume:
        tr.load(a.resume)
    elif a.warm_start:
        tr.warm_start(a.warm_start)
    files = None
    if a.data:
        files = sorted(glob.glob(os.path.join(a.data, "*.npy")))
        if not files:
            raise SystemExit("--data %s holds no *.npy sample" % a.data)
    log = (lambda *s: print(*s, flush=True)) if rank == 0 else (lambda *s: None)
    aug = pkg.augment.Augmentor(a.points, dev) if a.augment else None
    MX = pkg.mixup
    db = MX.ObjectDatabase.load(a.mixup, dev) if a.mixup else None
    sampler = MX.Sampler(db, seed=a.seed) if db is not None else None
    log("start at global_step %d: learning rate %.6g, bn decay %.6g, %d rank(s) x %d scenes"
        % (tr.global_step, solver.learning_rate(tr.global_step), solver.bn_decay(tr.global_step), world, a.batch))

    def save():
        if a.ckpt and rank == 0:
            os.makedirs(a.ckpt, exist_ok=True)
            path = os.path.join(a.ckpt, "model-%08d.npz" % tr.global_step)
            tr.save(path)
            log("Step %d, Checkpoint saved to %s" % (tr.global_step, path))

    last = time.time()
    for i in range(a.steps):
        step = tr.global_step
        if step >= solver.max_iterations:
            log("max_iterations %d reached" % solver.max_iterations)
            break
        if i and step % solver.checkpoint_interval == 0:
            save()
        if aug is not None:
            if files is None:
                cloud, offsets, sem, boxes, labels = synthetic_ragged(step, rank, world, a.batch, a.points, a.max_boxes)
                names = None
            else:
                (cloud, offsets, sem, boxes, labels), names = file_ragged(files, step, rank, world, a.batch)
            mix, rows, total = None, boxes.shape[1], cloud.shape[0]
            if sampler is not None:
                ids = sampler.ids(step, boxes.shape[0], rank)
                planes = (np.tile(np.asarray(MX.FLAT_PLANE, np.float64), (boxes.shape[0], 1)) if names is None else
                          np.stack([pkg.kitti_io.read_plane(pkg.kitti_io.plane_path(a.planes, n)) for n in names]))
                mix = MX.Mixup(db, ids, planes)
                lay = MX.layout(offsets, ids, db.host_offsets, boxes.shape[1])
                rows, total = lay.rows, lay.total
            gen = torch.Generator(device=dev).manual_seed(pkg.augment.draw_seed(a.seed, step, rank))
            draws = pkg.augment.draw(boxes.shape[0], rows, total, a.points, gen, dev)
            pts, boxes, labels = aug(cloud, offsets, sem, boxes, labels, draws, mixup=mix)
        elif files is None:
            pts, boxes, labels = synthetic_batch(step, rank, world, a.batch, a.points, a.max_boxes)
        else:
            pts, boxes, labels = file_batch(files, step, rank, world, a.batch, a.points)
        xyz, feat = pkg.tf_ops.split_points(pts.to(dev, non_blocking=True))
        losses = tr.step(xyz, feat, boxes.to(dev), labels.to(dev))
        if step % a.log_interval == 0 or i == a.steps - 1:
            vals = {k: float(v) for k, v in losses.items()}              # the one host read: synchronises
            now = time.time()
            log("**** STEP %08d ****" % step)
            log("Step %d, Total Loss %.3f, lr %.6g, bn decay %.6g, Time Elapsed %.3f s"
                % (step, vals["total"], solver.learning_rate(step), solver.bn_decay(step), now - last))
            for k in pkg.loss.LOSS_NAMES:
                log("Loss: %s: %.3f" % (k, vals[k]))
            if not np.isfinite(vals["total"]):
                raise SystemExit("the loss is not finite at step %d" % step)
            last = now
    save()
    timeouts = tr.dp.timeouts()
    if timeouts:
        raise SystemExit("%d exchange waits timed out" % timeouts)
    if world > 1:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
