"""Data-parallel training step of the 3DSSD backbone + head with the detection loss (dist.DataParallel): per rank
--batch scenes of --points points (synth.kitti_like_with_boxes), forward with the BN record, backward, exchange (clip,
rank-ordered allreduce mean, gather, BN update) and a torch.optim.Adam step.  Reports ms per step, the exchange's ms from
CUDA events around exchange(), and scenes/s over all ranks; prints the card name and power limit, asserts that no wait
timed out, and prints one JSON line (rank 0).

    python tools/train_dp.py --gpus 1 [--batch 4] [--points 16384] [--steps 5] [--warmup 2]
    torchrun --nproc_per_node G tools/train_dp.py --gpus G
"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("3dssd_b200")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--batch", type=int, default=4, help="scenes per rank (BATCH_SIZE of 3dssd.yaml)")
    ap.add_argument("--points", type=int, default=16384)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--max-boxes", type=int, default=40)
    ap.add_argument("--sync-bn", action="store_true",
                    help="normalise BatchNorm with the statistics of every GPU's scenes (MODEL.NETWORK.SYNC_BN)")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_dp.py measures on CUDA devices; none is available")
    D = pkg.dist
    rank, world, local = D.init_from_env()
    if world != a.gpus:
        raise SystemExit("--gpus %d but WORLD_SIZE is %d (launch G > 1 ranks with torchrun)" % (a.gpus, world))
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    card = torch.cuda.get_device_name(dev)
    try:
        power = subprocess.check_output(["nvidia-smi", "-i", str(local), "--query-gpu=power.limit,clocks.max.sm",
                                         "--format=csv,noheader"], text=True).strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        power = "unknown"
    arch = pkg.config.ARCH_3DSSD
    d = pkg.params.init_params(arch, 1, seed=0, random_bias=True)
    d.update(pkg.params.init_head_params(pkg.config.layer_channels(arch, 1)[-1], seed=1))
    tp = pkg.params.TrainableParams(d, dev)
    nbytes = D.DataParallel.symmetric_bytes(tp, world, sync_bn=a.sync_bn)
    if world > 1:
        dp = D.DataParallel(tp, D.PeerArena(nbytes, dev), sync_bn=a.sync_bn)
    else:
        sym = torch.zeros((nbytes,), dtype=torch.uint8, device=dev)
        dp = D.DataParallel(tp, peers=[sym.data_ptr()], world=1, rank=0, sync_bn=a.sync_bn)
    assert D.ALLREDUCE_CTAS <= pkg.tf_ops.peer_allreduce_resident_ctas()
    opt = torch.optim.Adam(tp.parameters(), lr=1e-3)
    synth = importlib.import_module("3dssd_b200.synth")
    p, b, l = synth.kitti_like_with_boxes(world * a.batch, a.points, a.max_boxes, seed=1)
    pts, boxes, labels = (D.shard_batch(torch.from_numpy(x), rank, world).to(dev) for x in (p, b, l))
    xyz, feat = pkg.tf_ops.split_points(pts)
    ev = []

    def step(timed):
        dp.zero_grad()
        with dp.recording():
            o = pkg.backbone.train_forward(arch, tp, xyz, feat)
        tg = pkg.loss.assign_targets(o.base_xyz, o.vote_base, boxes, labels)
        losses = pkg.loss.detection_loss(o.base_xyz, *o.head, o.vote_offsets[-1], tg)
        losses["total"].backward()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        mean = dp.exchange(losses)
        e.record()
        if timed:
            ev.append((s, e))
        opt.step()
        return mean

    for _ in range(a.warmup):
        step(False)
    torch.cuda.synchronize()
    s0, e0 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s0.record()
    for _ in range(a.steps):
        mean = step(True)
    e0.record()
    torch.cuda.synchronize()
    step_ms = s0.elapsed_time(e0) / a.steps
    ex_ms = sum(s.elapsed_time(e) for s, e in ev) / len(ev)
    timeouts = dp.timeouts()
    assert timeouts == 0, "%d exchange waits timed out" % timeouts
    if rank == 0:
        print("card: %s, power limit / max SM clock: %s" % (card, power))
        print(json.dumps({"card": card, "power_limit_max_sm_clock": power, "world": world, "scenes_per_rank": a.batch,
                          "points": a.points, "sync_bn": a.sync_bn, "step_ms": round(step_ms, 3), "exchange_ms": round(ex_ms, 4),
                          "scenes_per_s": round(world * a.batch / (step_ms * 1e-3), 2),
                          "grad_floats": dp.grad.numel(), "bn_stat_floats": dp.nstats, "timeouts": timeouts,
                          "total_loss": float(mean["total"])}))
    if world > 1:
        torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()
