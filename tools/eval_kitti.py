"""Evaluate a set of weights on KITTI the way the reference's evaluator does (lib/core/evaluator.py,
kitti_dataloader.py:336-437): run the inference network over preprocessed sample dicts in batches, build the
evaluator's detection rows, evaluate them against the label_2 files on the GPU, and print the precision_image /
precision_ground / precision_3d R40 tables as logger_and_select_best_map logs them.

    python tools/eval_kitti.py --samples <dir of .npy sample dicts> --labels <label_2 dir> --weights weights.npz

weights.npz: the reference checkpoint exported as INTEGRATION.md section D shows (TF variable name -> array).
"""
import argparse
import glob
import importlib
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--samples", required=True, help="directory of preprocessed sample dicts (*.npy)")
    ap.add_argument("--labels", required=True, help="KITTI label_2 directory (%%06d.txt per sample name)")
    ap.add_argument("--weights", required=True, help=".npz of TF variable name -> array")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--num-points", type=int, default=16384)
    ap.add_argument("--cls-thresh", type=float, default=0.3, help="score threshold of the detection rows (evaluator.py:26)")
    ap.add_argument("--classes", default="Car", help="comma-separated class list of the model")
    args = ap.parse_args(argv)

    import numpy as np
    import torch
    pkg = importlib.import_module("3dssd_b200")
    io, ev = pkg.kitti_io, pkg.evaluation
    if not torch.cuda.is_available():
        raise SystemExit("eval_kitti.py needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda", 0)
    paths = sorted(glob.glob(os.path.join(args.samples, "*.npy")))
    if not paths:
        raise SystemExit("no *.npy sample dicts under %s" % args.samples)
    weights = io.params_from_tf_variables(dict(np.load(args.weights)))
    head = pkg.DetectionHead(params=weights, device=dev)
    net = pkg.SABackbone(params=weights, in_channels=1, device=dev, head=head)
    cls_list = tuple(c.strip() for c in args.classes.split(","))
    acc = ev.EvalAccumulator(cls_list=cls_list, cls_thresh=args.cls_thresh)
    for i in range(0, len(paths), args.batch):
        samples = [io.read_sample(p) for p in paths[i:i + args.batch]]
        points, calibs, names = io.make_batch(samples, args.num_points, seed=i)
        xyz, feat = net.forward(points.to(dev, non_blocking=True))[:2]
        block, count = net.detections(xyz, feat)
        acc.add(block, count, calibs, [os.path.join(args.labels, "%06d.txt" % int(n)) for n in names])
    result = acc.evaluate(dev)
    print("evaluated %d frames" % len(acc))
    for line in ev.format_ap_tables([r.cpu().numpy() for r in result], cls_list):
        print(line)
    return 0


if __name__ == "__main__":
    sys.exit(main())
