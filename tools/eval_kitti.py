"""Evaluate a set of weights on KITTI the way the reference's evaluator does (lib/core/evaluator.py,
kitti_dataloader.py:336-437): run the inference network over preprocessed sample dicts in batches, build the
evaluator's detection rows, evaluate them against the label_2 files on the GPU, and print the precision_image /
precision_ground / precision_3d R40 tables as logger_and_select_best_map logs them.

    python tools/eval_kitti.py --samples <dir of .npy sample dicts> --labels <label_2 dir> --weights weights.npz

weights.npz: the reference checkpoint exported as INTEGRATION.md section D shows (TF variable name -> array).

--model pointrcnn runs PointRCNN's two-stage detector (tiny_pointrcnn_stage2_test.yaml, 3dssd_b200.PointRCNN) through the
same evaluator and AP tables; its weights are a full stage-2 checkpoint (rpn_*, roi_pool, rcnn_* variables).

--model pointrcnn-rpn runs PointRCNN's first stage (tiny_pointrcnn_stage1.yaml, TEST_MODE 'Recall') instead and prints
the proposal recall of evaluation.recall against each sample's label boxes.  As the reference's evaluator does
(lib/core/evaluator.py:116 -> kitti_dataloader.py:385), --cls-thresh is the recall's 3D-IoU threshold there.
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
    ap.add_argument("--cls-thresh", type=float, default=0.3, help="score threshold of the detection rows (evaluator.py:26); the recall's 3D-IoU threshold with --model pointrcnn-rpn")
    ap.add_argument("--classes", default="Car", help="comma-separated class list of the model")
    ap.add_argument("--model", default="3dssd", choices=("3dssd", "pointrcnn", "pointrcnn-rpn"))
    args = ap.parse_args(argv)
    pkg = importlib.import_module("3dssd_b200")
    try:
        cls_list = pkg.config.check_cls_list(args.classes)
    except ValueError as e:
        raise SystemExit("eval_kitti.py: --classes: %s" % e)

    import numpy as np
    import torch
    io, ev = pkg.kitti_io, pkg.evaluation
    if not torch.cuda.is_available():
        raise SystemExit("eval_kitti.py needs a CUDA device (there is no CPU path)")
    dev = torch.device("cuda", 0)
    paths = sorted(glob.glob(os.path.join(args.samples, "*.npy")))
    if not paths:
        raise SystemExit("no *.npy sample dicts under %s" % args.samples)
    weights = io.params_from_tf_variables(dict(np.load(args.weights)))
    if args.model == "3dssd":
        width = np.asarray(weights["pred_cls/weights"]).shape[-1] if "pred_cls/weights" in weights else None
        if width != len(cls_list):
            raise SystemExit("eval_kitti.py: the weights' pred_cls has %s class column(s), --classes names %d (%s)"
                             % (width, len(cls_list), ",".join(cls_list)))
    if args.model == "pointrcnn-rpn":
        return rpn_recall(pkg, args, paths, weights, dev)
    if args.model == "pointrcnn":
        rcnn = pkg.PointRCNN(params=weights, device=dev)
        detect = lambda pts: rcnn.forward(pts)
    else:
        head = pkg.DetectionHead(params=weights, device=dev, cls_num=len(cls_list))
        net = pkg.SABackbone(params=weights, in_channels=1, device=dev, head=head)
        detect = lambda pts: net.detections(*net.forward(pts)[:2])
    acc = ev.EvalAccumulator(cls_list=cls_list, cls_thresh=args.cls_thresh)
    for i in range(0, len(paths), args.batch):
        samples = [io.read_sample(p) for p in paths[i:i + args.batch]]
        points, calibs, names = io.make_batch(samples, args.num_points, seed=i)
        block, count = detect(points.to(dev, non_blocking=True))
        acc.add(block, count, calibs, [os.path.join(args.labels, "%06d.txt" % int(n)) for n in names])
    result = acc.evaluate(dev)
    print("evaluated %d frames" % len(acc))
    for line in ev.format_ap_tables([r.cpu().numpy() for r in result], cls_list):
        print(line)
    return 0


def rpn_recall(pkg, args, paths, weights, dev):
    """PointRCNN's RPN proposals (at most MAX_OUTPUT_NUM per frame after the IoU-0.85 NMS) against the label boxes."""
    import numpy as np
    import torch
    io, C = pkg.kitti_io, pkg.config
    head = pkg.DetectionHead(C.HEAD_POINTRCNN_RPN, weights, device=dev, stage=C.STAGE_POINTRCNN_RPN)
    net = pkg.SABackbone(C.ARCH_POINTRCNN_RPN, weights, in_channels=1, device=dev, head=head, aggregation=False)
    preds, gts = [], []
    for i in range(0, len(paths), args.batch):
        samples = [io.read_sample(p) for p in paths[i:i + args.batch]]
        points = io.make_batch(samples, args.num_points, seed=i)[0]
        xyz, feat = net.forward(points.to(dev, non_blocking=True))[:2]
        block, count = net.detections(xyz, feat)
        cnt = count.cpu().tolist()
        for s, smp in enumerate(samples):
            preds.append(block[s, :cnt[s], :7])
            gts.append(torch.from_numpy(np.asarray(smp[io.KEY_LABEL_BOXES_3D], np.float32).reshape(-1, 7)).to(dev))
    detected, total = pkg.evaluation.recall(preds, gts, args.cls_thresh)
    print("evaluated %d frames" % len(preds))
    print("recall: %d / %d = %.4f at 3D IoU %g" % (detected, total, detected / max(total, 1), args.cls_thresh))
    return 0


if __name__ == "__main__":
    sys.exit(main())
