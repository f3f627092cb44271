"""KITTI evaluation of detections: label files, the evaluator's detection rows, R40 AP, recall, and an accumulator
for a validation loop (DESIGN.md section 3.10).

The numbers are those the reference logs and keeps its best checkpoint by (lib/core/evaluator.py,
lib/dataset/dataloader/kitti_dataloader.py:336-437): its Evaluate op (tf_ops.evaluate here, on the GPU) gives
41-point precision curves per class, difficulty and metric, and logger_and_select_best_map reduces them to R40 AP.

    acc = EvalAccumulator(cls_list=("Car",))
    for points, calibs, names in batches:
        block, count = net.detections(*net.forward(points))
        acc.add(block, count, calibs, [os.path.join(label_dir, "%06d.txt" % int(n)) for n in names])
    result = acc.evaluate()                      # the six (3, 3, 41) arrays
    print("\\n".join(format_ap_tables(result)))   # precision_image / ground / 3d R40 tables
"""
import numpy as np

from . import kitti_io

# Type names compare case-insensitively (evaluate.cpp:587-598, strcasecmp); everything else is code 6.
TYPE_CODES = {"car": 0, "pedestrian": 1, "cyclist": 2, "van": 3, "person_sitting": 4, "dontcare": 5}
TYPE_OTHER = 6
CLASS_NAMES = ("Car", "Pedestrian", "Cyclist")
N_SAMPLE = 41
CLS_THRESH = 0.3              # the reference evaluator's score threshold (lib/core/evaluator.py:26)


def read_label_file(path):
    """A KITTI label_2 file -> (rows, 15) float64: type code, truncation, occlusion, alpha, x1, y1, x2, y2, h, w, l,
    t1, t2, t3, ry -- the 15 fields evaluate.cpp:365-393 reads, parsed as doubles (occlusion as an integer).

    Unlike the reference's fscanf token stream, which silently misaligns on a short or long line, a non-blank line
    without exactly 15 fields raises ValueError naming the file and line."""
    rows = []
    with open(path) as fh:
        for ln, line in enumerate(fh, 1):
            tok = line.split()
            if not tok:
                continue
            if len(tok) != 15:
                raise ValueError("%s:%d: a KITTI label line has 15 fields, this one has %d" % (path, ln, len(tok)))
            try:
                occ = int(tok[2])
                vals = [float(t) for t in tok[1:]]
            except ValueError:
                raise ValueError("%s:%d: malformed label line %r" % (path, ln, line.rstrip("\n"))) from None
            rows.append([float(TYPE_CODES.get(tok[0].lower(), TYPE_OTHER)), vals[0], float(occ)] + vals[2:])
    return np.asarray(rows, np.float64).reshape(-1, 15)


def detection_rows(det_block, det_count, calibs, cls_list=("Car",), cls_thresh=CLS_THRESH,
                   img_shape=kitti_io.KITTI_IMG_SHAPE):
    """The evaluator's detection rows of a batch, as evaluate_map builds them (kitti_dataloader.py:342-372), from the
    NMS block (det_block [B, K, 9] = x, y, z, l, h, w, ry, score, class; det_count [B]) and each frame's P2.
    Rows scoring below cls_thresh are dropped; the class index is shifted by one when 'Car' is not in cls_list.
    Returns (rows (n, 14) float32 = class, x1, y1, x2, y2, alpha = 0, t1, t2, t3, h, w, l, ry, score;
    numlist (B,) int32)."""
    det_block = np.asarray(det_block.cpu() if hasattr(det_block, "cpu") else det_block, np.float32)
    det_count = np.asarray(det_count.cpu() if hasattr(det_count, "cpu") else det_count).reshape(-1)
    out, nums = [], []
    for i in range(det_block.shape[0]):
        d = det_block[i, :int(det_count[i])]
        d = d[np.where(d[:, 7] >= cls_thresh)[0]]
        rows = np.zeros((d.shape[0], 14), np.float32)
        cat = d[:, 8].astype(np.int64)
        if "Car" not in cls_list:
            cat = cat + 1
        rows[:, 0] = cat
        if d.shape[0]:
            rows[:, 1:5] = kitti_io.project_boxes_to_image(d[:, :7], kitti_io.calib_p2(calibs[i]), img_shape)
        rows[:, 6:9] = d[:, 0:3]
        rows[:, 9] = d[:, 4]          # h
        rows[:, 10] = d[:, 5]         # w
        rows[:, 11] = d[:, 3]         # l
        rows[:, 12] = d[:, 6]         # ry
        rows[:, 13] = d[:, 7]         # score
        out.append(rows)
        nums.append(d.shape[0])
    rows = np.concatenate(out, 0) if out else np.zeros((0, 14), np.float32)
    return rows, np.asarray(nums, np.int32)


# ---- host steps of the evaluator (the GPU runs the overlaps and both statistics passes) ----------------------------
def _det_class(v):
    return int(v) if -1 < v < 3 else 3


def eval_flags(rows):
    """[metric][class]: a class is evaluated in a metric only if one of its detections has the fields that metric
    needs (evaluate.cpp:316-331): image x1 >= 0; ground t1, t3 != -1000 and w, l > 0; 3-D also t2 != -1000, h > 0."""
    rows = np.asarray(rows, np.float32).reshape(-1, 14)
    cls = np.array([_det_class(v) for v in rows[:, 0]], np.int64)
    pos = lambda c: rows[:, c] > 0
    known = lambda c: rows[:, c] != -1000
    tests = (rows[:, 1] >= 0, known(6) & known(8) & pos(10) & pos(11),
             known(6) & known(7) & known(8) & pos(9) & pos(10) & pos(11))
    return [[bool(np.any(t & (cls == c))) for c in range(3)] for t in tests]


def get_thresholds(scores, n_gt):
    """getThresholds (evaluate.cpp:539-572) in float64: the true-positive scores, sorted descending, at which recall
    steps past each of the 41 sample points; at most 41 of them."""
    v = sorted((float(s) for s in scores), reverse=True)
    out, current, n = [], 0.0, float(n_gt)
    for i in range(len(v)):
        l_recall = (i + 1) / n
        r_recall = (i + 2) / n if i < len(v) - 1 else l_recall
        if (r_recall - current) < (current - l_recall) and i < len(v) - 1:
            continue
        out.append(v[i])
        current += 1.0 / (N_SAMPLE - 1.0)
    return out


def precision_curve(tp, fp, n_thresholds):
    """eval_class (evaluate.cpp:897-923): precision tp / (tp + fp) in float64 at each threshold, 0 beyond; then each
    point below n_thresholds takes the maximum from it to the end, as std::max_element does it (so a 0 / 0 point stays
    NaN like the reference's); rounded to float32 last."""
    p = np.zeros(N_SAMPLE, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        p[:n_thresholds] = np.asarray(tp[:n_thresholds], np.float64) / np.asarray(tp[:n_thresholds] + fp[:n_thresholds],
                                                                                   np.float64)
    res = p.copy()
    for i in range(n_thresholds):
        best = p[i]
        for x in p[i + 1:]:
            if best < x:
                best = x
        res[i] = best
    return res.astype(np.float32)


# ---- what the reference logs ---------------------------------------------------------------------------------------
def kitti_ap(precision):
    """R40 AP of (3, 3, 41) precision curves: sum(precision[..., 1:]) / 40 with numpy's float32 sum, as
    logger_and_select_best_map computes it (kitti_dataloader.py:415-429) -> (3, 3) float32."""
    p = np.asarray(precision.cpu() if hasattr(precision, "cpu") else precision, np.float32)
    return np.sum(p[:, :, 1:], axis=-1) / 40.


def select_metric(result, cls_list=("Car",)):
    """The number the reference keeps its best checkpoint by (kitti_dataloader.py:432-435): 3-D moderate Car AP, or
    the mean of Pedestrian's and Cyclist's when Car is not a class."""
    ap = kitti_ap(result[4])
    return ap[0, 1] if "Car" in cls_list else (ap[1, 1] + ap[2, 1]) / 2.


def format_ap_tables(result, cls_list=("Car",)):
    """The lines logger_and_select_best_map logs: precision_image / precision_ground / precision_3d R40 tables
    ([class, easy / moderate / hard]) and the selected number."""
    lines = []
    for title, arr in (("precision_image:", result[0]), ("precision_ground:", result[2]), ("precision_3d:", result[4])):
        lines += [title, str(kitti_ap(arr))]
    lines.append("selected (3-D moderate): %s" % select_metric(result, cls_list))
    return lines


def recall(pred_boxes, gt_boxes, iou_threshold):
    """evaluate_recall (kitti_dataloader.py:385-408) over frames: pred_boxes / gt_boxes are sequences of (n, 7) and
    (m, 7) float32 CUDA tensors, one per frame.  A label counts as detected when it is the 3-D-IoU argmax of some
    prediction whose best IoU is >= iou_threshold.  A frame with no prediction or no label detects nothing (the
    reference's np.max would raise there).  Returns (detected labels, total labels)."""
    from . import tf_ops
    detected = total = 0
    for p, g in zip(pred_boxes, gt_boxes):
        total += int(g.shape[0])
        if p.shape[0] == 0 or g.shape[0] == 0:
            continue
        _, iou3 = tf_ops.calc_iou(p.reshape(1, -1, 7), g.reshape(1, -1, 7))
        iou3 = iou3[0].cpu().numpy()
        best = iou3.max(axis=1)
        arg = iou3.argmax(axis=1)[np.where(best >= iou_threshold)[0]]
        detected += len(np.unique(arg))
    return detected, total


class EvalAccumulator:
    """Collects a validation set batch by batch -- the NMS block, its counts, each frame's P2 and label file -- and
    evaluates it in one call."""

    def __init__(self, cls_list=("Car",), cls_thresh=CLS_THRESH, img_shape=kitti_io.KITTI_IMG_SHAPE):
        self.cls_list, self.cls_thresh, self.img_shape = tuple(cls_list), cls_thresh, img_shape
        self.rows, self.numlist, self.labels = [], [], []

    def add(self, det_block, det_count, calibs, labels):
        """labels: one label file path or one (rows, 15) array of read_label_file per frame."""
        rows, nums = detection_rows(det_block, det_count, calibs, self.cls_list, self.cls_thresh, self.img_shape)
        if len(labels) != len(nums):
            raise ValueError("add: %d frames of detections but %d label entries" % (len(nums), len(labels)))
        self.rows.append(rows)
        self.numlist.append(nums)
        self.labels += [np.asarray(l, np.float64) if not isinstance(l, (str, bytes)) and hasattr(l, "shape")
                        else read_label_file(l) for l in labels]

    def __len__(self):
        return len(self.labels)

    def evaluate(self, device="cuda"):
        """The six (3, 3, 41) float32 arrays of tf_ops.evaluate, on `device`."""
        import torch
        from . import tf_ops
        rows = np.concatenate(self.rows, 0) if self.rows else np.zeros((0, 14), np.float32)
        nl = np.concatenate(self.numlist, 0) if self.numlist else np.zeros((0,), np.int32)
        return tf_ops.evaluate_labels(torch.from_numpy(rows).to(device), self.labels,
                                      torch.from_numpy(nl.astype(np.int32)).to(device))
