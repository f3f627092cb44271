"""Readable float64 restatement of the reference's KITTI evaluator (test-only), and the loader of its C twin.

The rules are those of lib/utils/tf_ops/evaluation/evaluate.cpp in the reference: which overlap each metric uses
(:420-537), cleanData (:574-647), computeStatistics (:649-830), getThresholds (:539-572), eval_class (:835-928) and
eval (:1229-1343).  Angles go through math.sin / math.cos; the intersection of two rotated rectangles is the
detection rectangle clipped by the label rectangle.  The C twin (kitti_eval_twin.c) restates the same rules with the
arithmetic recipe the GPU kernels use (DESIGN.md section 3.10), so that it and the kernels agree bit for bit; this
module holds the twin to the rules.

Row layouts: detection rows are evaluate_map's 14 columns (class, x1, y1, x2, y2, alpha, t1, t2, t3, h, w, l, ry,
score); label rows are the 15 fields of a KITTI label line with the type replaced by a code (TYPE_CODES).
"""
import ctypes
import math
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_TWIN_SRC = os.path.join(_HERE, "kitti_eval_twin.c")
_TWIN_LIB = os.path.join(_HERE, "libkitti_eval_twin.so")
_twin = None

TYPE_CODES = {"car": 0, "pedestrian": 1, "cyclist": 2, "van": 3, "person_sitting": 4, "dontcare": 5}
CAR, PEDESTRIAN, CYCLIST, VAN, PERSON_SITTING, DONTCARE, OTHER = range(7)
N_SAMPLE = 41
MIN_HEIGHT = (40, 25, 25)
MAX_OCCLUSION = (0, 1, 2)
MAX_TRUNCATION = (0.15, 0.3, 0.5)
MIN_OVERLAP = (0.7, 0.5, 0.5)          # Car, Pedestrian, Cyclist; the same in every metric (evaluate.cpp:52)
NO_DETECTION = -10000000.0


# ---- overlaps ------------------------------------------------------------------------------------------------------
def rect(t1, t3, l, w, ry):
    """The four BEV corners toPolygon builds (evaluate.cpp:461-485), clockwise in (x, z)."""
    c, s = math.cos(ry), math.sin(ry)
    a, b = abs(l) / 2.0, abs(w) / 2.0
    return [(c * u + s * v + t1, -s * u + c * v + t3) for u, v in ((a, b), (a, -b), (-a, -b), (-a, b))]


def _side(p, q, r):
    return (q[0] - p[0]) * (r[1] - p[1]) - (q[1] - p[1]) * (r[0] - p[0])


def intersection_area(subject, clip):
    """Area of a convex polygon clipped by a clockwise convex polygon (Sutherland-Hodgman)."""
    poly = list(subject)
    for k in range(len(clip)):
        a, b = clip[k], clip[(k + 1) % len(clip)]
        out = []
        for i in range(len(poly)):
            s, e = poly[i - 1], poly[i]
            ds, de = _side(a, b, s), _side(a, b, e)
            if (de <= 0) != (ds <= 0):
                t = ds / (ds - de)
                out.append((s[0] + t * (e[0] - s[0]), s[1] + t * (e[1] - s[1])))
            if de <= 0:
                out.append(e)
        poly = out
        if not poly:
            return 0.0
    if len(poly) < 3:
        return 0.0
    acc = sum(poly[i][0] * poly[(i + 1) % len(poly)][1] - poly[(i + 1) % len(poly)][0] * poly[i][1] for i in range(len(poly)))
    return abs(acc) / 2.0


def _ratio(num, den):
    """A pair whose union (or detection) area / volume is <= 0 has overlap 0 (the reference divides 0 by 0)."""
    return num / den if den > 0 else 0.0


def image_overlap(d, g, criterion=-1):
    """Axis-aligned 2-D IoU of (x1, y1, x2, y2) rectangles (evaluate.cpp:420-454); criterion 0: over d's area."""
    w = min(d[2], g[2]) - max(d[0], g[0])
    h = min(d[3], g[3]) - max(d[1], g[1])
    if w <= 0 or h <= 0:
        return 0.0
    inter = w * h
    ad = (d[2] - d[0]) * (d[3] - d[1])
    ag = (g[2] - g[0]) * (g[3] - g[1])
    return _ratio(inter, ad + ag - inter) if criterion < 0 else _ratio(inter, ad)


def box_overlaps(d, g, criterion=-1):
    """(BEV, 3-D) overlap of two (t1, t2, t3, l, h, w, ry) boxes (evaluate.cpp:487-537); criterion 0: over d."""
    t1, t2, t3, l, h, w, ry = (float(x) for x in d)
    u1, u2, u3, gl, gh, gw, gry = (float(x) for x in g)
    inter = intersection_area(rect(t1, t3, l, w, ry), rect(u1, u3, gl, gw, gry))
    ad, ag = abs(l) * abs(w), abs(gl) * abs(gw)
    yov = max(0.0, min(t2, u2) - max(t2 - h, u2 - gh))
    iv = inter * yov
    vd, vg = h * l * w, gh * gl * gw
    if criterion < 0:
        return _ratio(inter, ad + ag - inter), _ratio(iv, vd + vg - iv)
    return _ratio(inter, ad), _ratio(iv, vd)


def det_box7(r):
    return (r[6], r[7], r[8], r[11], r[9], r[10], r[12])


def label_box7(r):
    return (r[11], r[12], r[13], r[10], r[8], r[9], r[14])


def pair_overlaps(det_row, label_row):
    """(image, BEV, 3-D IoU, then the same over the detection) for one detection row and one label row."""
    d = [float(x) for x in det_row]
    g = [float(x) for x in label_row]
    bev, v3 = box_overlaps(det_box7(d), label_box7(g))
    bev0, v30 = box_overlaps(det_box7(d), label_box7(g), 0)
    return (image_overlap(d[1:5], g[4:8]), bev, v3, image_overlap(d[1:5], g[4:8], 0), bev0, v30)


def calc_iou(dets, gts):
    """[b,n,7] x [b,m,7] -> ([b,n,m] BEV IoU, [b,n,m] 3-D IoU), float64."""
    dets, gts = np.asarray(dets, np.float64), np.asarray(gts, np.float64)
    b, n, m = dets.shape[0], dets.shape[1], gts.shape[1]
    bev, v3 = np.zeros((b, n, m)), np.zeros((b, n, m))
    for s in range(b):
        for i in range(n):
            for j in range(m):
                bev[s, i, j], v3[s, i, j] = box_overlaps(dets[s, i], gts[s, j])
    return bev, v3


# ---- the rules -----------------------------------------------------------------------------------------------------
def det_class(v):
    """int(row[0]) as evaluate.cpp:279-303 reads it; anything but 0, 1, 2 is a 'DontCare' detection (3)."""
    return int(v) if -1 < v < 3 else 3


def ignored_gt(row, cls, diff):
    """cleanData for a label row: 0 counted, 1 ignored (neighbour class, or the class but too hard), -1 other."""
    t = int(row[0])
    if t == cls:
        valid = 1
    elif (cls == PEDESTRIAN and t == PERSON_SITTING) or (cls == CAR and t == VAN):
        valid = 0
    else:
        valid = -1
    too_hard = int(row[2]) > MAX_OCCLUSION[diff] or row[1] > MAX_TRUNCATION[diff] or row[7] - row[5] <= MIN_HEIGHT[diff]
    if valid == 1 and not too_hard:
        return 0
    if valid == 0 or (too_hard and valid == 1):
        return 1
    return -1


def ignored_det(row, cls, diff):
    """cleanData for a detection row: the height truncated to int32 below the minimum -> 1, the class -> 0, else -1."""
    if int(abs(float(row[2]) - float(row[4]))) < MIN_HEIGHT[diff]:
        return 1
    return 0 if det_class(row[0]) == cls else -1


def frame_statistics(dets, labels, ov, cls, diff, metric, compute_fp, thresh=0.0):
    """computeStatistics for one frame.  ov[j][i] = overlap of detection j with label i in this metric (criterion 0
    for DontCare rows).  Returns (tp, fp, fn, scores of the true positives)."""
    nd, ng = len(dets), len(labels)
    idet = [ignored_det(dets[j], cls, diff) for j in range(nd)]
    below = [compute_fp and float(dets[j][13]) < thresh for j in range(nd)]
    assigned = [False] * nd
    tp = fp = fn = 0
    scores = []
    min_ov = MIN_OVERLAP[cls]
    for i in range(ng):
        ig = ignored_gt(labels[i], cls, diff)
        if ig == -1:
            continue
        det_idx, valid, max_overlap, assigned_ignored = -1, NO_DETECTION, 0.0, False
        for j in range(nd):
            if idet[j] == -1 or assigned[j] or below[j]:
                continue
            o = ov[j][i]
            if not compute_fp:
                # first pass: the highest-scoring candidate; ties keep the first
                if o > min_ov and float(dets[j][13]) > valid:
                    det_idx, valid = j, float(dets[j][13])
            elif o > min_ov and (o > max_overlap or assigned_ignored) and idet[j] == 0:
                # counting pass: the greatest overlap wins, and a counted detection displaces an ignored one
                det_idx, valid, max_overlap, assigned_ignored = j, 1.0, o, False
            elif o > min_ov and valid == NO_DETECTION and idet[j] == 1:
                det_idx, valid, assigned_ignored = j, 1.0, True
        if valid == NO_DETECTION:
            if ig == 0:
                fn += 1
        elif ig == 1 or idet[det_idx] == 1:
            assigned[det_idx] = True
        else:
            tp += 1
            scores.append(float(dets[det_idx][13]))
            assigned[det_idx] = True
    if compute_fp:
        free = [not (assigned[j] or idet[j] != 0 or below[j]) for j in range(nd)]
        fp = sum(free)
        stuff = 0
        for i in range(ng):
            if int(labels[i][0]) != DONTCARE:
                continue
            for j in range(nd):
                if not assigned[j] and idet[j] == 0 and not below[j] and ov[j][i] > min_ov:
                    assigned[j] = True
                    stuff += 1
        fp -= stuff
    return tp, fp, fn, scores


def get_thresholds(scores, n_gt):
    """The scores at which recall crosses the 41 sample points (evaluate.cpp:539-572), in float64."""
    v = sorted((float(s) for s in scores), reverse=True)
    out, current = [], 0.0
    for i in range(len(v)):
        l_recall = (i + 1) / float(n_gt)
        r_recall = (i + 2) / float(n_gt) if i < len(v) - 1 else l_recall
        if (r_recall - current) < (current - l_recall) and i < len(v) - 1:
            continue
        out.append(v[i])
        current += 1.0 / (N_SAMPLE - 1.0)
    return out


def _max_from(p, i):
    """std::max_element over p[i:]: the first of the largest, NaN never replacing a number nor being replaced."""
    best = p[i]
    for x in p[i + 1:]:
        if best < x:
            best = x
    return best


def precision_curve(tp, fp, n_thresholds):
    p = [tp[t] / float(tp[t] + fp[t]) if tp[t] + fp[t] else float("nan") for t in range(n_thresholds)]
    p += [0.0] * (N_SAMPLE - n_thresholds)
    return [_max_from(p, t) for t in range(n_thresholds)] + p[n_thresholds:]


def eval_flags(det_rows):
    """[metric][class]: whether a class is evaluated in a metric (evaluate.cpp:316-331)."""
    flags = [[False] * 3 for _ in range(3)]
    for r in det_rows:
        c = det_class(r[0])
        if c > 2:
            continue
        flags[0][c] |= bool(r[1] >= 0)
        flags[1][c] |= bool(r[6] != -1000 and r[8] != -1000 and r[10] > 0 and r[11] > 0)
        flags[2][c] |= bool(r[6] != -1000 and r[7] != -1000 and r[8] != -1000 and r[9] > 0 and r[10] > 0 and r[11] > 0)
    return flags


def evaluate(det_rows, labels, numlist, return_counts=False):
    """det_rows [N,14] float32, labels: one [R_f,15] float64 array per frame, numlist [F] -> the six [3,3,41] float32
    arrays (precision_image, aos_image, precision_ground, aos_ground, precision_3d, aos_3d).  AOS is never computed
    (the reference clears compute_aos and never sets it), so those three stay -1."""
    det_rows = np.asarray(det_rows, np.float32).reshape(-1, 14)
    offs = np.concatenate([[0], np.cumsum(numlist)]).astype(np.int64)
    frames = []
    for f, lab in enumerate(labels):
        d = [[float(x) for x in row] for row in det_rows[offs[f]:offs[f + 1]]]
        g = [[float(x) for x in row] for row in np.asarray(lab, np.float64).reshape(-1, 15)]
        ov = [[[0.0] * len(g) for _ in d] for _ in range(3)]
        for j, dr in enumerate(d):
            for i, gr in enumerate(g):
                o = pair_overlaps(dr, gr)
                for m in range(3):
                    ov[m][j][i] = o[m + 3] if int(gr[0]) == DONTCARE else o[m]
        frames.append((d, g, ov))
    out = np.full((6, 3, 3, N_SAMPLE), -1.0, np.float32)
    counts = {}
    flags = eval_flags(det_rows)
    for m in range(3):
        for c in range(3):
            if not flags[m][c]:
                continue
            for diff in range(3):
                scores, n_gt = [], 0
                for d, g, ov in frames:
                    n_gt += sum(ignored_gt(r, c, diff) == 0 for r in g)
                    scores += frame_statistics(d, g, ov[m], c, diff, m, False)[3]
                thr = get_thresholds(scores, n_gt)
                tp, fp, fn = [0] * len(thr), [0] * len(thr), [0] * len(thr)
                for d, g, ov in frames:
                    for t, th in enumerate(thr):
                        a, b, e, _ = frame_statistics(d, g, ov[m], c, diff, m, True, th)
                        tp[t] += a
                        fp[t] += b
                        fn[t] += e
                counts[(m, c, diff)] = (thr, tp, fp, fn)
                out[2 * m, c, diff] = np.asarray(precision_curve(tp, fp, len(thr)), np.float64).astype(np.float32)
    return (tuple(out), counts) if return_counts else tuple(out)


# ---- synthetic validation sets --------------------------------------------------------------------------------------
_DIMS = {CAR: (3.9, 1.55, 1.6), VAN: (5.0, 2.1, 1.9), PEDESTRIAN: (0.8, 1.75, 0.6), CYCLIST: (1.75, 1.7, 0.6),
         OTHER: (2.0, 1.5, 1.0)}       # l, h, w


def _label(rng, t):
    """One KITTI-like label row of type t: location in front of the camera, projected 2-D box of height
    720 * h / z px, truncation / occlusion drawn across every difficulty boundary, two decimals like label_2."""
    l, h, w = (d * rng.uniform(0.85, 1.15) for d in _DIMS[t])
    x, y, z = rng.uniform(-15, 15), rng.uniform(1.4, 1.9), rng.uniform(4, 55)
    ry = rng.uniform(-np.pi, np.pi)
    u, ph = 720.0 * x / z + 620.0, 720.0 * h / z
    pw = 720.0 * max(l, w) / z
    trunc = rng.choice([0.0, 0.0, 0.1, 0.2, 0.4, 0.6])
    occ = int(rng.choice([0, 0, 1, 2, 3]))
    r = [t, trunc, occ, 0.0, u - pw / 2, 190.0 - ph / 2, u + pw / 2, 190.0 + ph / 2, h, w, l, x, y, z, ry]
    return [round(float(v), 2) for v in r]


def _dontcare(rng):
    u, v = rng.uniform(0, 1100), rng.uniform(120, 250)
    return [DONTCARE, -1, -1, -10, u, v, u + rng.uniform(20, 140), v + rng.uniform(10, 60), -1, -1, -1, -1000, -1000, -1000, -10]


def _detection(rng, lab, cls, jitter=1.0):
    t, tr, oc, al, x1, y1, x2, y2, h, w, l, x, y, z, ry = lab
    j = lambda s: rng.normal(0, s * jitter)
    return [cls, x1 + j(3), y1 + j(3), x2 + j(3), y2 + j(3), 0.0, x + j(0.15), y + j(0.08), z + j(0.2), h * (1 + j(0.04)),
            w * (1 + j(0.04)), l * (1 + j(0.04)), ry + j(0.08), 0.0]


def synthetic_frames(n_frames, seed=0, max_labels=10, perfect=False, miss_all=False):
    """(det_rows (n, 14) float32, labels [per frame (r, 15) float64], numlist (frames,) int32): Car, Van, Pedestrian,
    Cyclist, Misc and DontCare labels; detections are jittered labels over three classes (Vans detected as Cars
    sometimes) plus duplicates, false positives, detections inside DontCare areas and tied scores.
    perfect: one exact detection per Car / Pedestrian / Cyclist label.  miss_all: detections far from every label."""
    rng = np.random.default_rng(seed)
    types = [CAR] * 5 + [VAN, PEDESTRIAN, PEDESTRIAN, CYCLIST, OTHER]
    rows, labels, nums = [], [], []
    for _ in range(n_frames):
        lab = [_label(rng, int(rng.choice(types))) for _ in range(int(rng.integers(0, max_labels + 1)))]
        lab += [_dontcare(rng) for _ in range(int(rng.integers(0, 3)))]
        det = []
        for r in lab:
            t = int(r[0])
            if perfect:
                if t in (CAR, PEDESTRIAN, CYCLIST):
                    det.append([t] + r[4:8] + [0.0] + r[11:14] + [r[8], r[9], r[10], r[14], rng.uniform(0.3, 1.0)])
                continue
            if miss_all:
                if t != DONTCARE:
                    d = _detection(rng, r, t if t < 3 else 0)
                    d[6] += 40.0
                    d[8] += 40.0
                    d[1:5] = [1300.0, 10.0, 1340.0, 60.0]
                    det.append(d)
                continue
            if t == DONTCARE:
                if rng.uniform() < 0.5:                   # a false positive inside the stuff area
                    d = _detection(rng, _label(rng, CAR), 0)
                    d[1:5] = [r[4] + 2, r[5] + 1, r[6] - 2, r[7] - 1]
                    det.append(d)
                continue
            cls = {CAR: 0, VAN: 0 if rng.uniform() < 0.3 else None, PEDESTRIAN: 1, CYCLIST: 2}.get(t)
            if cls is None or rng.uniform() > 0.85:
                continue
            det.append(_detection(rng, r, cls))
            if rng.uniform() < 0.15:
                det.append(_detection(rng, r, cls))         # duplicate
        for _ in range(0 if perfect or miss_all else int(rng.integers(0, 3))):     # false positives
            det.append(_detection(rng, _label(rng, int(rng.choice([CAR, PEDESTRIAN, CYCLIST]))), int(rng.integers(0, 3))))
        for d in det:
            if d[13] == 0.0:
                d[13] = round(float(rng.uniform(0.3, 1.0)), 2)    # a 0.01 grid: tied scores
        rows += det
        labels.append(np.asarray(lab, np.float64).reshape(-1, 15))
        nums.append(len(det))
    return np.asarray(rows, np.float32).reshape(-1, 14), labels, np.asarray(nums, np.int32)


def margin_ok(det_rows, labels, numlist, eps=1e-9):
    """True when no overlap of a frame lies within eps of 0.5 or 0.7, and no two distinct overlaps of one label row
    lie within eps of each other: then float64 rounding differences of ~1e-12 cannot change a decision."""
    off = 0
    for lab, n in zip(labels, numlist):
        d = det_rows[off:off + n]
        off += n
        if n == 0 or len(lab) == 0:
            continue
        o = twin_pair_overlaps(np.repeat(d, len(lab), 0), np.tile(lab, (n, 1))).reshape(n, len(lab), 6)
        if np.any(np.abs(o - 0.5) < eps) or np.any(np.abs(o - 0.7) < eps):
            return False
        for k in range(6):
            for i in range(len(lab)):
                v = np.sort(o[:, i, k])
                gap = np.diff(v)
                if np.any((gap > 0) & (gap < eps)):
                    return False
    return True


# ---- the C twin ----------------------------------------------------------------------------------------------------
def build(force=False):
    """Compile the twin with gcc, with liboracle.so's flags (seconds)."""
    if force or not os.path.exists(_TWIN_LIB) or os.path.getmtime(_TWIN_LIB) < os.path.getmtime(_TWIN_SRC):
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC",
                               "-o", _TWIN_LIB, _TWIN_SRC, "-lm"])
    return _TWIN_LIB


def twin():
    global _twin
    if _twin is None:
        build()
        l = ctypes.CDLL(_TWIN_LIB)
        P = ctypes.c_void_p
        l.kitti_sincos_n.argtypes = [ctypes.c_long, P, P, P]
        l.kitti_pair_overlaps.argtypes = [ctypes.c_long, P, P, P]
        l.kitti_box_iou.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, P, P, P, P]
        l.kitti_box_iou_matched.argtypes = [ctypes.c_long, P, P, P, P]
        l.kitti_get_thresholds.argtypes = [P, ctypes.c_long, ctypes.c_double, P]
        l.kitti_evaluate.argtypes = [ctypes.c_int, P, P, P, P, P]
        _twin = l
    return _twin


def _ptr(a):
    return ctypes.c_void_p(a.ctypes.data)


def twin_sincos(x):
    x = np.ascontiguousarray(x, np.float64)
    s, c = np.empty_like(x), np.empty_like(x)
    twin().kitti_sincos_n(x.size, _ptr(x), _ptr(s), _ptr(c))
    return s, c


def twin_pair_overlaps(det_rows, label_rows):
    d = np.ascontiguousarray(det_rows, np.float32).reshape(-1, 14)
    g = np.ascontiguousarray(label_rows, np.float64).reshape(-1, 15)
    out = np.empty((d.shape[0], 6))
    twin().kitti_pair_overlaps(d.shape[0], _ptr(d), _ptr(g), _ptr(out))
    return out


def twin_box_iou(dets, gts):
    d, g = np.ascontiguousarray(dets, np.float32), np.ascontiguousarray(gts, np.float32)
    b, n, m = d.shape[0], d.shape[1], g.shape[1]
    bev, v3 = np.zeros((b, n, m), np.float32), np.zeros((b, n, m), np.float32)
    twin().kitti_box_iou(b, n, m, _ptr(d), _ptr(g), _ptr(bev), _ptr(v3))
    return bev, v3


def twin_box_iou_matched(dets, gts):
    d, g = np.ascontiguousarray(dets, np.float32).reshape(-1, 7), np.ascontiguousarray(gts, np.float32).reshape(-1, 7)
    bev, v3 = np.zeros(d.shape[0], np.float32), np.zeros(d.shape[0], np.float32)
    twin().kitti_box_iou_matched(d.shape[0], _ptr(d), _ptr(g), _ptr(bev), _ptr(v3))
    return bev, v3


def twin_get_thresholds(scores, n_gt):
    v = np.array(scores, np.float64)
    t = np.zeros(N_SAMPLE)
    nt = twin().kitti_get_thresholds(_ptr(v), v.size, float(n_gt), _ptr(t))
    return t[:min(nt, N_SAMPLE)].tolist(), nt


def twin_evaluate(det_rows, labels, numlist):
    d = np.ascontiguousarray(det_rows, np.float32).reshape(-1, 14)
    lab = [np.asarray(x, np.float64).reshape(-1, 15) for x in labels]
    g = np.ascontiguousarray(np.concatenate(lab, 0) if lab else np.zeros((0, 15)), np.float64)
    nl = np.ascontiguousarray(numlist, np.int32)
    lc = np.array([x.shape[0] for x in lab], np.int32)
    out = np.empty((6, 3, 3, N_SAMPLE), np.float32)
    if twin().kitti_evaluate(len(lab), _ptr(d), _ptr(nl), _ptr(g), _ptr(lc), _ptr(out)) != 0:
        raise ValueError("kitti_evaluate: a frame has more than 1024 detections")
    return tuple(out)
