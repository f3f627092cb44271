"""numpy restatement of csrc/mixup.cu's recipe (include/ssd3d.h, ssd3d_mixup_*), operation by operation: the database
membership of the float32 planes of oracle/augment.py, the float32 BEV corners and collision test of the noise search,
the float64 height move rounded once, and the mixup chain in front of oracle/augment.py with its rule for absent slots
(a negative semantic label: no move, no survivor, zeros).  The reference's own functions are held to it by
tests/golden/mixup.npz."""
import numpy as np

from oracle import augment as OA

f32, f64 = np.float32, np.float64
MIN_POINTS = 5
ENLARGE = (f32(0.5), f32(0.5))                     # (l, w) of box_3d_collision_test


def members(points, boxes):
    """[G, N] bool: the points inside each valid row grown by 0.1 (False for a padded row)."""
    p = np.asarray(points, f32)
    b = np.asarray(boxes, f32).reshape(-1, 7)
    out = np.zeros((len(b), len(p)), bool)
    valid = OA.valid_rows(b)
    if valid.any():
        n, d = OA.planes(b, OA.EXPAND)
        for j in np.flatnonzero(valid):
            out[j] = OA.inside(p[:, 0], p[:, 1], p[:, 2], n[j], d[j])
    return out


def build_db(points, offsets, boxes, labels, classes=(1,), min_points=MIN_POINTS):
    """The object database of ragged frames -> dict(points, offsets, boxes, classes, frames, rows, counts [B, G])."""
    off = np.asarray(offsets, np.int64)
    B, G = boxes.shape[:2]
    counts = np.zeros((B, G), np.int32)
    pts, sizes, rec = [], [], []
    for s in range(B):
        p = np.asarray(points[off[s]:off[s + 1]], f32)
        m = members(p, boxes[s])
        counts[s] = m.sum(1)
        for j in range(G):
            if OA.valid_rows(boxes[s, j]) and labels[s, j] in classes and counts[s, j] >= min_points:
                pts.append(p[m[j]])
                sizes.append(int(counts[s, j]))
                rec.append((s, j))
    rec = np.asarray(rec, np.int32).reshape(-1, 2)
    return dict(points=np.concatenate(pts) if pts else np.zeros((0, 4), f32),
                offsets=np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64), boxes=boxes[rec[:, 0], rec[:, 1]].astype(f32),
                classes=labels[rec[:, 0], rec[:, 1]].astype(np.int32), frames=rec[:, 0], rows=rec[:, 1], counts=counts)


def corners(b, dl, dw):
    """[K, 4, 2] BEV corners of boxes b [K, 7] with dims dl, dw (box2d_to_corner_jit, float32)."""
    sn, cs = OA.sincos32(b[:, 6])
    a, bb = dl[:, None] * OA.NORM2[0], dw[:, None] * OA.NORM2[1]
    return np.stack([(a * cs[:, None] + bb * sn[:, None]) + b[:, 0:1], (bb * cs[:, None] - a * sn[:, None]) + b[:, 2:3]], -1)


def move_height(box, plane):
    a, b, c, d = (f64(v) for v in plane)
    return f64(box[1]) - (((-d - a * f64(box[0])) - c * f64(box[2])) / b)


def paste_scene(points, sem, boxes, labels, ids, db, plane):
    """One scene: -> (points [N + drawn, 4], sem [..] (-1: a dropped object's slot), boxes [G + S, 7], labels [G + S],
    accepted [S])."""
    b = np.asarray(boxes, f32).reshape(-1, 7)
    S = len(ids)
    valid = OA.valid_rows(b)
    q = corners(b[valid], b[valid, 3], b[valid, 5])
    acc = np.zeros(S, np.int32)
    out_b, out_l = [b[valid]], [np.asarray(labels)[valid]]
    out_p, out_s = [np.asarray(points, f32)], [np.asarray(sem, np.int32)]
    for i, oid in enumerate(ids):
        if oid < 0:
            continue
        d = db["boxes"][oid:oid + 1].astype(f32)
        e = corners(d, d[:, 3] + ENLARGE[0], d[:, 5] + ENLARGE[1])
        n = int(db["offsets"][oid + 1] - db["offsets"][oid])
        p = db["points"][db["offsets"][oid]:db["offsets"][oid + 1]].astype(f32).copy()
        if len(q) and OA.collide(e, q).any():
            out_p.append(np.zeros((n, 4), f32))
            out_s.append(np.full(n, -1, np.int32))
            continue
        acc[i] = 1
        q = np.concatenate([q, corners(d, d[:, 3], d[:, 5])])
        mh = move_height(d[0], plane)
        d = d.copy()
        d[0, 1] = f32(f64(d[0, 1]) - mh)
        p[:, 1] = (p[:, 1].astype(f64) - mh).astype(f32)
        out_b.append(d)
        out_l.append(db["classes"][oid:oid + 1])
        out_p.append(p)
        out_s.append(np.full(n, db["classes"][oid], np.int32))
    ob = np.zeros((len(b) + S, 7), f32)
    ol = np.zeros(len(b) + S, np.int32)
    cat_b, cat_l = np.concatenate(out_b), np.concatenate(out_l)
    ob[:len(cat_b)], ol[:len(cat_l)] = cat_b, cat_l
    return np.concatenate(out_p), np.concatenate(out_s), ob, ol, acc


def paste(points, offsets, sem, boxes, labels, ids, db, planes):
    """Every scene -> (points [T', 4], offsets [B + 1], sem [T'], boxes [B, G + S, 7], labels [B, G + S], accepted [B, S])."""
    off = np.asarray(offsets, np.int64)
    res = [paste_scene(points[off[s]:off[s + 1]], sem[off[s]:off[s + 1]], boxes[s], labels[s], ids[s], db, planes[s])
           for s in range(len(off) - 1)]
    out_off = np.concatenate([[0], np.cumsum([len(r[0]) for r in res])]).astype(np.int32)
    return (np.concatenate([r[0] for r in res]), out_off, np.concatenate([r[1] for r in res]), np.stack([r[2] for r in res]),
            np.stack([r[3] for r in res]), np.stack([r[4] for r in res]))


def augment(points, offsets, sem, boxes, labels, ids, db, planes, draws, num_points):
    """The mixup chain on host arrays: semantic labels (of the original boxes when sem is None), the paste, then
    oracle/augment.py's stages on the pasted layout, absent slots neither moved nor kept.  Returns (block, boxes, labels,
    dict of records)."""
    off = np.asarray(offsets, np.int64)
    if sem is None:
        sem = np.concatenate([OA.sem_labels(points[off[s]:off[s + 1]], boxes[s], labels[s]) for s in range(len(off) - 1)])
    pp, poff, psem, pb, pl, acc = paste(points, off, sem, boxes, labels, ids, db, planes)
    B, R = pb.shape[:2]
    scene_u, loc, rot_u, keys, refill = draws
    rec = dict(sem=sem, pasted_points=pp, pasted_offsets=poff, pasted_sem=psem, pasted_boxes=pb, accepted=acc,
               chosen=np.zeros((B, R), np.int32), points=[], sort_keys=[], moved_by=[], survivors=np.zeros(B, np.int32))
    out_b = np.zeros((B, R, 7), f32)
    block = np.zeros((B, num_points, 4), f32)
    for s in range(B):
        sl = slice(poff[s], poff[s + 1])
        out_b[s], rec["chosen"][s], st = OA.aug_boxes(pb[s], scene_u[s], loc[s], rot_u[s])
        tp, sk, mv = OA.aug_points(pp[sl], np.maximum(psem[sl], 0), keys[sl], st)
        absent = psem[sl] < 0
        tp[absent], sk[absent], mv[absent] = 0, OA.ALL_ONES, -1
        block[s] = OA.choose(tp, sk, refill[s])
        rec["survivors"][s] = int((sk != OA.ALL_ONES).sum())
        for k, v in (("points", tp), ("sort_keys", sk), ("moved_by", mv)):
            rec[k].append(v)
    for k in ("points", "sort_keys", "moved_by"):
        rec[k] = np.concatenate(rec[k])
    return block, out_b, pl, rec
