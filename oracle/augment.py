"""numpy restatement of csrc/augment.cu's recipe (include/ssd3d.h, ssd3d_augment_*), operation by operation: the float32
flip, noise search, corners and planes, the float64 translations and global transform rounded once, the context filter
and the point choice.  sin / cos go through the C twin of the evaluator (oracle/kitti_eval.py, twin_sincos), the
recipe the kernels share, so that this module and the kernels give the same bits.  The reference's own functions are
held to it by tests/golden/augment.npz."""
import numpy as np

from oracle.kitti_eval import twin_sincos

f32, f64 = np.float32, np.float64
TRIES = 100
EXPAND = f32(0.1)
GROW = (f32(0.5), f32(2.0), f32(0.5))               # (l, h, w)
ROT_PERTURB = np.pi / 3
GLOBAL_ROT = np.pi / 4
GLOBAL_SCALE = 0.1
PI32 = f32(np.pi)
NA = np.array([-0.5, -0.5, -0.5, -0.5, 0.5, 0.5, 0.5, 0.5], f32)
NB = np.array([-0.5, -0.5, 0.5, 0.5, -0.5, -0.5, 0.5, 0.5], f32)
NC = np.array([-1.0, 0.0, 0.0, -1.0, -1.0, 0.0, 0.0, -1.0], f32)
FACES = ((0, 1, 2), (7, 6, 5), (0, 3, 7), (1, 5, 6), (0, 4, 5), (3, 2, 6))
NORM2 = (np.array([-0.5, -0.5, 0.5, 0.5], f32), np.array([-0.5, 0.5, 0.5, -0.5], f32))
ALL_ONES = np.uint64(0xFFFFFFFFFFFFFFFF)


def sincos32(a):
    s, c = twin_sincos(np.asarray(a, f64))
    return s.astype(f32), c.astype(f32)


def rot_of(u):
    return -ROT_PERTURB + (2 * ROT_PERTURB) * np.asarray(u, f64)


def valid_rows(boxes):
    return np.any(np.asarray(boxes) != 0, axis=-1)


def planes(boxes, expand):
    """[K, 6, 3] normals and [K, 6] offsets of the box_planes of box_geom.cuh, boxes [K, 7] float32."""
    b = np.asarray(boxes, f32).reshape(-1, 7)
    sn, cs = sincos32(b[:, 6])
    c0, c1, c2 = b[:, 0:1], b[:, 2:3], b[:, 1:2]
    dl, dw, dh = (b[:, 3] + f32(expand))[:, None], (b[:, 5] + f32(expand))[:, None], (b[:, 4] + f32(expand))[:, None]
    p0, p1, p2 = dl * NA, dw * NB, dh * NC
    C = np.stack([(p0 * cs[:, None] + p1 * sn[:, None]) + c0, (p1 * cs[:, None] - p0 * sn[:, None]) + c1, p2 + c2], -1)
    n, d = np.zeros((len(b), 6, 3), f32), np.zeros((len(b), 6), f32)
    for f, (i, j, k) in enumerate(FACES):
        u, v = C[:, i] - C[:, j], C[:, j] - C[:, k]
        n[:, f] = np.stack([u[:, 1] * v[:, 2] - u[:, 2] * v[:, 1], u[:, 2] * v[:, 0] - u[:, 0] * v[:, 2],
                            u[:, 0] * v[:, 1] - u[:, 1] * v[:, 0]], -1)
        d[:, f] = -((n[:, f, 0] * C[:, i, 0] + n[:, f, 1] * C[:, i, 1]) + n[:, f, 2] * C[:, i, 2])
    return n, d


def inside(x, y, z, n, d):
    """[P] bool: the camera-frame points are inside the box of planes n [6, 3], d [6] (every face sign < 0)."""
    q = (x.astype(f32), z.astype(f32), y.astype(f32))
    out = np.ones(len(x), bool)
    for f in range(6):
        out &= (((q[0] * n[f, 0] + q[1] * n[f, 1]) + q[2] * n[f, 2]) + d[f]) < 0
    return out


def bev_corners(b):
    """[K, 4, 2] BEV corners (x, z) of boxes [K, 7] grown by 0.1 (box2d_to_corner_jit's order)."""
    dl, dw = b[:, 3] + EXPAND, b[:, 5] + EXPAND
    sn, cs = sincos32(b[:, 6])
    a, bb = dl[:, None] * NORM2[0], dw[:, None] * NORM2[1]
    return np.stack([(a * cs[:, None] + bb * sn[:, None]) + b[:, 0:1], (bb * cs[:, None] - a * sn[:, None]) + b[:, 2:3]], -1)


def _ccw_gt(A, B, C):
    return ((C[..., 1] - A[..., 1]) * (B[..., 0] - A[..., 0])) > ((B[..., 1] - A[..., 1]) * (C[..., 0] - A[..., 0]))


def _holds(a, q):
    ok = np.ones(np.broadcast_shapes(a.shape[:-2], q.shape[:-2]), bool)
    for l in range(4):
        for k in range(4):
            k1 = (k + 1) % 4
            v0, v1 = a[..., k1, 0] - a[..., k, 0], a[..., k1, 1] - a[..., k, 1]
            ok &= (v1 * (a[..., k, 0] - q[..., l, 0]) - v0 * (a[..., k, 1] - q[..., l, 1])) < 0
    return ok


def collide(a, q):
    """box_collision_test of rectangles a [..., 4, 2] against q [..., 4, 2] (broadcast), float32 op by op."""
    iw = np.minimum(a[..., 0].max(-1), q[..., 0].max(-1)) - np.maximum(a[..., 0].min(-1), q[..., 0].min(-1))
    ih = np.minimum(a[..., 1].max(-1), q[..., 1].max(-1)) - np.maximum(a[..., 1].min(-1), q[..., 1].min(-1))
    cross = np.zeros(iw.shape, bool)
    for k in range(4):
        A, B = a[..., k, :], a[..., (k + 1) % 4, :]
        for l in range(4):
            C, D = q[..., l, :], q[..., (l + 1) % 4, :]
            cross |= (_ccw_gt(A, C, D) != _ccw_gt(B, C, D)) & (_ccw_gt(A, B, C) != _ccw_gt(A, B, D))
    return (iw > 0) & (ih > 0) & (cross | _holds(a, q) | _holds(q, a))


def candidates(b, corners, loc, rot):
    """[T, 4, 2] candidate corners of box b for the tries' translations loc [T, 2] and angles rot [T]."""
    sr, cr = sincos32(rot)
    r0, r1 = corners[:, 0] - b[0], corners[:, 1] - b[2]
    q0 = r0[None] * cr[:, None] + r1[None] * sr[:, None]
    q1 = r1[None] * cr[:, None] - r0[None] * sr[:, None]
    tx, tz = f64(b[0]) + loc[:, 0], f64(b[2]) + loc[:, 1]
    return np.stack([(q0.astype(f64) + tx[:, None]).astype(f32), (q1.astype(f64) + tz[:, None]).astype(f32)], -1)


def scene_flags(u):
    return dict(flip=u[0] >= 0.5, noise=u[1] <= 0.5, grot=u[2] <= 0.5, gscale=u[3] <= 0.5)


def aug_boxes(boxes, u, loc, rot_u):
    """One scene: boxes [G, 7], u [6], loc [G, 100, 2], rot_u [G, 100] -> (boxes [G, 7], chosen try [G], state for
    aug_points)."""
    b = np.array(boxes, f32).reshape(-1, 7)
    g = len(b)
    fl = scene_flags(u)
    valid = valid_rows(b)
    if fl["flip"]:
        b[valid, 0] = -b[valid, 0]
        ry = b[valid, 6]
        b[valid, 6] = np.where(ry >= 0, PI32 - ry, -PI32 - ry)
    chosen = np.full(g, -1, np.int32)
    if fl["noise"] and valid.any():
        cur = np.zeros((g, 4, 2), f32)
        cur[valid] = bev_corners(b[valid])
        for i in np.flatnonzero(valid):
            cand = candidates(b[i], cur[i], np.asarray(loc[i], f64), rot_of(rot_u[i]))
            others = [k for k in np.flatnonzero(valid) if k != i]
            hit = collide(cand[:, None], cur[others][None]).any(1) if others else np.zeros(TRIES, bool)
            free = np.flatnonzero(~hit)
            if free.size:
                chosen[i] = free[0]
                cur[i] = cand[free[0]]
    st = dict(fl, valid=valid, chosen=chosen, pre=planes(b, EXPAND) if g else None, centre=b[:, :3].copy())
    st["sr"], st["cr"] = np.zeros(g, f32), np.ones(g, f32)
    st["loc"] = np.zeros((g, 2), f64)
    for j in np.flatnonzero(chosen >= 0):
        t = chosen[j]
        r = rot_of(rot_u[j, t])
        sr, cr = sincos32(np.array([r]))
        st["sr"][j], st["cr"][j] = sr[0], cr[0]
        st["loc"][j] = loc[j, t]
        b[j, 0] = f32(f64(b[j, 0]) + loc[j, t, 0])
        b[j, 2] = f32(f64(b[j, 2]) + loc[j, t, 1])
        b[j, 6] = f32(f64(b[j, 6]) + r)
    st["gs"], st["gc"], st["pscale"] = 0.0, 1.0, 1.0
    if fl["grot"]:
        a = (u[4] * 2.0 - 1.0) * GLOBAL_ROT
        s, c = twin_sincos(np.array([a]))
        st["gs"], st["gc"] = s[0], c[0]
        x, z = b[valid, 0].astype(f64), b[valid, 2].astype(f64)
        b[valid, 0] = (st["gc"] * x + st["gs"] * z).astype(f32)
        b[valid, 2] = (st["gc"] * z - st["gs"] * x).astype(f32)
        b[valid, 6] = b[valid, 6] + f32(a)
    if fl["gscale"]:
        f = (u[5] * 2.0 - 1.0) * GLOBAL_SCALE + 1.0
        b[valid, :6] = b[valid, :6] * f32(f)
        st["pscale"] = f if fl["grot"] else f64(f32(f))
    for k, e in zip((3, 4, 5), GROW):
        b[valid, k] = b[valid, k] + e
    st["fin"] = planes(b, f32(0.0)) if g else None
    for k, e in zip((3, 4, 5), GROW):
        b[valid, k] = b[valid, k] - e
    b[~valid] = 0
    return b, chosen, st


def aug_points(points, sem, keys, st):
    """One scene: points [N, 4], sem [N], keys [N] uint32 -> (points [N, 4], sort keys [N] uint64, moved_by [N])."""
    p = np.asarray(points, f32)
    x, y, z = p[:, 0].copy(), p[:, 1].copy(), p[:, 2].copy()
    n = len(p)
    if st["flip"]:
        x = -x
    mover = np.full(n, -1, np.int32)
    if st["noise"]:
        xo, yo, zo = x.copy(), y.copy(), z.copy()
        free = np.asarray(sem) != 0
        for j in np.flatnonzero(st["valid"]):
            m = free & inside(xo, yo, zo, st["pre"][0][j], st["pre"][1][j])
            free &= ~m
            if st["chosen"][j] < 0 or not m.any():
                continue
            mover[m] = j
            cx, cy, cz = st["centre"][j]
            p0, p1, p2 = xo[m] - cx, zo[m] - cz, yo[m] - cy
            sr, cr = st["sr"][j], st["cr"][j]
            q0, q1 = p0 * cr + p1 * sr, p1 * cr - p0 * sr
            x[m] = ((q0 + cx).astype(f64) + st["loc"][j, 0]).astype(f32)
            z[m] = ((q1 + cz).astype(f64) + st["loc"][j, 1]).astype(f32)
            y[m] = p2 + cy
    X, Y, Z = x.astype(f64), y.astype(f64), z.astype(f64)
    if st["grot"]:
        X, Z = st["gc"] * X + st["gs"] * Z, st["gc"] * Z - st["gs"] * X
    if st["gscale"]:
        X, Y, Z = X * st["pscale"], Y * st["pscale"], Z * st["pscale"]
    x, y, z = X.astype(f32), Y.astype(f32), Z.astype(f32)
    keep = np.ones(n, bool)
    neg = np.asarray(sem) == 0
    for j in np.flatnonzero(st["valid"]):
        keep &= ~(neg & inside(x, y, z, st["fin"][0][j], st["fin"][1][j]))
    out = np.stack([x, y, z, p[:, 3]], 1)
    sk = (np.asarray(keys).astype(np.uint32).astype(np.uint64) << np.uint64(32)) | np.arange(n, dtype=np.uint64)
    return out, np.where(keep, sk, ALL_ONES), mover


def choose(points, sort_keys, refill):
    """One scene: the ssd3d_augment_choose rule -> [M, 4]."""
    m = len(refill)
    kept = np.sort(sort_keys[sort_keys != ALL_ONES])
    n = len(kept)
    out = np.zeros((m, 4), f32)
    if n == 0:
        return out
    k = min(n, m)
    rank = np.arange(m, dtype=np.uint64)
    rank[k:] = (np.asarray(refill[k:]).astype(np.uint32).astype(np.uint64) * np.uint64(n)) >> np.uint64(32)
    idx = (kept[rank.astype(np.int64)] & np.uint64(0xFFFFFFFF)).astype(np.int64)
    return np.asarray(points, f32)[idx]


def sem_labels(points, boxes, labels):
    """One scene: class of the first valid box grown by 0.1 that holds the point, else 0."""
    p = np.asarray(points, f32)
    out = np.zeros(len(p), np.int32)
    free = np.ones(len(p), bool)
    valid = valid_rows(boxes)
    if not valid.any():
        return out
    n, d = planes(boxes, EXPAND)
    for j in np.flatnonzero(valid):
        m = free & inside(p[:, 0], p[:, 1], p[:, 2], n[j], d[j])
        out[m] = labels[j]
        free &= ~m
    return out


def augment(points, offsets, sem, boxes, labels, draws, num_points):
    """The whole Augmentor on host arrays; draws as numpy arrays (scene_u, loc_noise, rot_u, keys, refill).  Returns
    (block [B, M, 4], boxes [B, G, 7], dict of the per-kernel records)."""
    off = np.asarray(offsets, np.int64)
    B, G = boxes.shape[:2]
    scene_u, loc, rot_u, keys, refill = draws
    rec = dict(sem=[], chosen=np.zeros((B, G), np.int32), points=[], sort_keys=[], moved_by=[], survivors=np.zeros(B, np.int32))
    out_b = np.zeros((B, G, 7), f32)
    block = np.zeros((B, num_points, 4), f32)
    for s in range(B):
        pts = np.asarray(points[off[s]:off[s + 1]], f32)
        sl = sem_labels(pts, boxes[s], labels[s]) if sem is None else np.asarray(sem[off[s]:off[s + 1]])
        out_b[s], rec["chosen"][s], st = aug_boxes(boxes[s], scene_u[s], loc[s], rot_u[s])
        tp, sk, mv = aug_points(pts, sl, keys[off[s]:off[s + 1]], st)
        block[s] = choose(tp, sk, refill[s])
        rec["survivors"][s] = int((sk != ALL_ONES).sum())
        for k, v in (("sem", sl), ("points", tp), ("sort_keys", sk), ("moved_by", mv)):
            rec[k].append(v)
    for k in ("sem", "points", "sort_keys", "moved_by"):
        rec[k] = np.concatenate(rec[k])
    return block, out_b, rec
