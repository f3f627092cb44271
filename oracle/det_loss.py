"""numpy restatement of csrc/det_loss.cu's own recipe (include/ssd3d.h, ssd3d_det_assign / ssd3d_det_loss /
ssd3d_det_loss_grad): the float32 targets operation by operation, including the face planes as the kernel computes
them, and the float64 losses and gradients."""
import numpy as np

f32 = np.float32
EXPAND = f32(0.1)
SAMPLE_RANGE = f32(10.0)
CTR_EPS = 1e-6
NA = np.array([-0.5, -0.5, -0.5, -0.5, 0.5, 0.5, 0.5, 0.5], f32)
NB = np.array([-0.5, -0.5, 0.5, 0.5, -0.5, -0.5, 0.5, 0.5], f32)
NC = np.array([-1.0, 0.0, 0.0, -1.0, -1.0, 0.0, 0.0, -1.0], f32)
FACES = ((0, 1, 2), (7, 6, 5), (0, 3, 7), (1, 5, 6), (0, 4, 5), (3, 2, 6))
SX = np.array([1, 1, -1, -1, 1, 1, -1, -1], np.float64)
SZ = np.array([1, -1, -1, 1, 1, -1, -1, 1], np.float64)


def box_planes(box, expand=f32(0.0)):
    """[6, 3] normals and [6] offsets of one box in the (x, z, y) frame, float32 op by op."""
    box = box.astype(f32)
    c0, c1, c2 = box[0], box[2], box[1]                      # centre in (x, z, y)
    dl, dw, dh = box[3] + expand, box[5] + expand, box[4] + expand
    sn, cs = f32(np.sin(np.float64(box[6]))), f32(np.cos(np.float64(box[6])))
    p0, p1, p2 = dl * NA, dw * NB, dh * NC
    C = np.stack([(p0 * cs + p1 * sn) + c0, (p1 * cs - p0 * sn) + c1, p2 + c2], axis=1).astype(f32)
    n, d = np.zeros((6, 3), f32), np.zeros(6, f32)
    for k, (a, b, c) in enumerate(FACES):
        u, v = C[a] - C[b], C[b] - C[c]
        n[k] = (u[1] * v[2] - u[2] * v[1], u[2] * v[0] - u[0] * v[2], u[0] * v[1] - u[1] * v[0])
        d[k] = -((n[k, 0] * C[a, 0] + n[k, 1] * C[a, 1]) + n[k, 2] * C[a, 2])
    return n, d


def inside(pts, n, d):
    """pts [P, 3] camera frame -> [P] bool: every face gives sign < 0."""
    q = pts.astype(f32)[:, [0, 2, 1]]
    s = ((q[:, None, 0] * n[None, :, 0] + q[:, None, 1] * n[None, :, 1]) + q[:, None, 2] * n[None, :, 2]) + d[None, :]
    return np.all(s < 0, axis=1)


def floor_mod(a, b):
    m = np.fmod(a, b)
    fix = (m != 0) & ((m < 0) != (b < 0))
    return np.where(fix, m + b, m).astype(f32)


def encode_angle(ry, nbins=12):
    two_pi, per, half = f32(2 * np.pi), f32(2 * np.pi / nbins), f32(2 * np.pi / nbins / 2.0)
    a = floor_mod(f32(ry), two_pi)
    sh = floor_mod(f32(a + half), two_pi)
    cf = np.floor(f32(sh / per))
    b = np.minimum(cf.astype(np.int32), nbins - 1)
    res = f32(f32(sh - f32(f32(cf * per) + half)) / per)
    return b, res


def centerness(p, box):
    ry = np.float64(box[6])
    c, s = np.cos(ry), np.sin(ry)
    e = p.astype(np.float64) - box[:3].astype(np.float64)
    cx, cy, cz = c * e[0] - s * e[2], e[1], s * e[0] + c * e[2]
    l2, h, w2 = np.float64(box[3]) / 2, np.float64(box[4]), np.float64(box[5]) / 2
    fr, bk, bo, tp, le, ri = l2 - cx, cx + l2, -cy, cy + h, w2 - cz, cz + w2
    r = lambda a, b: min(a, b) / max(a, b)
    return f32(np.power(max(r(fr, bk) * r(bo, tp) * r(le, ri), CTR_EPS), 1.0 / 3.0))


def assign(base_xyz, vote_base, gt_boxes, gt_labels, nbins=12):
    """The ssd3d_det_assign record as a dict of numpy arrays."""
    B, N, _ = base_xyz.shape
    NV, G = vote_base.shape[1], gt_boxes.shape[1]
    out = dict(assigned_idx=np.zeros((B, N), np.int32), assigned_box=np.zeros((B, N, 7), f32), pmask=np.zeros((B, N), f32),
               nmask=np.zeros((B, N), f32), cls_label=np.zeros((B, N), f32), angle_bin=np.zeros((B, N), np.int32),
               angle_res=np.zeros((B, N), f32), offset_target=np.zeros((B, N, 6), f32), vote_mask=np.zeros((B, NV), f32),
               vote_target=np.zeros((B, NV, 3), f32))
    for s in range(B):
        valid = [j for j in range(G) if np.any(gt_boxes[s, j] != 0)]
        base, vb = base_xyz[s].astype(f32), vote_base[s].astype(f32)
        if not valid:
            out["nmask"][s] = 1
            continue
        hit = np.full(N, -1)
        vhit = np.full(NV, -1)
        for j in valid:
            m = inside(base, *box_planes(gt_boxes[s, j]))
            hit[(hit < 0) & m] = j
            vm = inside(vb, *box_planes(gt_boxes[s, j], EXPAND))
            vhit[(vhit < 0) & vm] = j
        first = valid[0]
        for p in range(N):
            a = hit[p] if hit[p] >= 0 else first
            bx = gt_boxes[s, a].astype(f32)
            d = base[p] - bx[:3]
            dist = np.sqrt(f32(f32(d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]))
            pos = hit[p] >= 0 and dist <= SAMPLE_RANGE
            out["assigned_idx"][s, p] = a
            out["assigned_box"][s, p] = bx
            out["pmask"][s, p] = pos
            out["nmask"][s, p] = hit[p] < 0
            if pos and gt_labels[s, a] == 1:
                out["cls_label"][s, p] = centerness(base[p], bx)
            out["angle_bin"][s, p], out["angle_res"][s, p] = encode_angle(bx[6], nbins)
            hh = bx[4] * f32(0.5)
            out["offset_target"][s, p] = (bx[0] - base[p, 0], (bx[1] - hh) - base[p, 1], bx[2] - base[p, 2],
                                          bx[3] * f32(0.5), hh, bx[5] * f32(0.5))
        for p in range(NV):
            a = vhit[p] if vhit[p] >= 0 else first
            bx = gt_boxes[s, a].astype(f32)
            out["vote_mask"][s, p] = vhit[p] >= 0
            out["vote_target"][s, p] = (bx[0] - vb[p, 0], (bx[1] - bx[4] / f32(2)) - vb[p, 1], bx[2] - vb[p, 2])
    return out


def huber(e):
    a = np.abs(e)
    q = np.minimum(a, 1.0)
    return 0.5 * q * q + (a - q)


def corners(ctr, lhw, ang):
    """get_box3d_corners_helper in float64: ctr [P, 3], lhw [P, 3], ang [P] -> [P, 8, 3]."""
    c, s = np.cos(ang)[:, None], np.sin(ang)[:, None]
    xc, yc, zc = SX[None] * lhw[:, :1] / 2, np.where(np.arange(8)[None] >= 4, -lhw[:, 1:2], 0.0), SZ[None] * lhw[:, 2:3] / 2
    return np.stack([c * xc + s * zc + ctr[:, :1], yc + ctr[:, 1:2], -s * xc + c * zc + ctr[:, 2:3]], axis=-1)


def interval(nbins=12):
    return np.float64(f32(2 * np.pi / nbins))


def losses(base_xyz, pred_cls, pred_offset, pred_angle_cls, pred_angle_res, vote_offset, tg, nbins=12):
    """float64 loss (6,) and norm (3,) of ssd3d_det_loss.  Head outputs as (B, N, [1,] C)."""
    B, N = base_xyz.shape[:2]
    d = lambda t: np.asarray(t, np.float64).reshape(B, -1, np.asarray(t).shape[-1])
    x, off, lg, rs, vo = d(pred_cls)[..., 0], d(pred_offset), d(pred_angle_cls), d(pred_angle_res), d(vote_offset)
    pm, nm = tg["pmask"].astype(np.float64), tg["nmask"].astype(np.float64)
    cm = pm + nm
    z = tg["cls_label"].astype(np.float64)
    part = np.zeros((B, 9))
    part[:, 0] = ((np.maximum(x, 0) - x * z + np.log1p(np.exp(-np.abs(x)))) * cm).sum(1)
    part[:, 1] = (huber(off - tg["offset_target"]).sum(-1) * pm).sum(1)
    bin_ = tg["angle_bin"]
    mx = lg.max(-1)
    lse = mx + np.log(np.exp(lg - mx[..., None]).sum(-1))
    part[:, 2] = ((lse - np.take_along_axis(lg, bin_[..., None], -1)[..., 0]) * pm).sum(1)
    res = np.take_along_axis(rs, bin_[..., None], -1)[..., 0]
    part[:, 3] = huber((res - tg["angle_res"]) * pm).sum(1)
    pc, gc, _ = _corners_pred_gt(base_xyz, off, res, tg, nbins)
    part[:, 4] = (huber(pc - gc).sum((-1, -2)).reshape(B, N) * pm).sum(1)
    vm = tg["vote_mask"].astype(np.float64)
    part[:, 5] = (huber(tg["vote_target"] - vo).sum(-1) * vm).sum(1)
    part[:, 6], part[:, 7], part[:, 8] = cm.sum(1), pm.sum(1), vm.sum(1)
    tot = part.sum(0)
    norm = np.maximum(1.0, tot[6:9])
    return tot[:6] / norm[[0, 1, 1, 1, 1, 2]], norm


def _corners_pred_gt(base_xyz, off, res, tg, nbins):
    B, N = base_xyz.shape[:2]
    o = off.reshape(-1, 6)
    base = base_xyz.reshape(-1, 3).astype(np.float64)
    ctr = base + o[:, :3]
    ctr[:, 1] += o[:, 4]
    two = (off.astype(f32) * f32(2.0)).reshape(-1, 6)[:, 3:6]
    pas = two >= f32(0.1)
    lhw = np.where(pas, two.astype(np.float64), np.float64(f32(0.1)))
    ang = (tg["angle_bin"].reshape(-1) + res.reshape(-1)) * interval(nbins)
    bx = tg["assigned_box"].reshape(-1, 7).astype(np.float64)
    return corners(ctr, lhw, ang), corners(bx[:, :3], bx[:, 3:6], bx[:, 6]), (pas, lhw, ang)
