"""Generates tests/golden/det_targets.npz by executing the REFERENCE's own numpy target functions on seeded scenes.

The reference modules import tensorflow / numba at the top, so the functions are pulled out of their source files with
`ast` and executed as they are (nothing is copied into this repo):
  lib/utils/voxelnet_aug.py         check_inside_points and its chain (center_to_corner_box3d, corners_nd,
                                    rotation_3d_in_axis, corner_to_surfaces_3d_jit, surface_equ_3d_jit,
                                    points_in_convex_polygon_3d_jit)
  lib/np_functions/gt_sampler.py    mask_assign_targets_anchors_np, vote_targets_np
  lib/utils/anchor_encoder.py       encode_angle2class_np, encode_dist_anchor_free_np
  lib/utils/box_3d_utils.py         get_box3d_corners_helper_np
numba.jit / numba.njit are replaced by identity decorators (numba 0.65 has no object mode, which
surface_equ_3d_jit's np.einsum needs) and np.int is supplied as int for encode_angle2class_np (numpy 2).
The scenes hold overlapping boxes, points exactly on faces, points only inside the 0.1 expansion, positives beyond
10 m, angles on the bin edges and +-pi, and one scene of padded rows only, whose expected answer (the reference's
argmax raises on it) is written by hand.  Each point's float64 distance to the nearest face plane of any box is
recorded so a test can leave out the points a float32 rounding may put on either side.
Needs a reference checkout (path in $REFERENCE):   REFERENCE=<checkout> python tests/golden/make_golden_det_targets.py
"""
import ast
import os
import types

import numpy as np

REF = os.path.join(os.environ.get("REFERENCE", "."), "lib")
HERE = os.path.dirname(os.path.abspath(__file__))
N, NV, G, B = 256, 256, 12, 4
EXPAND = 0.1


def pull(path, names, env):
    tree = ast.parse(open(path).read())
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name in names:
            exec(compile(ast.Module([node], []), path, "exec"), env)


def _jit(*a, **k):
    if len(a) == 1 and callable(a[0]) and not k:
        return a[0]
    return lambda f: f


def reference_env():
    np.int = int
    cfg = types.SimpleNamespace(TRAIN=types.SimpleNamespace(AUGMENTATIONS=types.SimpleNamespace(EXPAND_DIMS_LENGTH=EXPAND)))
    env = {"np": np, "numba": types.SimpleNamespace(jit=_jit, njit=_jit), "cfg": cfg}
    pull(os.path.join(REF, "utils", "voxelnet_aug.py"),
         {"check_inside_points", "center_to_corner_box3d", "corners_nd", "rotation_3d_in_axis", "corner_to_surfaces_3d_jit",
          "surface_equ_3d_jit", "points_in_convex_polygon_3d_jit"}, env)
    pull(os.path.join(REF, "np_functions", "gt_sampler.py"), {"mask_assign_targets_anchors_np", "vote_targets_np"}, env)
    pull(os.path.join(REF, "utils", "anchor_encoder.py"), {"encode_angle2class_np", "encode_dist_anchor_free_np"}, env)
    pull(os.path.join(REF, "utils", "box_3d_utils.py"), {"get_box3d_corners_helper_np"}, env)
    return env


def to_world(box, u):
    """canonical (x, y, z) offsets of a box (y up is negative, bottom at 0) -> camera frame, float64."""
    c, s = np.cos(box[6]), np.sin(box[6])
    return np.stack([c * u[:, 0] + s * u[:, 2] + box[0], u[:, 1] + box[1], -s * u[:, 0] + c * u[:, 2] + box[2]], 1)


def face_distance(pts, boxes, expand):
    """float64 distance of each point to the nearest face plane of any valid box (grown by `expand`)."""
    best = np.full(len(pts), np.inf)
    for b in boxes:
        if not np.any(b != 0):
            continue
        b = b.astype(np.float64)
        l, h, w = b[3] + expand, b[4] + expand, b[5] + expand
        c, s = np.cos(b[6]), np.sin(b[6])
        e = pts.astype(np.float64) - b[:3]
        cx, cy, cz = c * e[:, 0] - s * e[:, 2], e[:, 1], s * e[:, 0] + c * e[:, 2]
        d = np.min(np.abs(np.stack([cx - l / 2, cx + l / 2, cy, cy + h, cz - w / 2, cz + w / 2], 1)), 1)
        best = np.minimum(best, d)
    return best


def scenes():
    rng = np.random.default_rng(2026)
    per = 2 * np.pi / 12
    boxes = np.zeros((B, G, 7), np.float32)
    labels = np.zeros((B, G), np.int32)
    base = np.zeros((B, N, 3), np.float32)
    vote = np.zeros((B, NV, 3), np.float32)
    for s in range(B - 1):                                    # the last scene keeps only padded rows
        g = G - 2 * s
        for j in range(g):
            l, h, w = rng.uniform(3.2, 4.7), rng.uniform(1.4, 1.8), rng.uniform(1.5, 1.9)
            if j == 1:
                l = 26.0                                      # a long box: inside but beyond 10 m of its centre
            ry = rng.uniform(-np.pi, np.pi)
            if j % 3 == 0:
                ry = (j // 3) * per - per / 2                 # bin edges
            if j == 2:
                ry = np.pi if s % 2 == 0 else -np.pi
            if j == 4:
                ry = 0.0                                      # axis-aligned: exact corners, points exactly on faces
            ctr = (rng.uniform(-20, 20), 1.65, rng.uniform(5, 50))
            if j == 3:                                        # overlaps box 0
                ctr = (boxes[s, 0, 0] + 1.0, boxes[s, 0, 1], boxes[s, 0, 2] + 0.5)
            boxes[s, j] = (*ctr, l, h, w, ry)
            labels[s, j] = 1 if j != 5 else 2
        if s == 1:
            boxes[s, [2, 6]] = 0                              # padding between valid rows
            labels[s, [2, 6]] = 0
        for pts, n in ((base, N), (vote, NV)):
            k = 0
            for j in range(g):
                b = boxes[s, j].astype(np.float64)
                if not np.any(b != 0):
                    continue
                m = 14
                u = rng.uniform(-0.5, 0.5, (m, 3)) * [b[3], 0, b[5]]
                u[:, 1] = -rng.uniform(0, 1, m) * b[4]
                u[:4, 0] = np.sign(u[:4, 0]) * b[3] / 2           # exactly on the l faces (exact when ry = 0)
                u[4:6, 1] = [0.0, -b[4]]                          # on the bottom / top
                u[6:9, 0] = np.sign(u[6:9, 0]) * (b[3] / 2 + rng.uniform(0.001, 0.049, 3))   # only in the expansion
                u[9, 1] = 0.03                                    # below the bottom, inside the expansion
                pts[s, k:k + m] = to_world(b, u)
                k += m
            rest = n - k
            pts[s, k:] = np.stack([rng.uniform(-25, 25, rest), rng.uniform(0.0, 1.7, rest), rng.uniform(3, 55, rest)], 1)
            pts[s, k] = (0.0, 1.0, 20.0)                          # a negative with canonical x = 0 (the NaN of the reference)
    base[B - 1] = base[0]
    vote[B - 1] = vote[0]
    return base, vote, boxes, labels


def main():
    env = reference_env()
    base, vote, boxes, labels = scenes()
    idx, pm, nm = np.zeros((B, N), np.int32), np.zeros((B, N), np.float32), np.zeros((B, N), np.float32)
    vmask, vtarget = np.zeros((B, NV), np.float32), np.zeros((B, NV, 3), np.float32)
    ref = slice(0, B - 1)
    i, p, n = env["mask_assign_targets_anchors_np"](base[ref], base[ref][:, :, None, :], boxes[ref], labels[ref], -1, 0.5, 0.6, 0.45,
                                                   10.0, np.ones((B - 1, N, 1), np.float32))
    idx[ref], pm[ref], nm[ref] = i[..., 0], p[..., 0], n[..., 0]
    vm, vt = env["vote_targets_np"](vote[ref], boxes[ref])
    vmask[ref], vtarget[ref] = vm, vt
    nm[B - 1] = 1.0                                           # padded rows only: all negatives, zero targets (by hand)
    abox = np.take_along_axis(boxes, idx[..., None].astype(np.int64), 1)
    abox[B - 1] = 0
    ang_bin, ang_res = env["encode_angle2class_np"](abox[..., 6], 12)
    ctr, off = env["encode_dist_anchor_free_np"](abox[..., :3], abox[..., 3:6], base)
    ctr[B - 1] = 0                                            # by hand: zero targets without a valid box
    corners = env["get_box3d_corners_helper_np"](abox.reshape(-1, 7)[:, :3], abox.reshape(-1, 7)[:, 6], abox.reshape(-1, 7)[:, 3:6])
    fdist = np.stack([face_distance(base[s], boxes[s], 0.0) for s in range(B)])
    vdist = np.stack([face_distance(vote[s], boxes[s], EXPAND) for s in range(B)])
    np.savez_compressed(os.path.join(HERE, "det_targets.npz"), base_xyz=base, vote_base=vote, gt_boxes=boxes, gt_labels=labels,
                        assigned_idx=idx, pmask=pm, nmask=nm, vote_mask=vmask, vote_target=vtarget,
                        angle_bin=np.asarray(ang_bin, np.int32), angle_res=np.asarray(ang_res, np.float64),
                        encoded_ctr=np.asarray(ctr, np.float32), encoded_half=np.asarray(off, np.float32),
                        corners=np.asarray(corners, np.float32).reshape(B, N, 8, 3), face_dist=fdist, vote_face_dist=vdist)
    print("wrote det_targets.npz: pos %d neg %d vote %d" % (pm.sum(), nm.sum(), vmask.sum()))


if __name__ == "__main__":
    main()
