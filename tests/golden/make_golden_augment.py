"""Generates tests/golden/augment.npz by executing the REFERENCE's own augmentation on recorded draws.

DataAugmentor.kitti_forward (lib/builder/data_augmentor.py) and the chain it calls are pulled out of their source files
with `ast` and executed as they are (nothing is copied into this repo):
  lib/builder/data_augmentor.py  DataAugmentor (kitti_forward only; the instance is made without __init__, mixup off)
  lib/utils/kitti_aug.py         flip_points, flip_boxes_3d
  lib/utils/rotation_util.py     roty
  lib/utils/voxelnet_aug.py      noise_per_object_v3_, noise_per_box, box2d_to_corner_jit, box_collision_test,
                                 corner_to_standup_nd_jit, _rotation_box2d_jit_, _select_transform, points_transform_,
                                 _rotation_matrix_3d_, box3d_transform_, filter_points_boxes_3d, check_inside_points and
                                 the corner / surface chain of make_golden_det_targets.py
numba.jit / numba.njit become identity decorators.  numba compiles `flag is True` / `flag is False` on a boolean array
element as a comparison of values, which plain Python does not (a numpy bool is never the object True), so those
comparisons are rewritten to == / != before execution; nothing else is changed.  np.random is replaced by a stub that
hands out the recorded draws in call order: rand() the flip draw, rand(3) the three choices, then the rotation and scale
draws when their choice fires; normal(scale, size) = 0 + scale * the recorded (x, z) normals; uniform(lo, hi, size)
= lo + (hi - lo) * the recorded rotation draws (the per-object scale range is [1, 1]).  Each point carries its index in
points[:, 4] (float32, exact) so that the survivors can be matched.

Recorded besides the outputs: the try each box took (noise_per_box's return), the same search run in float64 (boxes
whose float32 and float64 decisions differ are near-ties), the box whose pre-noise grown corners hold each moved point
(points_transform_'s masks) and each point's float64 distance to the nearest face of those grown boxes.
Scenes: choice draws exactly at 0.5 with ry of 0, +-pi and bin edges; a packed 5 x 5 grid of cars whose first box
takes its last try and whose centre box exhausts all 100; a scene without boxes whose positives lie outside every box;
two overlapping boxes sharing points; a KITTI-like scene.
Needs a reference checkout (path in $REFERENCE):   REFERENCE=<checkout> python tests/golden/make_golden_augment.py
"""
import ast
import importlib
import os
import sys
import types

import numpy as np

REF = os.path.join(os.environ.get("REFERENCE", "."), "lib")
HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
TRIES, M = 100, 1024


class _IsToEq(ast.NodeTransformer):
    def visit_Compare(self, node):
        self.generic_visit(node)
        if len(node.ops) == 1 and isinstance(node.comparators[0], ast.Constant) and isinstance(node.comparators[0].value, bool):
            if isinstance(node.ops[0], ast.Is):
                node.ops = [ast.Eq()]
            elif isinstance(node.ops[0], ast.IsNot):
                node.ops = [ast.NotEq()]
        return node


def pull(path, names, env):
    tree = ast.parse(open(path).read())
    for node in tree.body:
        if isinstance(node, (ast.FunctionDef, ast.ClassDef)) and node.name in names:
            mod = ast.fix_missing_locations(_IsToEq().visit(ast.Module([node], [])))
            exec(compile(mod, path, "exec"), env)


def _jit(*a, **k):
    if len(a) == 1 and callable(a[0]) and not k:
        return a[0]
    return lambda f: f


class RandomStub:
    """np.random for one call of kitti_forward, handing out the recorded draws."""

    def __init__(self, u, loc, rot_u):
        self.u, self.loc, self.rot_u = u, loc, rot_u
        self.queue = [u[0]] + ([u[4]] if u[2] <= 0.5 else []) + ([u[5]] if u[3] <= 0.5 else [])

    def rand(self, *size):
        if size == (3,):
            return np.array(self.u[1:4], np.float64)
        assert not size
        return float(self.queue.pop(0))

    def normal(self, loc=0.0, scale=1.0, size=None):
        z = np.zeros(size)
        z[..., :2] = self.loc[:size[0]]
        return loc + scale * z

    def uniform(self, low=0.0, high=1.0, size=None):
        if size[-1] == 1:
            assert low == high
            return low + (high - low) * np.zeros(size)
        return low + (high - low) * self.rot_u[:size[0]]


class NumpyWithRandom:
    def __init__(self, rnd):
        self.random = rnd

    def __getattr__(self, k):
        return getattr(np, k)


def cfg_namespace():
    ns = types.SimpleNamespace
    single = ns(ROTATION_PERTURB=[-np.pi / 3, np.pi / 3], CENTER_NOISE_STD=[1.0, 1.0, 0.], RANDOM_SCALE_RANGE=[1.0, 1.0],
                SCALE_3_DIMS=False, FIX_LENGTH=False)
    aug = ns(OPEN=True, EXPAND_DIMS_LENGTH=0.1, PROB_TYPE="Simultaneously", PROB=[0.5, 0.5, 0.5],
             RANDOM_ROTATION_RANGE=45 / 180 * np.pi, RANDOM_SCALE_RANGE=0.1, FLIP=True, MIXUP=ns(OPEN=False), SINGLE_AUG=single)
    return ns(TRAIN=ns(AUGMENTATIONS=aug))


def reference(u, loc, rot_u, record, no_boxes=False):
    """A DataAugmentor whose np.random hands out (u, loc, rot_u); calls of noise_per_box / points_transform_ are
    recorded into `record`.  no_boxes: the filter's max over an empty box axis raises (the reference's loader never
    makes such a frame), so there it keeps every point, which is what it means."""
    npx = NumpyWithRandom(RandomStub(u, loc, rot_u))
    env = {"np": npx, "numba": types.SimpleNamespace(jit=_jit, njit=_jit), "cfg": cfg_namespace()}
    va = os.path.join(REF, "utils", "voxelnet_aug.py")
    pull(va, {"noise_per_object_v3_", "noise_per_box", "box2d_to_corner_jit", "box_collision_test", "corner_to_standup_nd_jit",
              "_rotation_box2d_jit_", "_select_transform", "points_transform_", "_rotation_matrix_3d_", "box3d_transform_",
              "filter_points_boxes_3d", "check_inside_points", "center_to_corner_box3d", "corners_nd", "rotation_3d_in_axis",
              "corner_to_surfaces_3d_jit", "surface_equ_3d_jit", "points_in_convex_polygon_3d_jit"}, env)
    nb, pt = env["noise_per_box"], env["points_transform_"]

    def noise_per_box(boxes, *a):
        out = nb(boxes, *a)
        record["chosen"] = out.copy()
        record["chosen64"] = nb(boxes.astype(np.float64), *a)          # the same search in float64
        return out

    def points_transform_(points, centers, point_masks, *a):
        record["masks"] = point_masks.copy()
        return pt(points, centers, point_masks, *a)

    env["noise_per_box"], env["points_transform_"] = noise_per_box, points_transform_
    if no_boxes:
        env["filter_points_boxes_3d"] = lambda boxes, points, sem, dists, enlarge_range: (boxes, points, sem, dists)
    kenv = {"np": npx}
    pull(os.path.join(REF, "utils", "kitti_aug.py"), {"flip_points", "flip_boxes_3d"}, kenv)
    renv = {"np": npx}
    pull(os.path.join(REF, "utils", "rotation_util.py"), {"roty"}, renv)
    env["kitti_aug"] = types.SimpleNamespace(flip_points=kenv["flip_points"], flip_boxes_3d=kenv["flip_boxes_3d"])
    env["rotation_util"] = types.SimpleNamespace(roty=renv["roty"])
    pull(os.path.join(REF, "builder", "data_augmentor.py"), {"DataAugmentor"}, env)
    aug = object.__new__(env["DataAugmentor"])
    aug.aug_flip, aug.aug_flip_prob, aug.mixup, aug.single_aug_prob = True, 0.5, False, [0.5, 0.5, 0.5]
    return aug, env


def face_distance(pts, boxes, expand):
    """float64 distance of each point to the nearest face plane of any valid box grown by `expand`."""
    best = np.full(len(pts), np.inf)
    for b in boxes:
        if not np.any(b != 0):
            continue
        b = b.astype(np.float64)
        l, h, w = b[3] + expand, b[4] + expand, b[5] + expand
        c, s = np.cos(b[6]), np.sin(b[6])
        e = pts.astype(np.float64) - b[:3]
        cx, cy, cz = c * e[:, 0] - s * e[:, 2], e[:, 1], s * e[:, 0] + c * e[:, 2]
        best = np.minimum(best, np.min(np.abs(np.stack([cx - l / 2, cx + l / 2, cy, cy + h, cz - w / 2, cz + w / 2], 1)), 1))
    return best


def car(x, z, ry, rng, y=1.65):
    return (x, y, z, rng.uniform(3.6, 4.2), rng.uniform(1.45, 1.7), rng.uniform(1.55, 1.8), ry)


def points_for(boxes, n_box, n_bg, rng, spread=(-30, 30, 3, 60)):
    """Points on and in the boxes (canonical offsets), a ring just outside them and a background."""
    out = []
    for b in boxes:
        u = rng.uniform(-0.5, 0.5, (n_box, 3))
        u[:, 1] = -rng.uniform(0, 1, n_box)
        u[: n_box // 4, 0] *= 1.2                                         # some in the 0.1 / 0.5 margins
        c, s = np.cos(b[6]), np.sin(b[6])
        cx, cy, cz = u[:, 0] * b[3], u[:, 1] * b[4], u[:, 2] * b[5]
        out.append(np.stack([c * cx + s * cz + b[0], cy + b[1], -s * cx + c * cz + b[2]], 1))
    out.append(np.stack([rng.uniform(spread[0], spread[1], n_bg), rng.uniform(0.0, 1.7, n_bg),
                         rng.uniform(spread[2], spread[3], n_bg)], 1))
    p = np.concatenate(out).astype(np.float32)
    return np.concatenate([p, rng.uniform(0, 1, (len(p), 1)).astype(np.float32)], 1)


def scenes():
    """(points [N, 4], boxes [G, 7], scene_u [6], loc [G, 100, 2], rot_u [G, 100], positives outside the boxes?)"""
    rng = np.random.default_rng(2026)
    per = 2 * np.pi / 12
    out = []
    # 1: every choice draw exactly at 0.5, angles 0, +-pi and bin edges
    ang = [0.0, np.pi, -np.pi, per / 2, -per / 2, 3 * per / 2, np.pi - per / 2, -np.pi + per / 2]
    b = np.array([car(-25 + 7 * i, 8 + 6 * (i % 3), a, rng) for i, a in enumerate(ang)], np.float32)
    out.append((points_for(b, 60, 600, rng), b, np.array([0.5, 0.5, 0.5, 0.5, 0.3, 0.8]), rng.standard_normal((8, TRIES, 2)),
                rng.uniform(size=(8, TRIES)), False))
    # 2: a packed 5 x 5 grid: box 0 collides on tries 0..98 and escapes on 99, the centre box (12) exhausts its tries
    b = np.array([(-10 + 4.3 * (k % 5), 1.65, 20 + 2.1 * (k // 5), 3.9, 1.6, 1.7, 0.0) for k in range(25)], np.float32)
    loc = rng.standard_normal((25, TRIES, 2))
    rot = rng.uniform(size=(25, TRIES))
    for k in (0, 12):
        loc[k] *= 0.05
        rot[k] = rng.uniform(0.8, 1.0, TRIES)
    loc[0, 99] = (-15.0, -15.0)
    out.append((points_for(b, 40, 500, rng, (-15, 15, 15, 35)), b, np.array([0.2, 0.1, 0.9, 0.3, 0.6, 0.25]), loc, rot, False))
    # 3: no boxes; positives outside every box
    p = points_for(np.zeros((0, 7)), 0, 800, rng)
    out.append((p, np.zeros((0, 7), np.float32), np.array([0.7, 0.9, 0.2, 0.4, 0.9, 0.1]), np.zeros((0, TRIES, 2)),
                np.zeros((0, TRIES)), True))
    # 4: two overlapping boxes share points (the first moves them), a third elsewhere, positives outside
    b = np.array([car(0.0, 20.0, 0.3, rng), car(0.8, 20.4, 0.5, rng), car(-12.0, 35.0, -2.0, rng)], np.float32)
    out.append((points_for(b, 120, 500, rng), b, np.array([0.9, 0.2, 0.1, 0.7, 0.15, 0.5]), rng.standard_normal((3, TRIES, 2)),
                rng.uniform(size=(3, TRIES)), True))
    # 5: KITTI-like
    synth = importlib.import_module("3dssd_b200.synth")
    p, b, l = synth.kitti_like_with_boxes(1, 4000, 15, seed=77)
    b = b[0][l[0] > 0]
    out.append((p[0], b, np.array([0.6, 0.4, 0.3, 0.2, 0.05, 0.95]), rng.standard_normal((len(b), TRIES, 2)),
                rng.uniform(size=(len(b), TRIES)), False))
    return out


def main():
    sc = scenes()
    B, G = len(sc), max(len(s[1]) for s in sc)
    rng = np.random.default_rng(7)
    pts, sems, mover, fdist, rpts, ridx = [], [], [], [], [], []
    boxes, labels = np.zeros((B, G, 7), np.float32), np.zeros((B, G), np.int32)
    rboxes = np.zeros((B, G, 7), np.float32)
    chosen, chosen64 = np.full((B, G), -1, np.int32), np.full((B, G), -1, np.int32)
    scene_u, loc, rot_u = np.zeros((B, 6)), np.zeros((B, G, TRIES, 2)), np.zeros((B, G, TRIES))
    for s, (p, b, u, lo, ro, pos_outside) in enumerate(sc):
        g, n = len(b), len(p)
        boxes[s, :g], labels[s, :g], scene_u[s], loc[s, :g], rot_u[s, :g] = b, 1, u, lo, ro
        env0 = reference(u, lo, ro, {})[1]
        sem = (env0["check_inside_points"](p, np.concatenate([b[:, :3], b[:, 3:6] + 0.1, b[:, 6:]], 1)).any(1).astype(np.int64)
               if g else np.zeros(n, np.int64))
        if pos_outside:
            sem[rng.choice(n, 40, replace=False)] = 1
        rec = {}
        aug, _ = reference(u, lo, ro, rec, no_boxes=g == 0)
        src = np.concatenate([p, np.arange(n, dtype=np.float32)[:, None]], 1)
        o_pts, o_sem, _, o_boxes, _ = aug.kitti_forward(src.copy(), sem.copy(), np.ones(n, np.float32), b.copy(), np.ones(g, np.int64),
                                                        None, 0)
        flipped = p[:, :3].copy()
        if u[0] >= 0.5:
            flipped[:, 0] = -flipped[:, 0]
        fb = b.copy()
        if u[0] >= 0.5 and g:
            fb = reference(u, lo, ro, {})[1]["kitti_aug"].flip_boxes_3d(b)
        mv = np.full(n, -1, np.int32)
        if "masks" in rec and rec["masks"].shape[1]:
            m = rec["masks"]
            pos = np.flatnonzero(sem)
            hit = m.any(1)
            mv[pos[hit]] = np.argmax(m[hit], 1)
        if "chosen" in rec:
            chosen[s, :g], chosen64[s, :g] = rec["chosen"], rec["chosen64"]
        pts.append(p)
        sems.append(sem.astype(np.int32))
        mover.append(mv)
        fdist.append(face_distance(flipped, fb, 0.1))
        rpts.append(np.asarray(o_pts[:, :4], np.float64))
        ridx.append(np.asarray(o_pts[:, 4]).astype(np.int64))
        rboxes[s, :g] = o_boxes
        print("scene %d: %d boxes, %d -> %d points, flags %s, tries %s" % (s, g, n, len(o_pts), (u[:4] >= 0.5).astype(int),
                                                                           chosen[s, :g].tolist()))
    off = np.concatenate([[0], np.cumsum([len(p) for p in pts])]).astype(np.int32)
    roff = np.concatenate([[0], np.cumsum([len(p) for p in rpts])]).astype(np.int32)
    T = int(off[-1])
    np.savez_compressed(os.path.join(HERE, "augment.npz"), points=np.concatenate(pts), offsets=off, sem_labels=np.concatenate(sems),
                        gt_boxes=boxes, gt_labels=labels, scene_u=scene_u, loc_noise=loc, rot_u=rot_u,
                        keys=rng.integers(0, 2 ** 32, T).astype(np.uint32).view(np.int32),
                        refill=rng.integers(0, 2 ** 32, (B, M)).astype(np.uint32).view(np.int32),
                        ref_points=np.concatenate(rpts), ref_index=np.concatenate(ridx), ref_offsets=roff, ref_boxes=rboxes,
                        ref_chosen=chosen, ref_chosen64=chosen64, ref_moved_by=np.concatenate(mover), face_dist=np.concatenate(fdist))
    print("wrote augment.npz")


if __name__ == "__main__":
    main()
