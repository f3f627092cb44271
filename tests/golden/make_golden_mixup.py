"""Generates tests/golden/mixup.npz by executing the REFERENCE's own mixup code on designed frames.

Pulled out of their source files with `ast` (make_golden_augment.pull, its numba and np.random stubs; nothing is copied
into this repo) and executed as they are:
  lib/dataset/dataloader/kitti_dataloader.py  KittiDataset.generate_mixup_sample (the method alone) with
                                              check_inside_points and its corner / surface chain
  lib/utils/voxelnet_aug.py                   box_3d_collision_test, box2d_to_corner_jit, box_collision_test
  lib/builder/mixup_sampler.py                MixupSampler._sample / _reset (np.random.shuffle hands out recorded
                                              permutations)
  lib/utils/kitti_util.py                     get_road_plane on written plane files
  lib/builder/data_augmentor.py               DataAugmentor.kitti_forward with mixup on, its sampler returning the
                                              database dicts of recorded ids
Frames and boxes are float32, as this project holds them.  Database frames: a box holding exactly 5 points and one
holding 4, two overlapping boxes sharing points, a row of another class, a KITTI-like frame.  Paste scenes: a drawn box
abutting a scene box (standup overlap 0), one containing a scene box and one contained in one, two overlapping drawn
boxes (the first kept, then the first dropped), every drawn object dropped, a scene without GT rows, tilted planes, a
KITTI-like scene.  Each pasted point carries its slot in the pasted layout in points[:, 4] so the survivors can be
matched.
Needs a reference checkout (path in $REFERENCE):   REFERENCE=<checkout> python tests/golden/make_golden_mixup.py
"""
import ast
import importlib
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_augment as MGA  # noqa: E402

REF = MGA.REF
TRIES, M, S = 100, 1024, 15
KEYS = types.SimpleNamespace(KEY_SAMPLED_GT_POINTS="sampled_gt_points", KEY_SAMPLED_GT_LABELS_3D="sampled_gt_labels_3d",
                             KEY_SAMPLED_GT_CLSES="sampled_gt_classes", KEY_LABEL_BOXES_3D="label_boxes_3d",
                             KEY_LABEL_CLASSES="label_classes", KEY_POINT_CLOUD="point_cloud")
CORNER_CHAIN = {"check_inside_points", "center_to_corner_box3d", "corners_nd", "rotation_3d_in_axis", "corner_to_surfaces_3d_jit",
                "surface_equ_3d_jit", "points_in_convex_polygon_3d_jit"}


def pull_method(path, cls, name, env):
    tree = ast.parse(open(path).read())
    for node in tree.body:
        if isinstance(node, ast.ClassDef) and node.name == cls:
            for f in node.body:
                if isinstance(f, ast.FunctionDef) and f.name == name:
                    exec(compile(ast.fix_missing_locations(ast.Module([f], [])), path, "exec"), env)
                    return env[name]
    raise KeyError(name)


def base_env(rnd=None):
    npx = MGA.NumpyWithRandom(rnd) if rnd is not None else np
    env = {"np": npx, "numba": types.SimpleNamespace(jit=MGA._jit, njit=MGA._jit), "maps_dict": KEYS}
    MGA.pull(os.path.join(REF, "utils", "voxelnet_aug.py"), CORNER_CHAIN | {"box_3d_collision_test", "box2d_to_corner_jit",
                                                                             "box_collision_test", "corner_to_standup_nd_jit"}, env)
    return env


def ref_db(frames):
    """generate_mixup_sample over the frames -> the Car dicts in frame order, and per frame the row of each."""
    env = base_env()
    env["cfg"] = types.SimpleNamespace(TRAIN=types.SimpleNamespace(AUGMENTATIONS=types.SimpleNamespace(EXPAND_DIMS_LENGTH=0.1)),
                                       DATASET=types.SimpleNamespace(MIN_POINTS_NUM=5))
    gen = pull_method(os.path.join(REF, "dataset", "dataloader", "kitti_dataloader.py"), "KittiDataset", "generate_mixup_sample", env)
    me = types.SimpleNamespace(idx2cls_dict={1: "Car", 2: "Pedestrian"})
    out, src = [], []
    for f, (p, b, l) in enumerate(frames):
        ds = gen(me, {KEYS.KEY_LABEL_BOXES_3D: b.copy(), KEYS.KEY_LABEL_CLASSES: l.copy(), KEYS.KEY_POINT_CLOUD: p.copy()}) or []
        valid = np.flatnonzero(env["check_inside_points"](p, np.concatenate([b[:, :3], b[:, 3:6] + 0.1, b[:, 6:]], 1)).sum(0) >= 5)
        for d, j in zip(ds, valid):
            if d[KEYS.KEY_SAMPLED_GT_CLSES] == "Car":
                out.append(d)
                src.append((f, j))
    return out, np.asarray(src, np.int32)


def ref_sampler(count, num, calls, rng):
    """MixupSampler._sample / _reset over `calls` calls; np.random.shuffle hands out recorded permutations."""
    perms = []

    class Rnd:
        @staticmethod
        def shuffle(v):
            perms.append(rng.permutation(len(v)))
            v[:] = perms[-1]

    env = {"np": MGA.NumpyWithRandom(Rnd())}
    MGA.pull(os.path.join(REF, "builder", "mixup_sampler.py"), {"MixupSampler"}, env)
    smp = object.__new__(env["MixupSampler"])
    smp.sample_num_list, smp.sv_perm, smp.sv_idx_list, smp._shuffle = {"Car": count}, {"Car": np.arange(count)}, {"Car": 0}, True
    Rnd.shuffle(smp.sv_perm["Car"])
    rets = [smp._sample(num, "Car").copy() for _ in range(calls)]
    return rets, perms


def ref_planes(rows):
    env = {"np": np}
    MGA.pull(os.path.join(REF, "utils", "kitti_util.py"), {"get_road_plane"}, env)
    d = tempfile.mkdtemp()
    for i, r in enumerate(rows):
        with open(os.path.join(d, "%06d.txt" % i), "w") as fh:
            fh.write("# Plane\nWidth 4\nHeight 1\n%s\n" % " ".join("%.6e" % v for v in r))
    texts = [open(os.path.join(d, "%06d.txt" % i)).read() for i in range(len(rows))]
    return np.stack([env["get_road_plane"](i, d) for i in range(len(rows))]), texts


def inside_pts(box, n, rng, frac=0.45):
    u = rng.uniform(-frac, frac, (n, 3))
    u[:, 1] = -rng.uniform(0.05, 0.95, n)
    c, s = np.cos(box[6]), np.sin(box[6])
    cx, cy, cz = u[:, 0] * box[3], u[:, 1] * box[4], u[:, 2] * box[5]
    p = np.stack([c * cx + s * cz + box[0], cy + box[1], -s * cx + c * cz + box[2], rng.uniform(0, 1, n)], 1)
    return p.astype(np.float32)


def db_frames(rng):
    synth = importlib.import_module("3dssd_b200.synth")
    B = lambda *v: np.array(v, np.float32)
    abut, big, small = B(4.0, 1.6, 20.0, 3.5, 1.5, 1.5, 0.0), B(-20.0, 1.7, 30.0, 6.0, 1.6, 4.0, 0.3), B(20.0, 1.6, 30.0, 2.0, 1.5, 1.0, 0.0)
    p1, p2 = B(0.0, 1.65, 45.0, 4.0, 1.5, 1.8, 0.5), B(2.0, 1.6, 45.5, 4.0, 1.5, 1.8, 0.2)
    five, four, ped = B(-8.0, 1.7, 12.0, 3.8, 1.5, 1.6, -1.0), B(8.0, 1.7, 12.0, 3.8, 1.5, 1.6, 1.2), B(0.0, 1.7, 8.0, 0.8, 1.7, 0.6, 0.0)
    bg = lambda n: np.concatenate([rng.uniform(-35, 35, (n, 1)), rng.uniform(0.5, 1.7, (n, 1)), rng.uniform(55, 70, (n, 1)),
                                   rng.uniform(0, 1, (n, 1))], 1).astype(np.float32)
    f0 = (np.concatenate([inside_pts(abut, 40, rng), inside_pts(big, 60, rng), inside_pts(small, 12, rng), bg(50)]),
          np.stack([abut, big, small]), np.array([1, 1, 1], np.int64))
    f1 = (np.concatenate([inside_pts(p1, 50, rng), inside_pts(p2, 50, rng), inside_pts(five, 5, rng), inside_pts(four, 4, rng),
                          inside_pts(ped, 20, rng), bg(40)]), np.stack([p1, p2, five, four, ped]), np.array([1, 1, 1, 1, 2], np.int64))
    p, b, l = synth.kitti_like_with_boxes(1, 3000, 10, seed=91)
    v = l[0] > 0
    f2 = (p[0], b[0][v], l[0][v].astype(np.int64))
    return [f0, f1, f2], dict(abut=abut, big=big, small=small, p1=p1, p2=p2)


def paste_scenes(rng, obj):
    """(points [N, 4], boxes [G, 7], labels [G], names of the drawn objects, plane row)"""
    synth = importlib.import_module("3dssd_b200.synth")
    B = lambda *v: np.array(v, np.float32)
    bg = lambda n: np.concatenate([rng.uniform(-30, 30, (n, 1)), rng.uniform(0.5, 1.7, (n, 1)), rng.uniform(5, 60, (n, 1)),
                                   rng.uniform(0, 1, (n, 1))], 1).astype(np.float32)
    flat, tilt, tilt2, up = (0.0, -1.0, 0.0, 1.65), (0.02, -0.99, 0.015, 1.7), (-0.03, -1.02, 0.01, 1.6), (0.0, 1.0, 0.0, -1.65)
    sc = []
    b0 = np.stack([B(0.0, 1.65, 20.0, 4.0, 1.5, 2.0, 0.0), B(-20.0, 1.65, 30.0, 1.0, 1.5, 1.0, 0.0), B(20.0, 1.65, 30.0, 8.0, 1.5, 6.0, 0.0)])
    sc.append((np.concatenate([inside_pts(b, 30, rng) for b in b0] + [bg(300)]), b0, np.ones(3, np.int32), ["abut", "big", "small"], flat))
    b1 = np.stack([B(-15.0, 1.65, 10.0, 4.0, 1.5, 1.8, 1.0)])
    sc.append((np.concatenate([inside_pts(b1[0], 30, rng), bg(300)]), b1, np.ones(1, np.int32), ["p1", "p2"], tilt))
    b2 = np.stack([B(-2.0, 1.65, 45.0, 1.5, 1.5, 1.5, 0.0)])
    sc.append((np.concatenate([inside_pts(b2[0], 20, rng), bg(300)]), b2, np.ones(1, np.int32), ["p1", "p2"], tilt2))
    b3 = np.stack([obj["abut"], obj["p1"], obj["small"]])
    sc.append((np.concatenate([inside_pts(b, 20, rng) for b in b3] + [bg(200)]), b3, np.ones(3, np.int32), ["abut", "p1", "small"], up))
    sc.append((bg(400), np.zeros((0, 7), np.float32), np.zeros(0, np.int32), ["big", "p2", "k0", "k1"], tilt))
    p, b, l = synth.kitti_like_with_boxes(1, 4000, 12, seed=17)
    v = l[0] > 0
    sc.append((p[0], b[0][v], l[0][v], ["abut", "k0", "k1", "k2", "k3", "k4", "p2"], flat))
    return sc


def main():
    rng = np.random.default_rng(2027)
    frames, obj = db_frames(rng)
    dicts, src = ref_db(frames)
    name_of = {}
    for k, (f, j) in enumerate(src):
        for nm, b in obj.items():
            if f < 2 and np.array_equal(frames[f][1][j], b):
                name_of[nm] = k
    kitti = [k for k, (f, _) in enumerate(src) if f == 2]
    for i, k in enumerate(kitti):
        name_of["k%d" % i] = k
    scenes = paste_scenes(rng, obj)
    plane_rows = [s[4] for s in scenes]
    planes, plane_texts = ref_planes(plane_rows)
    # the reference's collision test and the whole kitti_forward with mixup on, per scene
    Bn, G = len(scenes), max(len(s[1]) for s in scenes)
    ids = np.full((Bn, S), -1, np.int32)
    pts, offs, sems, gtb, gtl = [], [0], [], np.zeros((Bn, G, 7), np.float32), np.zeros((Bn, G), np.int32)
    acc = np.zeros((Bn, S), np.int32)
    ref_boxes, ref_pts, ref_idx, ref_roff = [], [], [], [0]
    scene_u, loc, rot_u = np.zeros((Bn, 6)), np.zeros((Bn, G + S, TRIES, 2)), np.zeros((Bn, G + S, TRIES))
    env_c = base_env()
    for s, (p, b, l, names, _) in enumerate(scenes):
        g, n = len(b), len(p)
        ids[s, :len(names)] = [name_of[nm] for nm in names]
        gtb[s, :g], gtl[s, :g] = b, l
        sem = (env_c["check_inside_points"](p, np.concatenate([b[:, :3], b[:, 3:6] + 0.1, b[:, 6:]], 1)).any(1).astype(np.int64)
               if g else np.zeros(n, np.int64))
        drawn = [dicts[k] for k in ids[s] if k >= 0]
        st = n + np.concatenate([[0], np.cumsum([len(d[KEYS.KEY_SAMPLED_GT_POINTS]) for d in drawn])])
        # box_3d_collision_test alone: which drawn boxes it keeps
        q, qc, P, sl, sd = env_c["box_3d_collision_test"](
            np.stack([d[KEYS.KEY_SAMPLED_GT_LABELS_3D] for d in drawn]).astype(np.float32), b.copy(), [1] * len(drawn), l.copy(),
            [d[KEYS.KEY_SAMPLED_GT_POINTS].copy() for d in drawn], p.copy(), sem.copy(), np.ones(n, np.float32), planes[s])
        kept_boxes = q[g:]
        for i, d in enumerate(drawn):
            bx = d[KEYS.KEY_SAMPLED_GT_LABELS_3D]
            acc[s, i] = int(any(np.array_equal(kb[[0, 2, 3, 4, 5, 6]], bx[[0, 2, 3, 4, 5, 6]]) for kb in kept_boxes))
        # kitti_forward with mixup on: the sampler hands out these dicts, each point tagged with its pasted slot
        u = np.array([rng.uniform(0.05, 0.95), rng.uniform(0, 1), rng.uniform(0, 1), rng.uniform(0, 1), rng.uniform(), rng.uniform()])
        u[1:4] = [[0.3, 0.7, 0.2], [0.6, 0.3, 0.4], [0.2, 0.2, 0.9], [0.9, 0.9, 0.9], [0.4, 0.6, 0.1], [0.1, 0.1, 0.1]][s]
        lo, ro = rng.standard_normal((G + S, TRIES, 2)), rng.uniform(size=(G + S, TRIES))
        scene_u[s], loc[s], rot_u[s] = u, lo, ro
        rec = {}
        rows = int(g + acc[s].sum())
        aug, env = MGA.reference(u, lo[:rows], ro[:rows], rec)
        MGA.pull(os.path.join(REF, "utils", "voxelnet_aug.py"), {"box_3d_collision_test"}, env)
        env["maps_dict"] = KEYS
        tagged = [dict(d, **{KEYS.KEY_SAMPLED_GT_POINTS: np.concatenate(
            [d[KEYS.KEY_SAMPLED_GT_POINTS], (st[i] + np.arange(len(d[KEYS.KEY_SAMPLED_GT_POINTS])))[:, None]], 1).astype(np.float32)})
            for i, d in enumerate(drawn)]
        aug.mixup, aug.cls2idx_dict = True, {"Car": 1}
        aug.mixup_sampler_list = {0: types.SimpleNamespace(sample=lambda t=tagged: t)}
        src_pts = np.concatenate([p, np.arange(n, dtype=np.float32)[:, None]], 1)
        o_pts, _, _, o_boxes, _ = aug.kitti_forward(src_pts, sem.copy(), np.ones(n, np.float32), b.copy(), l.astype(np.int64).copy(),
                                                    planes[s], 0)
        pts.append(p)
        offs.append(offs[-1] + n)
        sems.append(sem.astype(np.int32))
        rb = np.zeros((G + S, 7), np.float32)
        rb[:len(o_boxes)] = o_boxes
        ref_boxes.append(rb)
        ref_pts.append(np.asarray(o_pts[:, :4], np.float64))
        ref_idx.append(np.asarray(o_pts[:, 4]).astype(np.int64))
        ref_roff.append(ref_roff[-1] + len(o_pts))
        print("scene %d: %d rows, drawn %s, kept %s, %d -> %d points" % (s, g, ids[s, :len(names)].tolist(), acc[s, :len(names)].tolist(),
                                                                         n, len(o_pts)))
    counts = [len(d[KEYS.KEY_SAMPLED_GT_POINTS]) for d in dicts]
    smp_rets, smp_perms = ref_sampler(37, 15, 10, rng)
    fr_off = np.concatenate([[0], np.cumsum([len(f[0]) for f in frames])]).astype(np.int32)
    Gf = max(len(f[1]) for f in frames)
    fb, fl = np.zeros((len(frames), Gf, 7), np.float32), np.zeros((len(frames), Gf), np.int32)
    for f, (_, b, l) in enumerate(frames):
        fb[f, :len(b)], fl[f, :len(l)] = b, l
    T = offs[-1] + sum(counts[k] for k in ids.reshape(-1) if k >= 0)
    np.savez_compressed(
        os.path.join(HERE, "mixup.npz"),
        db_frame_points=np.concatenate([f[0] for f in frames]).astype(np.float32), db_frame_offsets=fr_off, db_frame_boxes=fb,
        db_frame_labels=fl, ref_db_points=np.concatenate([d[KEYS.KEY_SAMPLED_GT_POINTS] for d in dicts]).astype(np.float32),
        ref_db_offsets=np.concatenate([[0], np.cumsum(counts)]).astype(np.int64),
        ref_db_boxes=np.stack([d[KEYS.KEY_SAMPLED_GT_LABELS_3D] for d in dicts]).astype(np.float32), ref_db_src=src,
        points=np.concatenate(pts), offsets=np.asarray(offs, np.int32), sem_labels=np.concatenate(sems), gt_boxes=gtb, gt_labels=gtl,
        ids=ids, plane_rows=np.asarray(plane_rows, np.float64), plane_texts=np.asarray(plane_texts), ref_planes=planes,
        ref_accepted=acc, scene_u=scene_u, loc_noise=loc, rot_u=rot_u,
        keys=rng.integers(0, 2 ** 32, T + sum(counts) * 2).astype(np.uint32).view(np.int32),
        refill=rng.integers(0, 2 ** 32, (Bn, M)).astype(np.uint32).view(np.int32),
        ref_points=np.concatenate(ref_pts), ref_index=np.concatenate(ref_idx), ref_offsets=np.asarray(ref_roff, np.int32),
        ref_boxes=np.stack(ref_boxes), sampler_count=37, sampler_num=15, sampler_rets=np.concatenate(smp_rets),
        sampler_ret_sizes=np.array([len(r) for r in smp_rets]), sampler_perms=np.stack(smp_perms))
    print("wrote mixup.npz: %d database objects, %d points" % (len(dicts), sum(counts)))


if __name__ == "__main__":
    main()
