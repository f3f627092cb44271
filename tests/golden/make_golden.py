"""Generates tests/golden/*.npz by running the REFERENCE's own CUDA kernels (oracle/_ref/libref_ops.so,
compiled unmodified from the reference sources by `make -C oracle ref`) on seeded inputs.

Must run on a GPU:   python tests/golden/make_golden.py <dir>
then copy <dir>/*.npz into tests/golden/ and commit.  The fixtures pin the CPU oracle
(tests/test_oracle_cpu.py::test_oracle_against_reference_golden_vectors) -- the reference itself ships no
golden vectors for this path (SURVEY.md section 8c).
"""
import importlib
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref_ops  # noqa: E402

synth = importlib.import_module("3dssd_b200.synth")


def t(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def main(out_dir):
    os.makedirs(out_dir, exist_ok=True)
    rng = np.random.default_rng(20260923)

    def save(name, **kw):
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), **kw)
        print("wrote", name)

    # ---- FPS: random, KITTI-like with duplicate padding, lattice (ties), n < 1024, generic c
    cases = {
        "fps_kitti_2x4096_m512": (synth.kitti_like(2, 4096, seed=7)[..., :3], 512),
        "fps_lattice_2x3000_m256": (synth.lattice(2, 3000, seed=3), 256),
        "fps_small_3x300_m64": (rng.uniform(-1, 1, (3, 300, 3)).astype(np.float32), 64),
        "fps_dups_1x1500_m200": (np.repeat(rng.uniform(-1, 1, (1, 500, 3)).astype(np.float32), 3, axis=1), 200),
        "fps_feat67_2x512_m128": (rng.standard_normal((2, 512, 67)).astype(np.float32), 128),
    }
    for name, (inp, m) in cases.items():
        out = ref_ops.farthest_point_sample(m, t(inp)).cpu().numpy()
        save(name, op="farthest_point_sample", npoint=m, inp=inp, out=out)

    # ---- FPS with distance matrix (values are arbitrary floats: use a random symmetric matrix and a real one)
    f = rng.standard_normal((2, 384, 9)).astype(np.float32)
    d = ((f[:, :, None, :] - f[:, None, :, :]) ** 2).sum(-1).astype(np.float32)
    out = ref_ops.farthest_point_sample_with_distance(96, t(d)).cpu().numpy()
    save("fpsdist_2x384_m96", op="farthest_point_sample_with_distance", npoint=96, dist=d, out=out)
    dq = np.round(d * 2) / 2     # quantised: many exact ties
    out = ref_ops.farthest_point_sample_with_distance(96, t(dq.astype(np.float32))).cpu().numpy()
    save("fpsdist_ties_2x384_m96", op="farthest_point_sample_with_distance", npoint=96, dist=dq.astype(np.float32), out=out)

    # ---- ball queries
    pts = synth.kitti_like(2, 4096, seed=11)[..., :3]
    q = np.ascontiguousarray(pts[:, ::8][:, :384])
    for r, k in ((0.4, 16), (1.6, 32)):
        idx, cnt = ref_ops.query_ball_point(r, k, t(pts), t(q))
        save("bq_kitti_r%g_k%d" % (r, k), op="query_ball_point", radius=r, nsample=k, xyz1=pts, xyz2=q,
             idx=idx.cpu().numpy(), cnt=cnt.cpu().numpy())
    for lo, hi, k in ((0.0, 0.4, 32), (0.4, 0.8, 32), (0.8, 1.6, 64)):
        idx, cnt = ref_ops.query_ball_point_dilated(lo, hi, k, t(pts), t(q))
        save("bqd_kitti_%g_%g_k%d" % (lo, hi, k), op="query_ball_point_dilated", min_radius=lo, max_radius=hi,
             nsample=k, xyz1=pts, xyz2=q, idx=idx.cpu().numpy(), cnt=cnt.cpu().numpy())
    lat = synth.lattice(1, 1500, seed=5)           # distances exactly on the radius boundaries
    ql = np.ascontiguousarray(lat[:, :200])
    idx, cnt = ref_ops.query_ball_point(0.5, 24, t(lat), t(ql))
    save("bq_lattice_r0.5_k24", op="query_ball_point", radius=0.5, nsample=24, xyz1=lat, xyz2=ql,
         idx=idx.cpu().numpy(), cnt=cnt.cpu().numpy())
    idx, cnt = ref_ops.query_ball_point_dilated(0.25, 0.5, 24, t(lat), t(ql))
    save("bqd_lattice_0.25_0.5_k24", op="query_ball_point_dilated", min_radius=0.25, max_radius=0.5, nsample=24,
         xyz1=lat, xyz2=ql, idx=idx.cpu().numpy(), cnt=cnt.cpu().numpy())
    far = (q + 1000.0).astype(np.float32)          # empty balls
    idx, cnt = ref_ops.query_ball_point(0.4, 8, t(pts), t(far))
    save("bq_empty_r0.4_k8", op="query_ball_point", radius=0.4, nsample=8, xyz1=pts, xyz2=far,
         idx=idx.cpu().numpy(), cnt=cnt.cpu().numpy())

    # ---- gather / group
    feats = rng.standard_normal((2, 700, 13)).astype(np.float32)
    gi = rng.integers(0, 700, (2, 90)).astype(np.int32)
    save("gather_2x700x13", op="gather_point", inp=feats, idx=gi, out=ref_ops.gather_point(t(feats), t(gi)).cpu().numpy())
    gidx = rng.integers(-1, 700, (2, 40, 6)).astype(np.int32)
    save("group_2x700x13", op="group_point", points=feats, idx=gidx,
         out=ref_ops.group_point(t(feats), t(gidx)).cpu().numpy())

    # ---- three_nn / three_interpolate
    u = rng.uniform(0, 1, (2, 600, 3)).astype(np.float32)
    kn = rng.uniform(0, 1, (2, 150, 3)).astype(np.float32)
    dist, idx = ref_ops.three_nn(t(u), t(kn))
    save("three_nn_2x600_150", op="three_nn", xyz1=u, xyz2=kn, dist=dist.cpu().numpy(), idx=idx.cpu().numpy())
    ul = synth.lattice(1, 400, seed=8); kl = synth.lattice(1, 120, seed=9)
    dist, idx2 = ref_ops.three_nn(t(ul), t(kl))
    save("three_nn_lattice", op="three_nn", xyz1=ul, xyz2=kl, dist=dist.cpu().numpy(), idx=idx2.cpu().numpy())
    pf = rng.standard_normal((2, 150, 20)).astype(np.float32)
    w = rng.uniform(0, 1, (2, 600, 3)).astype(np.float32)
    out = ref_ops.three_interpolate(t(pf), idx, t(w)).cpu().numpy()
    save("three_interpolate_2x600", op="three_interpolate", points=pf, idx=idx.cpu().numpy(), weight=w, out=out)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "golden_out"))
