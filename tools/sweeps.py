"""BASELINE.json configs[2] and configs[3] (SURVEY.md 8d "Config 3" / "Config 4"), timed with CUDA events next to the
reference's own kernels (oracle/_ref) on the same GPU.  Writes one JSON file.

  python tools/sweeps.py fps [out.json]   D-FPS (xyz) and F-FPS (xyz + 64 features ~N(0,1)) at N in {4096, 16384, 65536},
                                          M = N/4, B = 8: ms, ns per round, effective-stream GB/s, reference kernel ms.
                                          F-FPS routes: 'direct' (matrix-free, matrix arithmetic; n <= 4096), 'matrix'
                                          (calc_square_dist + with_distance; where B*N^2*4 fits), 'fused' (generic-c kernel
                                          semantics, any N -- the only route the reference itself has for N >= 16384).
  python tools/sweeps.py bq [out.json]    N=16384 -> M=4096 D-FPS queries, r in {0.2,0.4,0.8} x K in {16,32,64}, C=64,
                                          MLP [64,64,128], B=8: ball query ms, fused gather+MLP+max ms, bf16 TFLOP/s issued,
                                          on synthetic-KITTI clouds and on U(0,1)^3 cubes (K saturates).
"""
import importlib
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("3dssd_b200")
P = pkg.params
synth = importlib.import_module("3dssd_b200.synth")
from oracle import ref_ops  # noqa: E402


def timeit(fn, warmup=2, iters=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def fps_sweep():
    dev = torch.device("cuda:0")
    B, rows = 8, []
    have_ref = ref_ops.available()
    rng = np.random.default_rng(0)
    for n in (4096, 16384, 65536):
        m = n // 4
        reps = max(1, n // 16384)
        xyz_np = np.concatenate([synth.kitti_like(B, min(n, 16384), seed=300 + i)[..., :3] for i in range(reps)], 1)[:, :n]
        xyz = torch.from_numpy(np.ascontiguousarray(xyz_np)).to(dev)
        feat = torch.from_numpy(rng.standard_normal((B, n, 64)).astype(np.float32)).to(dev)
        both = torch.cat([xyz, feat], -1).contiguous()
        r = {"N": n, "M": m, "B": B}
        ms = timeit(lambda: pkg.farthest_point_sample(m, xyz))
        r["dfps_ms"] = ms
        r["dfps_ns_per_round"] = ms * 1e6 / (m - 1)
        r["dfps_effective_stream_gbs"] = B * (m - 1) * n * 16 / (ms * 1e-3) / 1e9
        r["dfps_compulsory_bytes"] = B * (n * 12 + m * 4)
        if have_ref:
            r["ref_dfps_ms"] = timeit(lambda: ref_ops.farthest_point_sample(m, xyz, sync=False), 1, 2)
            r["dfps_speedup_vs_ref"] = r["ref_dfps_ms"] / ms
            r["dfps_matches_ref"] = bool(torch.equal(pkg.farthest_point_sample(m, xyz), ref_ops.farthest_point_sample(m, xyz)))
        if pkg.tf_ops.ffps_supported(n, 67):
            ms = timeit(lambda: pkg.tf_ops.farthest_point_sample_features(m, xyz, feat))
            r["ffps_direct_ms"] = ms
            r["ffps_direct_ns_per_round"] = ms * 1e6 / (m - 1)
        if B * n * n * 4 <= 8 << 30:
            dist = pkg.calc_square_dist(both)
            r["ffps_matrix_sqdist_ms"] = timeit(lambda: pkg.calc_square_dist(both))
            r["ffps_matrix_sample_ms"] = timeit(lambda: pkg.farthest_point_sample_with_distance(m, dist))
            if have_ref:
                r["ref_ffps_with_distance_ms"] = timeit(lambda: ref_ops.farthest_point_sample_with_distance(m, dist, sync=False), 1, 2)
            if "ffps_direct_ms" in r:
                r["ffps_direct_equals_matrix"] = bool(torch.equal(pkg.tf_ops.farthest_point_sample_features(m, xyz, feat),
                                                                 pkg.farthest_point_sample_with_distance(m, dist)))
            del dist
        try:
            ms = timeit(lambda: pkg.farthest_point_sample(m, both), 1, 3)
            r["ffps_fused_ms"] = ms
            r["ffps_fused_ns_per_round"] = ms * 1e6 / (m - 1)
            r["ffps_fused_effective_stream_gbs"] = B * (m - 1) * n * (67 * 4 + 4) / (ms * 1e-3) / 1e9
            if have_ref and n <= 16384:
                r["ref_ffps_generic_c_ms"] = timeit(lambda: ref_ops.farthest_point_sample(m, both, sync=False), 1, 1)
        except Exception as e:  # noqa: BLE001
            r["ffps_fused_ms"] = "ERR " + str(e)
        rows.append(r)
        print(json.dumps(r), flush=True)
    return {"config": "configs[2]: F-FPS vs D-FPS sweep, B=8, M=N/4", "gpu": torch.cuda.get_device_name(0), "rows": rows}


def bq_sweep():
    dev = torch.device("cuda:0")
    B, n, m, c = 8, 16384, 4096, 64
    mlp = [64, 64, 128]
    rng = np.random.default_rng(0)
    have_ref = ref_ops.available()
    out = []
    for dname, gen in (("synthetic-kitti", lambda: synth.kitti_like(B, n, seed=1000)[..., :3].copy()),
                       ("uniform-cube", lambda: synth.uniform_cube(B, n, seed=5))):
        xyz = torch.from_numpy(np.ascontiguousarray(gen())).to(dev)
        feat = torch.from_numpy(rng.standard_normal((B, n, c)).astype(np.float32)).to(dev)
        new_xyz = pkg.gather_point(xyz, pkg.farthest_point_sample(m, xyz))
        prm, scopes, cin = {}, [], c + 3
        for j, co in enumerate(mlp):
            P._conv_init(rng, prm, "s/conv0_%d" % j, cin, co, True)
            scopes.append("s/conv0_%d" % j)
            cin = co
        pp = P.prepare(prm, dev)
        stack = pp.fused_stack(scopes, True, c + 3, limit=0)
        zconv, wxs, n1s = pp.hoisted(["s/conv0_0"], True, c)
        hstack = pp.fused_stack(scopes[1:], True, n1s[0], limit=0)
        p_hi, p_lo = pkg.tf_ops.split_rows(feat)
        z, _ = pkg.tf_ops.linear_tc(p_hi, p_lo, zconv, relu=False, want_f32=True, want_split=False)
        for radius in (0.2, 0.4, 0.8):
            for k in (16, 32, 64):
                r = {"data": dname, "r": radius, "K": k}
                r["ball_query_ms"] = timeit(lambda: pkg.query_ball_point(radius, k, xyz, new_xyz))
                idx, cnt = pkg.query_ball_point(radius, k, xyz, new_xyz)
                r["mean_cnt"] = float(cnt.float().mean())
                if have_ref:
                    r["ref_ball_query_ms"] = timeit(lambda: ref_ops.query_ball_point(radius, k, xyz, new_xyz, sync=False), 1, 2)
                rows = B * m * k
                ms = timeit(lambda: pkg.tf_ops.sa_mlp_fused(xyz, feat, new_xyz, idx, cnt, stack))
                fl = 3 * 2.0 * rows * (80 * 64 + 64 * 64 + 64 * 128)
                r["fused_literal_ms"] = ms
                r["fused_literal_tflops_bf16_issued"] = fl / (ms * 1e-3) / 1e12
                ms = timeit(lambda: pkg.tf_ops.sa_mlp_fused_hoisted(xyz, z, 0, wxs[0], new_xyz, idx, cnt, hstack))
                fl = 3 * 2.0 * rows * (64 * 64 + 64 * 128)
                r["fused_hoisted_ms"] = ms
                r["fused_hoisted_tflops_bf16_issued"] = fl / (ms * 1e-3) / 1e12
                r["algorithmic_gflop"] = 2.0 * rows * (67 * 64 + 64 * 64 + 64 * 128) / 1e9
                out.append(r)
                print(json.dumps(r), flush=True)
    return {"config": "configs[3]: ball-query r x K sweep fused with group + MLP [64,64,128], N=16384 -> M=4096, C=64, B=8",
            "gpu": torch.cuda.get_device_name(0), "rows": out}


if __name__ == "__main__":
    which = sys.argv[1]
    res = fps_sweep() if which == "fps" else bq_sweep()
    path = sys.argv[2] if len(sys.argv) > 2 else os.path.join(ROOT, "gpurun_out", "r02_sweep_%s.json" % which)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
