"""The skip rule of the 4-CTA F-FPS with bucket pruning (ffps_bucket_kernel, csrc/fps.cu) and its launch plan, without a
GPU.  tests/ffps_prune_model.c runs the F-FPS with the kernel's fp32 arithmetic and bucket bounds and counts, every
round, the points of skipped buckets whose value would have been below their running distance: there must be none, on
the benchmark's layer-2 operands and on scenes where the bound is tight, and the sampled indices must be the oracle's.
With the rounding margin dropped the same model must find such points."""
import ctypes
import importlib
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def model(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("ffps_model") / "libffps_prune_model.so")
    subprocess.check_call(["cc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC", "-o", so,
                           os.path.join(HERE, "ffps_prune_model.c"), "-lm"])
    lib = ctypes.CDLL(so)
    lib.ffps_prune_model.restype = ctypes.c_longlong
    lib.ffps_prune_model.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                     ctypes.c_void_p, ctypes.c_void_p]

    def run(x, m, with_margin=True):
        x = np.ascontiguousarray(x, np.float32)
        idx = np.zeros(m, np.int32)
        touched = ctypes.c_longlong(0)
        bad = lib.ffps_prune_model(x.shape[0], x.shape[1], m, x.ctypes.data, int(with_margin), idx.ctypes.data,
                                   ctypes.byref(touched))
        assert bad >= 0
        return bad, idx, touched.value / ((m - 1) * ((x.shape[0] + 31) // 32))
    return run


def _scene(kind, n, seed):
    rng = np.random.default_rng(seed)
    xyz = np.stack([rng.uniform(-40, 40, n), rng.uniform(-3, 1, n), 70 * rng.uniform(0, 1, n) ** 2], -1)
    feat = np.maximum(rng.normal(0.0, 0.5, (n, 64)), 0.0)
    if kind == "dups":
        src = rng.integers(0, n, n // 3)
        xyz[n - n // 3:], feat[n - n // 3:] = xyz[src], feat[src]
    elif kind == "quantised":
        feat = np.round(feat * 2) / 2
    elif kind == "zero":
        feat[:] = 0.0
    elif kind == "offset":
        feat = feat + 1e4
    elif kind == "ties":
        xyz = rng.integers(0, 8, (n, 3)).astype(np.float64)
        feat = rng.integers(0, 2, (n, 64)).astype(np.float64)
    return np.concatenate([xyz, feat], 1).astype(np.float32)


@pytest.mark.parametrize("kind", ["plain", "dups", "quantised", "zero", "offset", "ties"])
def test_skip_rule_never_changes_a_distance(model, oracle_ops, kind):
    x = _scene(kind, 4096, 5)
    bad, idx, _ = model(x, 512)
    assert bad == 0
    assert np.array_equal(idx, oracle_ops.farthest_point_sample_features(512, x[None, :, :3], x[None, :, 3:])[0])


def test_skip_rule_on_bench_operands(model, oracle_ops):
    """Layer-1 output of the benchmark's first two scenes (the layer-2 F-FPS operands): exact, and a round touches
    about a tenth of the buckets (tools/ffps_prune_sim.py: mean 0.10 over the eight scenes)."""
    pkg = importlib.import_module("3dssd_b200")
    synth = importlib.import_module("3dssd_b200.synth")
    from oracle import layers as olayers
    arch = pkg.config.ARCH_3DSSD
    xyz_l, feat_l, _ = olayers.backbone_forward(arch[:1], synth.kitti_like(2, 16384, seed=1000),
                                                pkg.params.init_params(arch, 1, seed=0))
    for s in range(2):
        x = np.concatenate([xyz_l[1][s], feat_l[1][s]], 1)
        bad, idx, phi = model(x, 512)
        assert bad == 0
        assert phi < 0.2, phi
        assert np.array_equal(idx, oracle_ops.farthest_point_sample_features(512, xyz_l[1][s:s + 1], feat_l[1][s:s + 1])[0])


def test_skip_rule_needs_its_margin(model):
    """Features offset by 1e4: the values' rounding error (~ 8e-6 * |x|^2, hundreds) dwarfs the true distances, so
    without E the bound skips points whose computed value is below their running distance."""
    bad, _, _ = model(_scene("offset", 4096, 5), 512, with_margin=False)
    assert bad > 0


PLAN_CPP = r"""
#include <cstdio>
#include "%s"
using namespace ssd3d;
int main() {
    const int ns[] = {1, 2048, 2049, 3000, 4096, 4097}, cs[] = {2, 3, 67, 68, 69, 132}, cls[] = {0, -1, -2, -4, -8, -16};
    for (int n : ns) for (int c : cs) for (int cl : cls) for (int part = 0; part < 2; part++) {
        const FpsPlan a = plan_ffps_cl(n, c, cl, part != 0), b = plan_ffps(n, c, part != 0);
        std::printf("%%d %%d %%d %%d %%d %%d %%d %%zu %%ld %%d %%d %%d %%d %%zu %%ld %%d\n", n, c, cl, part, (int)a.kind, a.cl, a.p,
                    a.smem, a.temp, (int)a.rounds, (int)b.kind, b.cl, b.p, b.smem, b.temp, (int)b.rounds);
    }
}
"""


def test_plan_ffps_cl(tmp_path):
    """The capped plan picks the bucket kernel (4 CTAs, 4 slots per thread) exactly for full-range calls with
    2048 < n <= 4096, 3 <= c <= 68 and a cap below 8 CTAs; everything else is plan_ffps's plan."""
    src = tmp_path / "plan.cpp"
    src.write_text(PLAN_CPP % os.path.join(os.path.dirname(HERE), "3dssd_b200", "csrc", "fps_plan.h"))
    exe = str(tmp_path / "plan")
    subprocess.check_call(["c++", "-std=c++17", "-O1", "-Wall", "-Werror", "-o", exe, str(src)])
    lines = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split("\n")[:-1]
    assert len(lines) == 6 * 6 * 6 * 2
    picked = 0
    for line in lines:
        n, c, cl, part, *v = map(int, line.split())
        a, b = v[:6], v[6:]
        bucket = part == 0 and cl in (-1, -2, -4) and 2048 < n <= 4096 and 3 <= c <= 68
        if bucket:
            picked += 1
            assert a[0] == b[0] and a[1:4] == [4, 4, 2 * 256 * 68 * 4 + 4096 * 8 + 8 * 4 * 72 * 4 + 2 * 8 * 72 * 4 + 2 * 4 * 288]
            assert a[4] == 0 and a[5] == 0
        else:
            assert a == b, line
    assert picked == 3 * 3 * 3            # n in (2049, 3000, 4096), c in (3, 67, 68), cap in (-1, -2, -4)
