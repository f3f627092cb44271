"""ctypes front-end of oracle/_ref/libref_ops.so: the REFERENCE's own CUDA kernels
(lib/utils/tf_ops/{sampling/tf_sampling_g.cu, grouping/tf_grouping_g.cu,
interpolation/tf_interpolate_g.cu}) compiled unmodified for sm_90 by oracle/Makefile (`make ref`).

TEST INFRASTRUCTURE ONLY.  Used (a) as the bit-exactness oracle of the `-m gpu` tests, (b) to
produce tests/golden/*.npz (make_golden.py), and (c) as the GPU leg of bench.py --impl reference.

The launchers use C++ linkage, so they are bound by their mangled names; they launch on the legacy
default stream (`<<<g,b>>>` without a stream argument, e.g. tf_sampling_g.cu:393), hence the
explicit synchronisation around every call.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "_ref", "libref_ops.so")
_lib = None


def available():
    return os.path.exists(LIB_PATH)


def lib():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(LIB_PATH)
    return _lib


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _check(t, dtype):
    assert t.is_cuda and t.is_contiguous() and t.dtype == dtype, (t.device, t.dtype, t.is_contiguous())


def _call(name, *args, sync=True):
    if sync:
        torch.cuda.synchronize()
    getattr(lib(), name)(*args)
    if sync:
        torch.cuda.synchronize()


def farthest_point_sample(npoint, inp, sync=True):
    _check(inp, torch.float32)
    b, n, c = inp.shape
    out = torch.empty((b, npoint), dtype=torch.int32, device=inp.device)
    temp = torch.empty((b, n), dtype=torch.float32, device=inp.device)
    _call("_Z29farthestpointsamplingLauncheriiiiPKfPfPi", b, n, c, int(npoint), _p(inp), _p(temp), _p(out), sync=sync)
    return out


def farthest_point_sample_with_distance(npoint, dist, sync=True):
    _check(dist, torch.float32)
    b, n, _ = dist.shape
    out = torch.empty((b, npoint), dtype=torch.int32, device=dist.device)
    temp = torch.empty((b, n), dtype=torch.float32, device=dist.device)
    _call("_Z37farthestpointsamplingwithdistLauncheriiiPKfPfPi", b, n, int(npoint), _p(dist), _p(temp), _p(out), sync=sync)
    return out


def gather_point(inp, idx, sync=True):
    _check(inp, torch.float32); _check(idx, torch.int32)
    b, n, c = inp.shape
    m = idx.shape[1]
    out = torch.empty((b, m, c), dtype=torch.float32, device=inp.device)
    _call("_Z19gatherpointLauncheriiiiPKfPKiPf", b, n, m, c, _p(inp), _p(idx), _p(out), sync=sync)
    return out


def query_ball_point(radius, nsample, xyz1, xyz2, sync=True):
    _check(xyz1, torch.float32); _check(xyz2, torch.float32)
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    # zero-initialised: the reference leaves rows with cnt==0 unwritten (tf_grouping.cpp:291-304)
    idx = torch.zeros((b, m, nsample), dtype=torch.int32, device=xyz1.device)
    cnt = torch.zeros((b, m), dtype=torch.int32, device=xyz1.device)
    _call("_Z22queryBallPointLauncheriiifiPKfS0_PiS1_", b, n, m, ctypes.c_float(radius), int(nsample),
          _p(xyz1), _p(xyz2), _p(idx), _p(cnt), sync=sync)
    return idx, cnt


def query_ball_point_dilated(min_radius, max_radius, nsample, xyz1, xyz2, sync=True):
    _check(xyz1, torch.float32); _check(xyz2, torch.float32)
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    idx = torch.zeros((b, m, nsample), dtype=torch.int32, device=xyz1.device)
    cnt = torch.zeros((b, m), dtype=torch.int32, device=xyz1.device)
    _call("_Z29queryBallPointDilatedLauncheriiiffiPKfS0_PiS1_", b, n, m, ctypes.c_float(min_radius),
          ctypes.c_float(max_radius), int(nsample), _p(xyz1), _p(xyz2), _p(idx), _p(cnt), sync=sync)
    return idx, cnt


def group_point(points, idx, sync=True):
    _check(points, torch.float32); _check(idx, torch.int32)
    b, n, c = points.shape
    _, m, ns = idx.shape
    out = torch.empty((b, m, ns, c), dtype=torch.float32, device=points.device)
    _call("_Z18groupPointLauncheriiiiiPKfPKiPf", b, n, c, m, ns, _p(points), _p(idx), _p(out), sync=sync)
    return out


def three_nn(xyz1, xyz2, sync=True):
    _check(xyz1, torch.float32); _check(xyz2, torch.float32)
    b, n, _ = xyz1.shape
    m = xyz2.shape[1]
    dist = torch.empty((b, n, 3), dtype=torch.float32, device=xyz1.device)
    idx = torch.empty((b, n, 3), dtype=torch.int32, device=xyz1.device)
    _call("_Z15ThreeNNLauncheriiiPKfS0_PfPi", b, n, m, _p(xyz1), _p(xyz2), _p(dist), _p(idx), sync=sync)
    return dist, idx


def three_interpolate(points, idx, weight, sync=True):
    _check(points, torch.float32); _check(idx, torch.int32); _check(weight, torch.float32)
    b, m, c = points.shape
    n = idx.shape[1]
    out = torch.empty((b, n, c), dtype=torch.float32, device=points.device)
    _call("_Z24ThreeInterpolateLauncheriiiiPKfPKiS0_Pf", b, m, c, n, _p(points), _p(idx), _p(weight), _p(out), sync=sync)
    return out
