"""Recorded outputs of the reference's own CUDA kernels (oracle/ref_ops.py), so that the GPU tests that compare with
them run where the reference sources are not available.

Every call is keyed by the function name, its scalar arguments and the bytes of its input tensors.  `Recorder` runs
the live kernels (oracle/_ref/libref_ops.so) and keeps their outputs; `save()` writes them to an .npz file
(tests/golden/ref_kernels.npz).  `Replay` answers the same calls from that file and fails loudly on a call it has no
record of -- the inputs of the tests are seeded, so a miss means the inputs changed and the file must be recorded
again:

    SSD3D_RECORD_REF=/path/ref_kernels.npz python -m pytest -m gpu tests     (on a GPU, with oracle/_ref built)
"""
import hashlib

import numpy as np
import torch

FUNCS = ("farthest_point_sample", "farthest_point_sample_with_distance", "query_ball_point", "query_ball_point_dilated",
         "three_nn", "three_interpolate")


def _key(name, args):
    h = hashlib.sha1(name.encode())
    for a in args:
        if isinstance(a, torch.Tensor):
            h.update(str((tuple(a.shape), str(a.dtype))).encode())
            h.update(a.detach().contiguous().cpu().numpy().tobytes())
        else:
            h.update(repr(float(a)).encode())
    return "%s_%s" % (name, h.hexdigest()[:20])


def _as_tuple(out):
    return out if isinstance(out, tuple) else (out,)


class Recorder:
    def __init__(self, live):
        self.live, self.records = live, {}
        for name in FUNCS:
            setattr(self, name, self._wrap(name))

    def _wrap(self, name):
        def call(*args):
            out = getattr(self.live, name)(*args)
            for i, t in enumerate(_as_tuple(out)):
                self.records["%s_%d" % (_key(name, args), i)] = t.cpu().numpy()
            return out
        return call

    def save(self, path):
        small = {}
        for k, v in self.records.items():      # int32 indices / counts below 2^15 are stored as int16 (file size)
            small[k] = v.astype(np.int16) if v.dtype == np.int32 and v.size and 0 <= v.min() and v.max() < 32768 else v
        np.savez_compressed(path, **small)


class Replay:
    def __init__(self, path):
        self.data = np.load(path)
        for name in FUNCS:
            setattr(self, name, self._wrap(name))

    def _wrap(self, name):
        def call(*args):
            key = _key(name, args)
            if key + "_0" not in self.data:
                raise KeyError("no recorded reference output for %s(...) with these inputs (%s): record %s again"
                               % (name, key, "tests/golden/ref_kernels.npz"))
            dev = next(a.device for a in args if isinstance(a, torch.Tensor))
            outs, i = [], 0
            while "%s_%d" % (key, i) in self.data:
                a = self.data["%s_%d" % (key, i)]
                outs.append(torch.from_numpy(a.astype(np.int32) if a.dtype == np.int16 else a).to(dev))
                i += 1
            return outs[0] if len(outs) == 1 else tuple(outs)
        return call
