"""Builds tests/golden/realscan_16384.npz and tests/golden/realscan_full.npz from the reference's sample KITTI scan
(SURVEY.md section 8d, distribution B).

mayavi/kitti_sample_scan.txt of the reference holds 123 398 velodyne points (x forward, y left, z up).

realscan_16384.npz: they are mapped to the rect camera frame of configs/kitti/3dssd/3dssd.yaml:3 (x_r = -y_v, y_r = -z_v,
z_r = x_v), cropped to the detection range x in (-40, 40), y in (-5, 3), z in (0, 70) and |x| < z (about 90 degrees of
field of view), and a seeded choice of 16 384 of them is stored with a U(0,1) intensity: one real LiDAR scene in the
loader's [16384, 4] layout.

realscan_full.npz: every velodyne point, in the scan's own order and frame, from which tests/test_realscan_cpu.py builds
its scenes.  The scan is printed in millimetres, so it is stored as integer millimetres, differenced along the scan order
(consecutive returns are close) and column by column -- `mm_delta` [3, 123398] int32, a third of the size of the float
array once compressed -- plus the flat [n, 3] positions of the text's "-0.000" entries (`neg_zero`) and a seeded uniform
intensity code `intensity_code` [123398] uint8.  decode_full() restores the float32 points bit for bit (float64
millimetres / 1000, rounded once: what parsing the text to float32 gives; -0 where the text says so) with intensity
(code + 0.5) / 256.

A file whose arrays already equal the computed ones is left as it is, so rerunning the script changes no bytes.
Needs a reference checkout (path in $REFERENCE):   REFERENCE=<checkout> python tests/golden/make_realscan.py
"""
import os

import numpy as np

SRC = os.path.join(os.environ.get("REFERENCE", "."), "mayavi", "kitti_sample_scan.txt")
HERE = os.path.dirname(os.path.abspath(__file__))


def encode_full(v, code):
    """velodyne xyz [n, 3] float32 as parsed from the text, intensity codes [n] uint8 -> the arrays of realscan_full.npz"""
    mm = np.round(v.astype(np.float64) * 1000.0).astype(np.int64)
    delta = np.diff(mm, axis=0, prepend=0).T
    assert np.abs(delta).max() < 2 ** 31
    neg_zero = np.flatnonzero((v == 0) & np.signbit(v)).astype(np.int32)
    return dict(mm_delta=np.ascontiguousarray(delta, dtype=np.int32), neg_zero=neg_zero,
                intensity_code=np.asarray(code, np.uint8))


def decode_full(mm_delta, neg_zero, intensity_code):
    """the arrays of realscan_full.npz -> [n, 4] float32 (velodyne xyz, intensity)"""
    xyz = np.ascontiguousarray(np.cumsum(mm_delta.astype(np.int64), axis=1).T / 1000.0, dtype=np.float32)
    xyz.reshape(-1)[neg_zero] = np.float32(-0.0)
    inten = ((intensity_code.astype(np.float32) + np.float32(0.5)) / np.float32(256)).astype(np.float32)
    return np.ascontiguousarray(np.concatenate([xyz, inten[:, None]], axis=1), dtype=np.float32)


def _save(name, **arrays):
    path = os.path.join(HERE, name)
    if os.path.exists(path):
        old = np.load(path)
        if sorted(old.files) == sorted(arrays) and all(np.array_equal(old[k], np.asarray(v)) for k, v in arrays.items()):
            print(name, "unchanged")
            return
    np.savez_compressed(path, **arrays)
    print("wrote", name)


def main():
    v = np.loadtxt(SRC, dtype=np.float32)
    r = np.stack([-v[:, 1], -v[:, 2], v[:, 0]], axis=1)
    keep = (np.abs(r[:, 0]) < 40) & (r[:, 1] > -5) & (r[:, 1] < 3) & (r[:, 2] > 0) & (r[:, 2] < 70) & (np.abs(r[:, 0]) < r[:, 2])
    r = r[keep]
    rng = np.random.default_rng(1000)
    sel = rng.choice(r.shape[0], 16384, replace=False)
    pts = np.concatenate([r[sel], rng.uniform(0, 1, (16384, 1)).astype(np.float32)], axis=1).astype(np.float32)
    _save("realscan_16384.npz", points=pts, source="mayavi/kitti_sample_scan.txt", kept=int(keep.sum()))
    print("kept", int(keep.sum()), "of", v.shape[0], "->", pts.shape, pts.min(0), pts.max(0))

    arrays = encode_full(v, np.random.default_rng(1001).integers(0, 256, v.shape[0], dtype=np.uint8))
    full = decode_full(**arrays)
    assert np.array_equal(full[:, :3].view(np.int32), v.view(np.int32)), "the millimetre code must restore the scan exactly"
    _save("realscan_full.npz", source="mayavi/kitti_sample_scan.txt", frame="velodyne", **arrays)
    print("full scan", full.shape)


if __name__ == "__main__":
    main()
