"""Generates tests/golden/kitti_io.npz by executing the REFERENCE's own numpy helpers on seeded boxes.

The reference modules import tensorflow at the top, which is not installed here, so the three pure-numpy functions
are pulled out of their source files with `ast` and executed as they are (nothing is copied into this repo):
  lib/utils/box_3d_utils.py   get_box3d_corners_helper_np
  lib/utils/kitti_util.py     project_to_image
  lib/utils/anchors_util.py   project_to_image_space_corners
Needs a reference checkout (path in $REFERENCE):   REFERENCE=<checkout> python tests/golden/make_golden_io.py
"""
import ast
import os
import types

import numpy as np

REF = os.path.join(os.environ.get("REFERENCE", "."), "lib", "utils")
HERE = os.path.dirname(os.path.abspath(__file__))


def pull(path, names, env):
    src = open(path).read()
    tree = ast.parse(src)
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name in names:
            exec(compile(ast.Module([node], []), path, "exec"), env)


def main():
    env = {"np": np}
    pull(os.path.join(REF, "kitti_util.py"), {"project_to_image"}, env)
    env["kitti_util"] = types.SimpleNamespace(project_to_image=env["project_to_image"])
    pull(os.path.join(REF, "box_3d_utils.py"), {"get_box3d_corners_helper_np"}, env)
    pull(os.path.join(REF, "anchors_util.py"), {"project_to_image_space_corners"}, env)

    rng = np.random.default_rng(77)
    n = 64
    boxes = np.empty((n, 7), np.float32)
    boxes[:, 0] = rng.uniform(-30, 30, n)
    boxes[:, 1] = rng.uniform(0.8, 2.2, n)
    boxes[:, 2] = rng.uniform(3, 70, n)
    boxes[:, 3] = rng.uniform(3.0, 5.0, n)
    boxes[:, 4] = rng.uniform(1.3, 1.9, n)
    boxes[:, 5] = rng.uniform(1.4, 2.0, n)
    boxes[:, 6] = rng.uniform(-np.pi, np.pi, n)
    p2 = np.array([[721.5377, 0.0, 609.5593, 44.85728],
                   [0.0, 721.5377, 172.854, 0.2163791],
                   [0.0, 0.0, 1.0, 0.002745884]], np.float32)
    corners = env["get_box3d_corners_helper_np"](boxes[:, :3], boxes[:, -1], boxes[:, 3:-1])
    rect = env["project_to_image_space_corners"](corners, p2)
    np.savez_compressed(os.path.join(HERE, "kitti_io.npz"), boxes=boxes, p2=p2, corners=corners.astype(np.float32),
                        rect=rect)
    print("wrote kitti_io.npz", corners.shape, rect.shape)


if __name__ == "__main__":
    main()
