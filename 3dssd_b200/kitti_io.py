"""Data formats either side of the SA path (SURVEY.md section 8f, row f4).

What enters the path: the reference's preprocessed KITTI sample files -- one pickled dict per frame written by
its preprocessing pass and read back in /root/reference/lib/dataset/dataloader/kitti_dataloader.py:103-158 (keys in
lib/dataset/maps_dict.py).  What leaves it: one KITTI result .txt per frame (kitti_dataloader.py:460-492) built from
the post-processed boxes, and the network weights, which the reference keeps in a TF checkpoint whose variable
names follow the scopes in params.py.

Everything here is host-side byte shuffling on a few hundred boxes / a few MB of points per frame; it feeds pinned
host buffers that the backbone copies to HBM, no kernels involved.
"""
import os

import numpy as np

# maps_dict.py:4-36
KEY_POINT_CLOUD = "point_cloud"
KEY_STEREO_CALIB = "stereo_calib"
KEY_SAMPLE_NAME = "sample_name"
KEY_LABEL_BOXES_3D = "label_boxes_3d"
KEY_LABEL_CLASSES = "label_classes"

KITTI_IMG_SHAPE = (375, 1242)       # anchors_util.py:54 default (h, w)


# ------------------------------------------------------------------------------------------------------------------
# input side
# ------------------------------------------------------------------------------------------------------------------
def read_sample(path):
    """One preprocessed frame -> dict.  The file is a 0-d object array holding the dict (kitti_dataloader.py:110)."""
    arr = np.load(path, allow_pickle=True)
    d = arr.item() if isinstance(arr, np.ndarray) and arr.shape == () else arr
    if not isinstance(d, dict) or KEY_POINT_CLOUD not in d:
        raise ValueError("%s: not a 3DSSD sample dict (no '%s' key)" % (path, KEY_POINT_CLOUD))
    return d


def choose_points(num_have, num_want, rng):
    """Indices of the fixed-size point set fed to the network (kitti_dataloader.py:137-147): a random subset without
    replacement when the frame has enough points, otherwise every point once (shuffled) followed by a random refill
    with replacement."""
    if num_have <= 0:
        raise ValueError("choose_points: empty point cloud")
    if num_have >= num_want:
        return rng.choice(num_have, num_want, replace=False)
    first = rng.choice(num_have, num_have, replace=False)
    refill = rng.choice(num_have, num_want - num_have, replace=True)
    return np.concatenate([first, refill], axis=0)


def calib_p2(calib):
    """3x4 camera projection of a sample: the reference stores a calibration object with a .P attribute
    (kitti_dataloader.py:158); a bare array is accepted too."""
    p = getattr(calib, "P", calib)
    p = np.asarray(p, np.float32)
    if p.shape != (3, 4):
        raise ValueError("calibration P must be 3x4, got %s" % (p.shape,))
    return p


def make_batch(samples, num_points=16384, seed=0, pin=True):
    """Stack frames into the [B, num_points, C] fp32 host block the backbone consumes (pinned, so the H2D copy inside
    the timed path is asynchronous).  Returns (points tensor, [P2 per frame], [sample name per frame])."""
    import torch
    rng = np.random.default_rng(seed)
    clouds, calibs, names = [], [], []
    for s in samples:
        pts = np.asarray(s[KEY_POINT_CLOUD], np.float32)
        clouds.append(pts[choose_points(pts.shape[0], num_points, rng)])
        calibs.append(calib_p2(s[KEY_STEREO_CALIB]) if KEY_STEREO_CALIB in s else None)
        names.append(s.get(KEY_SAMPLE_NAME, len(names)))
    block = torch.from_numpy(np.stack(clouds, axis=0))
    if pin and torch.cuda.is_available():
        block = block.pin_memory()
    return block, calibs, names


# ------------------------------------------------------------------------------------------------------------------
# output side
# ------------------------------------------------------------------------------------------------------------------
def box_corners(boxes):
    """[N,7] (x, y, z, l, h, w, ry) camera-frame boxes, origin at the bottom-face centre -> [N,8,3] corners in the order
    of box_3d_utils.py:62-87 (bottom face first, y pointing down so the top face is at y - h)."""
    boxes = np.asarray(boxes, np.float32).reshape(-1, 7)
    l, h, w, ry = boxes[:, 3], boxes[:, 4], boxes[:, 5], boxes[:, 6]
    sx = np.array([1, 1, -1, -1, 1, 1, -1, -1], np.float32) * 0.5
    sz = np.array([1, -1, -1, 1, 1, -1, -1, 1], np.float32) * 0.5
    sy = np.array([0, 0, 0, 0, -1, -1, -1, -1], np.float32)
    cx, cy, cz = l[:, None] * sx, h[:, None] * sy, w[:, None] * sz            # [N,8] box-frame offsets
    c, s = np.cos(ry)[:, None], np.sin(ry)[:, None]
    out = np.empty((boxes.shape[0], 8, 3), np.float32)
    out[:, :, 0] = c * cx + s * cz + boxes[:, 0:1]
    out[:, :, 1] = cy + boxes[:, 1:2]
    out[:, :, 2] = -s * cx + c * cz + boxes[:, 2:3]
    return out


def project_boxes_to_image(boxes, p2, img_shape=KITTI_IMG_SHAPE):
    """[N,7] boxes -> [N,4] (x1, y1, x2, y2) image rectangles clipped to the frame (anchors_util.py:54-91 with
    kitti_util.py:329-348)."""
    corners = box_corners(boxes).reshape(-1, 3)
    hom = np.concatenate([corners, np.ones((corners.shape[0], 1), corners.dtype)], axis=1)
    uvw = hom.astype(np.float64) @ np.asarray(p2, np.float64).T
    uv = (uvw[:, :2] / uvw[:, 2:3]).reshape(-1, 8, 2)
    h, w = img_shape
    rect = np.stack([np.clip(uv[:, :, 0].min(1), 0, w), np.clip(uv[:, :, 1].min(1), 0, h),
                     np.clip(uv[:, :, 0].max(1), 0, w), np.clip(uv[:, :, 1].max(1), 0, h)], axis=-1)
    return rect.astype(np.float32)


def format_kitti_result(boxes, scores, classes, p2, cls_list=("Car",), cls_thresh=0.0, img_shape=KITTI_IMG_SHAPE):
    """KITTI result lines of one frame (kitti_dataloader.py:474-490): type, truncation 0.00, occlusion 0, alpha -10,
    2-D rectangle, dimensions as h w l, location, ry, score -- boxes below cls_thresh are dropped."""
    boxes = np.asarray(boxes, np.float32).reshape(-1, 7)
    scores = np.asarray(scores, np.float32).reshape(-1)
    classes = np.asarray(classes).reshape(-1)
    keep = np.where(scores >= cls_thresh)[0]
    boxes, scores, classes = boxes[keep], scores[keep], classes[keep]
    rect = project_boxes_to_image(boxes, p2, img_shape) if len(boxes) else np.zeros((0, 4), np.float32)
    lines = []
    for b, s, c, r in zip(boxes, scores, classes, rect):
        lines.append("%s %0.2f %d %d %0.2f %0.2f %0.2f %0.2f %0.2f %0.2f %0.2f %0.2f %0.2f %0.2f %0.2f %0.9f\n" % (
            cls_list[int(c)], 0.0, 0, -10, float(r[0]), float(r[1]), float(r[2]), float(r[3]),
            float(b[4]), float(b[5]), float(b[3]), float(b[0]), float(b[1]), float(b[2]), float(b[6]), float(s)))
    return "".join(lines)


def write_kitti_result(out_dir, sample_name, boxes, scores, classes, p2, **kw):
    """One '<out_dir>/kitti_result/%06d.txt' per frame, like save_predictions (kitti_dataloader.py:465,474)."""
    sv_dir = os.path.join(out_dir, "kitti_result")
    os.makedirs(sv_dir, exist_ok=True)
    path = os.path.join(sv_dir, "%06d.txt" % int(sample_name))
    with open(path, "w") as fid:
        fid.write(format_kitti_result(boxes, scores, classes, p2, **kw))
    return path


def write_detections(out_dir, sample_names, det_block, det_count, calibs, **kw):
    """Writes the fixed-size detection block the backbone returns ([B, K, 9] = box7, score, class; counts [B])."""
    det_block = np.asarray(det_block, np.float32)
    paths = []
    for i, name in enumerate(sample_names):
        k = int(det_count[i])
        d = det_block[i, :k]
        paths.append(write_kitti_result(out_dir, name, d[:, :7], d[:, 7], d[:, 8].astype(np.int64), calibs[i], **kw))
    return paths


# ------------------------------------------------------------------------------------------------------------------
# weights
# ------------------------------------------------------------------------------------------------------------------
_SKIP_SUFFIXES = ("/Adam", "/Adam_1", "/Momentum", "/ExponentialMovingAverage")
_SKIP_NAMES = ("global_step", "beta1_power", "beta2_power")


def params_from_tf_variables(variables):
    """name -> array mapping exported from a reference checkpoint (see INTEGRATION.md for the three-line export that a
    TF-equipped machine runs; TF itself is not needed here) -> the params dict of params.py.

    Kernels are squeezed to [cin, cout]: tf_util.conv2d stores [1,1,cin,cout] (tf_util.py:88-112), conv1d
    [1,cin,cout] (tf_util.py:164-190).  Optimiser slots and counters are dropped; ':0' tensor suffixes are stripped.
    """
    out = {}
    for name, val in dict(variables).items():
        name = name[:-2] if name.endswith(":0") else name
        if name in _SKIP_NAMES or name.endswith(_SKIP_SUFFIXES):
            continue
        a = np.asarray(val, np.float32)
        if name.endswith("/weights"):
            if a.ndim < 2 or any(d != 1 for d in a.shape[:-2]):
                raise ValueError("%s: expected a 1x1 kernel, got shape %s" % (name, a.shape))
            a = a.reshape(a.shape[-2], a.shape[-1])
        out[name] = np.ascontiguousarray(a)
    for name in list(out):
        if name.endswith("/weights"):
            scope = name[: -len("/weights")]
            cout = out[name].shape[1]
            for leaf in ("biases", "bn/gamma", "bn/beta", "bn/moving_mean", "bn/moving_variance"):
                v = out.get(scope + "/" + leaf)
                if v is not None and v.shape != (cout,):
                    raise ValueError("%s/%s: shape %s does not match %d output channels" % (scope, leaf, v.shape, cout))
    return out


def make_label_batch(samples):
    """The labels of a batch of frames padded with zeros to the batch's largest count, as the reference's data provider
    concatenates them (lib/dataset/data_provider/data_provider.py:610-626): (gt_boxes [B, G, 7] fp32, gt_labels [B, G]
    int32), G = max over the frames (0 when no frame has a label).  Rows of zeros are the padding the target assigner
    skips."""
    boxes = [np.asarray(s[KEY_LABEL_BOXES_3D], np.float32).reshape(-1, 7) for s in samples]
    classes = [np.asarray(s[KEY_LABEL_CLASSES]).reshape(-1).astype(np.int32) for s in samples]
    g = max((len(b) for b in boxes), default=0)
    out_b = np.zeros((len(samples), g, 7), np.float32)
    out_c = np.zeros((len(samples), g), np.int32)
    for i, (b, c) in enumerate(zip(boxes, classes)):
        if len(b) != len(c):
            raise ValueError("frame %d has %d boxes but %d classes" % (i, len(b), len(c)))
        out_b[i, :len(b)] = b
        out_c[i, :len(c)] = c
    return out_b, out_c


KEY_LABEL_SEM_SEG = "label_sem_seg"


def make_ragged_batch(samples, pin=True):
    """The full clouds of a batch of frames for the augmentor (augment.Augmentor), in host buffers (pinned when a GPU is
    present): (points [T, 4] fp32 packed frame after frame, offsets [B + 1] int32, semantic labels [T] int32 or None when
    a frame has none, gt_boxes [B, G, 7] fp32, gt_labels [B, G] int32 padded as make_label_batch pads them)."""
    import torch
    clouds = [np.asarray(s[KEY_POINT_CLOUD], np.float32).reshape(-1, 4) for s in samples]
    offsets = np.zeros(len(clouds) + 1, np.int32)
    offsets[1:] = np.cumsum([len(c) for c in clouds])
    sem = None
    if samples and all(KEY_LABEL_SEM_SEG in s for s in samples):
        sem = np.concatenate([np.asarray(s[KEY_LABEL_SEM_SEG]).reshape(-1).astype(np.int32) for s in samples])
        if len(sem) != offsets[-1]:
            raise ValueError("label_sem_seg holds %d labels for %d points" % (len(sem), offsets[-1]))
    boxes, labels = make_label_batch(samples)
    out = [torch.from_numpy(np.concatenate(clouds, 0) if clouds else np.zeros((0, 4), np.float32)), torch.from_numpy(offsets),
           None if sem is None else torch.from_numpy(sem), torch.from_numpy(boxes), torch.from_numpy(labels)]
    if pin and torch.cuda.is_available():
        out = [t if t is None else t.pin_memory() for t in out]
    return tuple(out)


# ------------------------------------------------------------------------------------------------------------------
# ground planes (the mixup paste stands its objects on them, mixup.py)
# ------------------------------------------------------------------------------------------------------------------
def plane_path(planes_dir, sample_name):
    """'<planes_dir>/%06d.txt', the plane file of a frame (kitti_util.py:295)."""
    return os.path.join(planes_dir, "%06d.txt" % int(sample_name))


def read_plane(path):
    """get_road_plane (kitti_util.py:286-318): the 4th line of a KITTI plane file -> (a, b, c, d) float64 with the normal
    facing up (negated when b > 0: +y points down) and divided by the norm of (a, b, c).  A missing file raises."""
    if not os.path.isfile(path):
        raise FileNotFoundError("ground plane file %s does not exist" % path)
    with open(path) as fh:
        lines = fh.readlines()
    if len(lines) < 4:
        raise ValueError("%s: a plane file holds the plane on its 4th line" % path)
    plane = np.asarray([float(v) for v in lines[3].split()], np.float64)
    if plane.shape != (4,):
        raise ValueError("%s: the plane line must hold 4 numbers" % path)
    if plane[1] > 0:
        plane = -plane
    return plane / np.linalg.norm(plane[0:3])


# ------------------------------------------------------------------------------------------------------------------
# raw KITTI frames (the preprocessing pass of prepare.py reads them)
# ------------------------------------------------------------------------------------------------------------------
KEY_LABEL_DIST = "label_dist"
KEY_LABEL_NUM = "label_num"
CALIB_KEYS = ("Tr_velo_to_cam", "R0_rect", "P2")
CALIB_SHAPES = {"Tr_velo_to_cam": (3, 4), "R0_rect": (3, 3), "P2": (3, 4)}
_PNG_MAGIC = b"\x89PNG\r\n\x1a\n"


def read_velodyne(path):
    """load_velo_scan (kitti_util.py:323-326): the float32 words of a velodyne .bin as [N, 4] (x, y, z, reflectance)."""
    raw = np.fromfile(path, dtype=np.float32)
    if raw.size % 4:
        raise ValueError("%s: %d float32 words is not a whole number of (x, y, z, r) points" % (path, raw.size))
    return raw.reshape(-1, 4)


def read_calib(path):
    """read_calib_file (kitti_util.py:120-138): 'key: v v v ...' lines -> dict of float64 arrays; blank lines are
    skipped, a line without ':' or a value that is not a float list is skipped as the reference skips dates.  The three
    matrices the preprocessing needs (Tr_velo_to_cam, R0_rect, P2) must be present with 12, 9 and 12 values."""
    data = {}
    with open(path) as fh:
        for line in fh:
            line = line.rstrip()
            if not line:
                continue
            if ":" not in line:
                raise ValueError("%s: calibration line without ':': %r" % (path, line[:40]))
            key, value = line.split(":", 1)
            try:
                data[key] = np.array([float(x) for x in value.split()], np.float64)
            except ValueError:
                pass
    for k in CALIB_KEYS:
        if k not in data:
            raise ValueError("%s: no %s in the calibration file" % (path, k))
        if data[k].size != int(np.prod(CALIB_SHAPES[k])):
            raise ValueError("%s: %s holds %d values, expected %d" % (path, k, data[k].size, int(np.prod(CALIB_SHAPES[k]))))
    return data


def calib_block(calib):
    """The [33] float64 calibration block of csrc/prepare.cu: Tr_velo_to_cam (12), R0_rect (9), P2 (12), row-major."""
    return np.concatenate([np.asarray(calib[k], np.float64).reshape(-1) for k in CALIB_KEYS])


def read_label(path, cls_list=("Car",)):
    """read_label + Object3d (kitti_util.py:13-44, 279-284) and object_label_to_box_3d (box_3d_utils.py:5-22) for the
    types in cls_list: (boxes [G, 7] float64 (x, y, z, l, h, w, ry) in file order, classes [G] int64, 1-based index in
    cls_list).  Each line is rstripped and split on single spaces; fields 1.. must be floats (15 or 16 fields)."""
    boxes, classes = [], []
    with open(path) as fh:
        lines = [ln.rstrip() for ln in fh]
    for k, line in enumerate(lines):
        data = line.split(" ")
        if len(data) not in (15, 16):
            raise ValueError("%s:%d: a label line holds 15 or 16 fields, got %d" % (path, k + 1, len(data)))
        try:
            v = [float(x) for x in data[1:]]
        except ValueError:
            raise ValueError("%s:%d: label fields 1.. must be numbers: %r" % (path, k + 1, line[:60])) from None
        if data[0] in cls_list:
            h, w, l, x, y, z, ry = v[7], v[8], v[9], v[10], v[11], v[12], v[13]
            boxes.append((x, y, z, l, h, w, ry))
            classes.append(cls_list.index(data[0]) + 1)
    return np.asarray(boxes, np.float64).reshape(-1, 7), np.asarray(classes, np.int64)


def png_size(path):
    """(H, W) of a PNG from its IHDR chunk (the preprocessing uses the image shape only, never the pixels)."""
    with open(path, "rb") as fh:
        head = fh.read(24)
    if len(head) < 24 or head[:8] != _PNG_MAGIC or head[12:16] != b"IHDR":
        raise ValueError("%s: not a PNG file" % path)
    w, h = int.from_bytes(head[16:20], "big"), int.from_bytes(head[20:24], "big")
    if w <= 0 or h <= 0:
        raise ValueError("%s: PNG size %d x %d" % (path, w, h))
    return h, w
