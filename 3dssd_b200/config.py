"""Backbone architecture tables, as data.

ARCH_3DSSD is the FIRST_STAGE.ARCHITECTURE list of /root/reference/configs/kitti/3dssd/3dssd.yaml:46-67, with the
16 positional fields documented at /root/reference/lib/core/config.py:207-219:
  0 xyz_index, 1 feature_index, 2 radius_list, 3 nsample_list, 4 mlp_list, 5 bn,
  6 fps_sample_range_list, 7 fps_method_list, 8 npoint_list, 9 former_fps_idx, 10 use_attention,
  11 layer_type, 12 scope, 13 dilated_group, 14 vote_ctr_index, 15 aggregation_channel
"""

ARCH_3DSSD = [
    [[0], [0], [0.2, 0.4, 0.8], [32, 32, 64], [[16, 16, 32], [16, 16, 32], [32, 32, 64]], True,
     [-1], ['D-FPS'], [4096],
     -1, False, 'SA_Layer', 'layer1', True, -1, 64],
    [[1], [1], [0.4, 0.8, 1.6], [32, 32, 64], [[64, 64, 128], [64, 64, 128], [64, 96, 128]], True,
     [-1], ['FS'], [512],
     -1, False, 'SA_Layer', 'layer2', True, -1, 128],
    [[2], [2], [1.6, 3.2, 4.8], [32, 32, 32], [[128, 128, 256], [128, 192, 256], [128, 256, 256]], True,
     [512, -1], ['F-FPS', 'D-FPS'], [256, 256],
     -1, False, 'SA_Layer', 'layer3', True, -1, 256],
    [[3], [3], [], [], [], True,
     [256, -1], ['F-FPS', 'D-FPS'], [256, 0],
     -1, False, 'SA_Layer', 'vote', False, -1, 256],
    [[4], [4], -1, -1, [128], True,
     [-1], [-1], [-1],
     -1, -1, 'Vote_Layer', 'vote', False, -1, -1],
    [[3], [3], [4.8, 6.4], [16, 32], [[256, 256, 512], [256, 512, 1024]], True,
     [-1], ['D-FPS'], [256],
     -1, False, 'SA_Layer', 'layer4', False, 5, 512],
]

# MODEL.MAX_TRANSLATE_RANGE (3dssd.yaml:39)
MAX_TRANSLATE_RANGE = (-3.0, -2.0, -3.0)
# MODEL.NETWORK.AGGREGATION_SA_FEATURE (3dssd.yaml:44)
AGGREGATION_SA_FEATURE = True
# points per scene after the loader's resampling (3dssd.yaml:36, lib/dataset/placeholders.py:26)
POINTS_NUM = 16384
INPUT_CHANNELS = 4  # x, y, z, intensity

# PointRCNN's first stage (the RPN): FIRST_STAGE.ARCHITECTURE of
# /root/reference/configs/kitti/pointrcnn/tiny_pointrcnn_stage1.yaml:48-81.  The model sets AGGREGATION_SA_FEATURE to
# False (yaml:45), so the aggregation_channel fields below are not used: build it with aggregation=False.
ARCH_POINTRCNN_RPN = [
    [[0], [0], [0.1, 0.5], [16, 32], [[16, 16, 32], [32, 32, 64]], True,
     [-1], ['D-FPS'], [4096],
     -1, False, 'SA_Layer', 'rpn_layer1', False, -1, 128],
    [[1], [1], [0.5, 1.0], [16, 32], [[64, 64, 128], [64, 96, 128]], True,
     [-1], ['D-FPS'], [1024],
     -1, False, 'SA_Layer', 'rpn_layer2', False, -1, 256],
    [[2], [2], [1.0, 2.0], [16, 32], [[128, 196, 256], [128, 196, 256]], True,
     [-1], ['D-FPS'], [256],
     -1, False, 'SA_Layer', 'rpn_layer3', False, -1, 256],
    [[3], [3], [2.0, 4.0], [16, 32], [[256, 256, 512], [256, 384, 512]], True,
     [-1], ['D-FPS'], [64],
     -1, False, 'SA_Layer', 'rpn_layer4', False, -1, 256],
    [[3, 4], [3, 4], -1, -1, [512, 512], True,
     [], [], [],
     -1, False, 'FP_Layer', 'rpn_fp_layer4', False, -1, 256],
    [[2, 5], [2, 5], -1, -1, [512, 512], True,
     [], [], [],
     -1, False, 'FP_Layer', 'rpn_fp_layer3', False, -1, 256],
    [[1, 6], [1, 6], -1, -1, [256, 256], True,
     [], [], [],
     -1, False, 'FP_Layer', 'rpn_fp_layer2', False, -1, 256],
    [[0, 7], [0, 7], -1, -1, [128, 128], True,
     [], [], [],
     -1, False, 'FP_Layer', 'rpn_fp_layer1', False, -1, 256],
]
AGGREGATION_POINTRCNN = False      # MODEL.NETWORK.AGGREGATION_SA_FEATURE (tiny_pointrcnn_stage1.yaml:45)

# The class list of the single-stage model (DATASET.KITTI.CLS_LIST): label k is the 1-based place of the class in the
# list, 0 is padding.  The valid names are the eight KITTI keys of g_type_mean_size (lib/utils/model_util.py:19-26),
# with their mean (l, h, w) in metres.
SYNC_BN = False                # MODEL.NETWORK.SYNC_BN: BatchNorm statistics over every GPU's scenes (dist.DataParallel)
CLS_LIST = ('Car',)
CLASS_MEAN_SIZE = {
    'Car': (3.88311640418, 1.62856739989, 1.52563191462), 'Van': (5.06763659, 1.9007158, 2.20532825),
    'Truck': (10.13586957, 2.58549199, 3.2520595), 'Pedestrian': (0.84422524, 1.76255119, 0.66068622),
    'Person_sitting': (0.80057803, 1.27450867, 0.5983815), 'Cyclist': (1.76282397, 1.73698127, 0.59706367),
    'Tram': (16.17150617, 2.53246914, 3.53079012), 'Misc': (3.64300781, 1.54298177, 1.92320313),
}


def check_cls_list(cls_list):
    """A class list as a tuple of names: a comma-separated string or a sequence of 1..8 distinct names of
    CLASS_MEAN_SIZE.  Anything else raises ValueError."""
    names = tuple(c.strip() for c in cls_list.split(",")) if isinstance(cls_list, str) else tuple(cls_list)
    bad = [c for c in names if c not in CLASS_MEAN_SIZE]
    if bad:
        raise ValueError("unknown class name(s) %s; the valid names are %s" % (bad, ", ".join(CLASS_MEAN_SIZE)))
    if not 1 <= len(names) <= len(CLASS_MEAN_SIZE) or len(set(names)) != len(names):
        raise ValueError("a class list holds 1..%d distinct names, got %r" % (len(CLASS_MEAN_SIZE), names))
    return names


# Detection heads: (xyz_index, feature_index, op_type, mlp_list, bn, layer_type, scope), with the MODEL.FIRST_STAGE
# constants that select and parametrise their regression and post-processing.
HEAD_3DSSD = [[6], [6], 'conv1d', [128], True, 'Det', '']                     # 3dssd.yaml:68
STAGE_3DSSD = {"REGRESSION": "Dist-Anchor-free", "MAX_OUTPUT_NUM": 100, "NMS_THRESH": 0.1}   # 3dssd.yaml:70-72
HEAD_POINTRCNN_RPN = [[8], [8], 'conv1d', [], True, 'Det', 'rpn_head']       # tiny_pointrcnn_stage1.yaml:82
STAGE_POINTRCNN_RPN = {                                                        # tiny_pointrcnn_stage1.yaml:102-116
    "REGRESSION": "Bin-Anchor", "MAX_OUTPUT_NUM": 100, "NMS_THRESH": 0.85,
    "HALF_BIN_SEARCH_RANGE": 3.0, "BIN_CLASS_NUM": 12, "CLS_ACTIVATION": "Sigmoid",
    # the Car mean size (l, h, w), the one anchor of CLS_LIST ('Car',): g_type_mean_size['Kitti_Car'] (lib/utils/model_util.py:19)
    "ANCHOR_SIZE": (3.88311640418, 1.62856739989, 1.52563191462),
}

# PointRCNN's two-stage detector at test time: /root/reference/configs/kitti/pointrcnn/tiny_pointrcnn_stage2_test.yaml.
# The RPN is ARCH_POINTRCNN_RPN / HEAD_POINTRCNN_RPN with the test yaml's FIRST_STAGE post-processing (yaml:104-117: NMS
# at 0.8 instead of stage1.yaml's 0.85).
STAGE_POINTRCNN_RPN_TEST = dict(STAGE_POINTRCNN_RPN, NMS_THRESH=0.8)
# NETWORK.FIRST_STAGE.POINTS_POOLER (yaml:85): type, info keys, info conv channels, points per proposal, context range,
# (PointsPool-only voxel grid), (PointsPool-only VFE channels), bn, scope
POINTS_POOLER_POINTRCNN = ['RegionPool', ['mask', 'dist'], [128], 512, 1.0, [6, 6, 6, 10], [128], True, 'roi_pool']
POOLER_MASK_THRESHOLD = 0.5        # NETWORK.FIRST_STAGE.POOLER_MASK_THRESHOLD (yaml:86)
# NETWORK.SECOND_STAGE.ARCHITECTURE (yaml:89-102).  Index 0 of its lists is the proposal centres
# (cast_bottom_to_center(proposals)[..., :3], double_stage_detector.py:192,210), index 1 the pooled points.
ARCH_POINTRCNN_RCNN = [
    [[1], [1], [0.2], [64], [[128, 128, 128]], True,
     [-1], ['D-FPS'], [128],
     -1, False, 'SA_Layer', 'rcnn_layer1', False, -1, 128],
    [[2], [2], [0.4], [64], [[128, 128, 256]], True,
     [-1], ['D-FPS'], [32],
     -1, False, 'SA_Layer', 'rcnn_layer2', False, -1, 256],
    [[3], [3], [], [], [256, 256, 512], True,
     [], [], [],
     -1, False, 'SA_Layer_SSG_Last', 'rcnn_layer3', False, -1, 256],
]
HEAD_POINTRCNN_RCNN = [[0], [4], 'conv1d', [256], True, 'Det', 'rcnn_head']   # yaml:103
STAGE_POINTRCNN_RCNN = {                                                        # MODEL.SECOND_STAGE, yaml:118-136
    "REGRESSION": "Bin-Anchor", "MAX_OUTPUT_NUM": 100, "NMS_THRESH": 0.1,
    "HALF_BIN_SEARCH_RANGE": 1.5, "BIN_CLASS_NUM": 6, "CLS_ACTIVATION": "Softmax",
}

# BASELINE.json configs[0] / SURVEY.md section 8d "config 1": one SA layer N=4096 -> 1024, plain ball query
ARCH_SINGLE_SA = [
    [[0], [0], [0.4], [32], [[64, 64, 128]], True,
     [-1], ['D-FPS'], [1024],
     -1, False, 'SA_Layer', 'layer1', False, -1, -1],
]


def layer_channels(arch, in_channels, aggregation=None):
    """Feature channel count after every layer of `arch` (index 0 = network input).  aggregation: whether SA layers end
    in their aggregation conv (MODEL.NETWORK.AGGREGATION_SA_FEATURE); None takes AGGREGATION_SA_FEATURE."""
    aggregation = AGGREGATION_SA_FEATURE if aggregation is None else aggregation
    ch = [in_channels]
    for spec in arch:
        ltype, mlps, agg = spec[11], spec[4], spec[15]
        cin = ch[spec[1][0]]
        if ltype == 'SA_Layer':
            if len(spec[2]) == 0:
                ch.append(cin)
            elif agg is not None and agg != -1 and aggregation:
                ch.append(agg)
            else:
                ch.append(sum(m[-1] for m in mlps))
        elif ltype == 'Vote_Layer':
            ch.append(mlps[-1])
        elif ltype in ('SA_Layer_SSG_Last', 'FP_Layer'):
            ch.append(mlps[-1])
        else:
            raise ValueError(ltype)
    return ch
