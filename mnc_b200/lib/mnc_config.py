"""cfg constants consumed by the inference path and the TRAIN phase of the cascade bridge and
RPN-stage layers -- reference lib/mnc_config.py (values at :12-28, :36-105, :112-152).  Only the keys those read are
present; the YAML merge machinery is out of scope."""
import numpy as np


class _AttrDict(dict):
    __getattr__ = dict.__getitem__
    __setattr__ = dict.__setitem__


cfg = _AttrDict()
cfg.MNC_MODE = True                          # :12
cfg.USE_GPU_NMS = True                       # :16
cfg.GPU_ID = 0                               # :17
cfg.PIXEL_MEANS = np.array([[[102.9801, 115.9465, 122.7717]]])  # :20
cfg.BINARIZE_THRESH = 0.4                    # :26
cfg.MASK_SIZE = 21                           # :28
cfg.TRAIN = _AttrDict(MAX_SIZE=1000, SCALES=(600,))
cfg.TRAIN.BATCH_SIZE = 64                    # :36
cfg.TRAIN.FG_FRACTION = [0.3]                # :49
cfg.TRAIN.FG_THRESH_HI = [1.0]               # :50
cfg.TRAIN.FG_THRESH_LO = [0.5]               # :51
cfg.TRAIN.BG_FRACTION = [0.85, 0.15]         # :53
cfg.TRAIN.BG_THRESH_HI = [0.5, 0.1]          # :54
cfg.TRAIN.BG_THRESH_LO = [0.1, 0.0]          # :55
# experiments/cfgs/VGG16/mnc_5stage.yml:6 sets True for the 5-stage net; the default is :64's
cfg.TRAIN.BBOX_NORMALIZE_TARGETS_PRECOMPUTED = False
cfg.TRAIN.BBOX_THRESH = 0.5                  # :65
cfg.TRAIN.BBOX_NORMALIZE_MEANS = (0.0, 0.0, 0.0, 0.0)   # :66
cfg.TRAIN.BBOX_NORMALIZE_STDS = (0.1, 0.1, 0.2, 0.2)    # :67
cfg.TRAIN.BBOX_INSIDE_WEIGHTS = (1.0, 1.0, 1.0, 1.0)    # :69
cfg.TRAIN.RPN_POSITIVE_OVERLAP = 0.7         # :75
cfg.TRAIN.RPN_NEGATIVE_OVERLAP = 0.3         # :77
cfg.TRAIN.RPN_CLOBBER_POSITIVES = False      # :79
cfg.TRAIN.RPN_FG_FRACTION = 0.5              # :82
cfg.TRAIN.RPN_BATCHSIZE = 256                # :84
cfg.TRAIN.RPN_NMS_THRESH = 0.7               # :86
cfg.TRAIN.RPN_PRE_NMS_TOP_N = 12000          # :88
# :90 sets 2000; experiments/cfgs/VGG16/mnc_5stage.yml:4 sets 300 for the 5-stage net
cfg.TRAIN.RPN_POST_NMS_TOP_N = 300
cfg.TRAIN.RPN_MIN_SIZE = 16                  # :92
cfg.TRAIN.RPN_BBOX_INSIDE_WEIGHTS = (1.0, 1.0, 1.0, 1.0)   # :94
cfg.TRAIN.RPN_POSITIVE_WEIGHT = -1.0         # :98
cfg.TRAIN.MIX_INDEX = True                   # :100
cfg.TRAIN.FG_SEG_THRESH = 0.5                # :105
cfg.TEST = _AttrDict()
cfg.TEST.SCALES = (600,)                     # :115
cfg.TEST.MAX_SIZE = 1000                     # :118
cfg.TEST.NMS = 0.3                           # :122
cfg.TEST.RPN_NMS_THRESH = 0.7                # :126
cfg.TEST.RPN_PRE_NMS_TOP_N = 6000            # :128
cfg.TEST.RPN_POST_NMS_TOP_N = 300            # :130
cfg.TEST.RPN_MIN_SIZE = 16                   # :132
cfg.TEST.MASK_MERGE_IOU_THRESH = 0.5         # :136
cfg.TEST.MASK_MERGE_NMS_THRESH = 0.3         # :137
cfg.TEST.USE_MASK_MERGE = True               # :151
cfg.TEST.USE_GPU_MASK_MERGE = True           # :152
cfg.TEST.CFM_INPUT_MASK_SIZE = 14            # :138
cfg.TEST.MAX_ROIS_GPU = [2000]               # :144
cfg.TEST.GROUP_SCALE = 1                     # :145
cfg.TEST.USE_TOP_K_MCG = 0                   # :148
