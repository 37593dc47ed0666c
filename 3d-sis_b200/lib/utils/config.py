"""Global `cfg` for the hot path -- same access pattern as the reference (`from lib.utils.config
import cfg`, attribute access, yml overrides; lib/utils/config.py:16-247,288-298) but only the keys
the inference path reads carry defaults here; any other key found in a yml is stored verbatim so the
reference's experiment files load unchanged.
"""
from __future__ import annotations

import os

import yaml


class AttrDict(dict):
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = AttrDict(v) if isinstance(v, dict) and not isinstance(v, AttrDict) else v


def _defaults():
    c = AttrDict()
    c.TEST = AttrDict(RPN_NMS_THRESH=0.35, RPN_PRE_NMS_TOP_N=6000, RPN_POST_NMS_TOP_N=300)
    c.TRAIN = AttrDict(RPN_NMS_THRESH=0.7, RPN_PRE_NMS_TOP_N=12000, RPN_POST_NMS_TOP_N=2000)
    c.update(ALLOW_BORDER=0, RPN_CHANNELS=256, CLASS_POOLING_SIZE=2, CLASS_THRESH=0.9, MASK_THRESH=0.5, MAP_THRESH=0.25,
             MASK_USE_IMAGES=False, MASK_ONLY_IMAGES=False, MAX_IMAGE=400, MAX_VOLUME=2000000,
             NUM_CLASSES=0, BATCH_SIZE=1, VOXEL_SIZE=0.09375, TRUNCATED=3.0,
             NUM_ANCHORS_LEVEL1=9, NUM_ANCHORS_LEVEL2=9, NUM_ANCHORS_LEVEL3=9,
             ANCHORS_TYPE_LEVEL1="suncg", ANCHORS_TYPE_LEVEL2="suncg", ANCHORS_TYPE_LEVEL3="suncg",
             FILTER_ANCHOR_LEVEL1="", FILTER_ANCHOR_LEVEL2="", FILTER_ANCHOR_LEVEL3="",
             USE_BACKBONE=False, USE_RPN=False, USE_CLASS=False, USE_MASK=True,
             NET="ScanNet_Backbone", MASK_BACKBONE="MaskBackbone",
             USE_IMAGES=False, ONLY_IMAGES=False, USE_IMAGES_GT=True, NUM_IMAGES=1, NUM_2D_CLASSES=41,
             PRETRAINED_ENET_PATH="", IMAGE_SHAPE=[328, 256], DEPTH_SHAPE=[41, 32], NUM_IMAGE_CHANNELS=128,
             PROJ_DEPTH_MIN=0.1, PROJ_DEPTH_MAX=4.0, TEST_SAVE_DIR="", LABEL_MAP="", MODE="",
             BASE_IMAGE_PATH="", IMAGE_TYPE="color2", IMAGE_EXT=".jpg",  # frame folders (reference config.py:191-219)
             COLOR_MEAN=[0.47083, 0.44685, 0.40733], COLOR_STD=[0.27861, 0.27409, 0.28844],
             INTRINSIC=[[35.5070229, 0, 20, 0], [0, 36.9504013, 15.5, 0], [0, 0, 1, 0], [0, 0, 0, 1]])
    # where anchor tables live; the reference opens 'experiments/anchors/<name>' relative to its cwd
    c.ANCHOR_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))),
                                "experiments", "anchors")
    return c


cfg = _defaults()


def _merge(src, dst):
    for k, v in src.items():
        if isinstance(v, dict) and isinstance(dst.get(k), dict):
            _merge(v, dst[k])
        else:
            dst[k] = AttrDict(v) if isinstance(v, dict) else v


def cfg_from_file(filename):
    """Merge a yml file into the defaults (reference: lib/utils/config.py:288-298)."""
    with open(filename, "r") as f:
        _merge(yaml.safe_load(f) or {}, cfg)
    return cfg


def cfg_reset():
    cfg.clear()
    cfg.update(_defaults())
    return cfg
