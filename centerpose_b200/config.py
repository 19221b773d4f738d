"""Minimal cfg object with the attribute paths the hot path reads (SURVEY.md §5 "Config").

The reference uses a yacs ``CfgNode`` (``lib/config/default.py:5-177``).  Anything exposing the
same attribute paths works with this package — a yacs node, or the :class:`Cfg` attribute-dict
below (built from defaults or from one of the reference's ``experiments/*.yaml`` files).
"""
from __future__ import annotations

import copy

import yaml


class Cfg(dict):
    """dict with attribute access (``cfg.MODEL.NAME`` and ``cfg['MODEL']['NAME']``)."""

    def __init__(self, d=None):
        super().__init__()
        for k, v in (d or {}).items():
            self[k] = Cfg(v) if isinstance(v, dict) and not isinstance(v, Cfg) else v

    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def __setattr__(self, k, v):
        self[k] = v

    def __deepcopy__(self, memo):
        return Cfg({k: copy.deepcopy(v, memo) for k, v in self.items()})

    # yacs compatibility no-ops (tools/demo.py:87-92 calls defrost()/freeze())
    def defrost(self): pass
    def freeze(self): pass


_ARCH = {
    # arch: (HEAD_CONV, INTERMEDIATE_CHANNEL)   experiments/{dla_34,res_50}_512x512.yaml:28-30
    "dla_34": (256, 64),
    "res_50": (64, 256),
    "mobilenetv3": (256, 24),  # experiments/mobilenetv3_512x512.yaml:28-29
    "hrnet": (64, 32),        # experiments/hrnet_w32_512.yaml:62,73 (MODEL.EXTRA defaults to W32, archs/hrnet.py)
    "hardnet": (256, 48),     # experiments/hardnet_512x512.yaml:24,29
    "mobilenetv2": (256, 24),  # experiments/mobilenetv2_512x512.yaml:28-29
    "ghostnet": (256, 160),   # experiments/ghost_net.yaml:28-29
}

_DEFAULT = {
    "DEBUG": 0, "DEBUG_THEME": "white", "SAMPLE_METHOD": "coco_hp", "SEED": 317,
    "MODEL": {"NAME": "dla_34", "HEADS_NAME": "keypoint", "HEADS_NUM": [1, 2, 34, 2, 17, 2],
              "HEAD_CONV": 256, "INTERMEDIATE_CHANNEL": 64, "DOWN_RATIO": 4, "NUM_CLASSES": 1,
              "INPUT_H": 512, "INPUT_W": 512, "INPUT_RES": 512, "OUTPUT_RES": 128, "PAD": 31,
              "NUM_KEYPOINTS": 17, "INIT_WEIGHTS": False, "PRETRAINED": ""},
    "LOSS": {"HM_HP": True, "MSE_LOSS": False, "REG_OFFSET": True, "REG_HP_OFFSET": True, "REG_BBOX": True},
    "DATASET": {"MEAN": [0.408, 0.447, 0.470], "STD": [0.289, 0.274, 0.278]},
    "TEST": {"MODEL_PATH": "", "TASK": "multi_pose", "FLIP_TEST": False, "TEST_SCALES": [1],
             "TOPK": 100, "NMS": False, "FIX_RES": True, "VIS_THRESH": 0.3},
    # additive (not in the reference): activation precision of the CUDA backbone
    "B200": {"PRECISION": "fp16x2"},      # parity-qualified tensor-core precision; "bf16" = fast mode, "fp32" = CUDA cores
}


def default_cfg(arch: str = "dla_34") -> Cfg:
    if arch not in _ARCH:
        raise KeyError(f"no built-in defaults for arch {arch!r}; known: {sorted(_ARCH)}")
    cfg = Cfg(copy.deepcopy(_DEFAULT))
    cfg.MODEL.NAME = arch
    cfg.MODEL.HEAD_CONV, cfg.MODEL.INTERMEDIATE_CHANNEL = _ARCH[arch]
    return cfg


def load_cfg(yaml_path: str) -> Cfg:
    """Read one of the reference's experiment YAMLs (``update_config``, default.py:173-177)."""
    cfg = Cfg(copy.deepcopy(_DEFAULT))
    with open(yaml_path) as f:
        user = yaml.safe_load(f)

    def merge(dst, src):
        for k, v in src.items():
            if isinstance(v, dict) and isinstance(dst.get(k), dict):
                merge(dst[k], v)
            else:
                dst[k] = Cfg(v) if isinstance(v, dict) else v
    merge(cfg, user)
    return cfg
