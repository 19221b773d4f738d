"""ORACLE (test infrastructure, not product): functional torch-CPU fp32 restatement of the reference's MobileNetV2 (width
0.5) + MobileNetUp backbone (``'mobilenetv2'`` arch), evaluated from a reference-format ``state_dict``.

Follows ``/root/reference/lib/models/backbones/mobilenet/mobilenetv2.py``:
  * ``:34-41``    ConvBNReLU (conv, pad (k-1)//2 -> BN -> ReLU6)                -> :func:`_cbr`
  * ``:44-71``    InvertedResidual                                               -> :func:`_inverted`
  * ``:98-101``   the strides of the first block of each stage                   -> :data:`STAGE_STRIDE`
  * ``:162-183``  IDAUp (ConvTranspose2d k 2 s 2 + BN(eps 1e-3) + ReLU, + 1x1 ConvBNReLU(eps 1e-3))  -> :func:`_ida`
  * ``:185-219``  MobileNetUp                                                    -> :func:`mobilenetv2_backbone`
Block counts and channel widths come from the state_dict; strides come from the table.  Restated independently of the
product (centerpose_b200/archs/mobilenetv2.py).  Pinned by ``oracle/make_golden_mobilenetv2_ghostnet.py`` against the
reference module (``tests/golden/mbv2_*.npz``).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .dla_ref import keypoint_head

FEATS = ("feature_1", "feature_2", "feature_4", "feature_6")
# stride of each block, per feature (stages (t, c, n, s) of mobilenetv2.py:77-85 grouped at feat_id 1, 2, 4, 6)
STAGE_STRIDE = {"feature_1": [1, 2, 1], "feature_2": [2, 1, 1], "feature_4": [2, 1, 1, 1, 1, 1, 1],
                "feature_6": [2, 1, 1, 1]}


def _bn(sd, x, p, eps=1e-5):
    return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"], False,
                        0.0, eps)


def _cbr(sd, x, p, stride=1):
    w = sd[p + ".0.weight"]
    groups = x.shape[1] if w.shape[1] == 1 and x.shape[1] > 1 else 1
    return F.relu6(_bn(sd, F.conv2d(x, w, stride=stride, padding=(w.shape[2] - 1) // 2, groups=groups), p + ".1"))


def _inverted(sd, x, p, stride):
    expand = (p + ".conv.3.weight") in sd                   # conv.0 = expand, conv.1 = dw, conv.2/.3 = projection
    h = _cbr(sd, x, p + ".conv.0") if expand else x
    i = 1 if expand else 0
    h = _cbr(sd, h, f"{p}.conv.{i}", stride)
    out = _bn(sd, F.conv2d(h, sd[f"{p}.conv.{i + 1}.weight"]), f"{p}.conv.{i + 2}")
    return x + out if stride == 1 and x.shape[1] == out.shape[1] else out


def _ida(sd, x, layer, p):
    c = x.shape[1]
    up = F.relu(_bn(sd, F.conv_transpose2d(x, sd[p + ".up.0.weight"], stride=2, groups=c), p + ".up.1", 1e-3))
    lat = F.relu(_bn(sd, F.conv2d(layer, sd[p + ".conv.0.weight"]), p + ".conv.1", 1e-3))
    return up + lat


def mobilenetv2_backbone(sd, x, p="backbone_model"):
    layers = []
    for name in FEATS:
        j = 0
        if name == "feature_1":                             # the stem: ConvBNReLU(3, 16, stride 2)
            x = _cbr(sd, x, f"{p}.base.feature_1.0", 2)
            j = 1
        for stride in STAGE_STRIDE[name]:
            x = _inverted(sd, x, f"{p}.base.{name}.{j}", stride)
            j += 1
        assert f"{p}.base.{name}.{j}.conv.0.0.weight" not in sd
        layers.append(x)
    x = F.relu(_bn(sd, F.conv2d(layers[-1], sd[p + ".dla_up.conv.0.weight"]), p + ".dla_up.conv.1", 1e-3))
    for i in range(len(layers) - 1):
        x = _ida(sd, x, layers[len(layers) - 2 - i], f"{p}.dla_up.up_{i}")
    return F.relu(_bn(sd, F.conv2d(x, sd[p + ".dla_up.conv_last.0.weight"], padding=1), p + ".dla_up.conv_last.1"))


@torch.no_grad()
def forward(sd, x):
    """state_dict + (B,3,H,W) -> [hm, wh, hps, reg, hm_hp, hp_offset] logits (NCHW), as ``dla_ref.forward``."""
    sd = {k: v.to(x.device, x.dtype) for k, v in sd.items() if v.dtype.is_floating_point}
    return keypoint_head(sd, mobilenetv2_backbone(sd, x))
