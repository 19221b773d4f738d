"""ORACLE (test infrastructure, not product): functional torch-CPU fp32 restatement of the reference's GhostNet backbone
(``'ghostnet'`` arch), evaluated from a reference-format ``state_dict``.

Follows ``/root/reference/lib/models/backbones/ghost_net.py``:
  * ``:31-45``    SELayer (avg pool -> Linear -> ReLU -> Linear -> clamp(0, 1) -> x * gate)  -> :func:`_se`
  * ``:48-53``    depthwise_conv (dw conv -> BN [-> ReLU])                                  -> :func:`_dw`
  * ``:56-78``    GhostModule (1x1 primary, 3x3 depthwise cheap, concat, [:oup])            -> :func:`_ghost`
  * ``:81-110``   GhostBottleneck                                                           -> :func:`_bottleneck`
  * ``:153-158``  GhostNet.forward (features, then bilinear align_corners to 128 x 128)     -> :func:`ghostnet_backbone`
Which blocks have a stride-2 depthwise conv, an SE layer or a conv shortcut, and every width, come from the state_dict;
the stride of a block is 2 exactly when its bottleneck holds the depthwise conv (``:92``).  Restated independently of
the product (centerpose_b200/archs/ghostnet.py).  Pinned by ``oracle/make_golden_mobilenetv2_ghostnet.py`` against the
reference module (``tests/golden/ghostnet_512.npz``).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .dla_ref import _bn, keypoint_head


def _dw(sd, x, p, stride, relu):
    w = sd[p + ".0.weight"]
    y = _bn(sd, F.conv2d(x, w, stride=stride, padding=w.shape[2] // 2, groups=x.shape[1]), p + ".1")
    return F.relu(y) if relu else y


def _ghost(sd, x, p, oup, relu):
    x1 = _bn(sd, F.conv2d(x, sd[p + ".primary_conv.0.weight"]), p + ".primary_conv.1")
    x1 = F.relu(x1) if relu else x1
    x2 = _dw(sd, x1, p + ".cheap_operation", 1, relu)
    return torch.cat([x1, x2], 1)[:, :oup]


def _se(sd, x, p):
    y = F.adaptive_avg_pool2d(x, 1).flatten(1)
    y = F.relu(F.linear(y, sd[p + ".fc.0.weight"], sd[p + ".fc.0.bias"]))
    y = F.linear(y, sd[p + ".fc.2.weight"], sd[p + ".fc.2.bias"])
    return x * torch.clamp(y, 0, 1)[:, :, None, None]


def _bottleneck(sd, x, p):
    hid = sd[p + ".conv.0.primary_conv.0.weight"].shape[0] + sd[p + ".conv.0.cheap_operation.0.weight"].shape[0]
    oup = sd[p + ".conv.3.primary_conv.0.weight"].shape[0] + sd[p + ".conv.3.cheap_operation.0.weight"].shape[0]
    stride = 2 if (p + ".conv.1.0.weight") in sd else 1
    h = _ghost(sd, x, p + ".conv.0", hid, True)
    if stride == 2:
        h = _dw(sd, h, p + ".conv.1", 2, False)
    if (p + ".conv.2.fc.0.weight") in sd:
        h = _se(sd, h, p + ".conv.2")
    y = _ghost(sd, h, p + ".conv.3", oup, False)
    if (p + ".shortcut.1.weight") in sd:
        sc = _dw(sd, x, p + ".shortcut.0", stride, True)
        sc = _bn(sd, F.conv2d(sc, sd[p + ".shortcut.1.weight"]), p + ".shortcut.2")
    else:
        sc = x
    return y + sc


def ghostnet_backbone(sd, x, p="backbone_model"):
    x = F.relu(_bn(sd, F.conv2d(x, sd[p + ".features.0.0.weight"], stride=2, padding=1), p + ".features.0.1"))
    i = 1
    while f"{p}.features.{i}.conv.0.primary_conv.0.weight" in sd:
        x = _bottleneck(sd, x, f"{p}.features.{i}")
        i += 1
    return F.interpolate(x, size=(128, 128), mode="bilinear", align_corners=True)


@torch.no_grad()
def forward(sd, x):
    """state_dict + (B,3,H,W) fp32 -> [hm, wh, hps, reg, hm_hp, hp_offset] logits (NCHW), as ``dla_ref.forward``."""
    sd = {k: v.float() for k, v in sd.items() if v.dtype.is_floating_point}
    return keypoint_head(sd, ghostnet_backbone(sd, x))
