"""ORACLE (test infrastructure, not product): functional torch-CPU fp32 restatement of the reference's HarDNet backbone
(``'hardnet'`` arch), evaluated from a reference-format ``state_dict``.

Follows ``/root/reference/lib/models/backbones/hardnet.py``:
  * ``:12-22``    ConvLayer (conv k x k, pad k//2, no bias -> BN -> ReLU)   -> :func:`_conv_layer`
  * ``:25-86``    HarDBlock.forward                                         -> :func:`_block`
  * ``:89-103``   TransitionUp (bilinear, align_corners=True, then concat)  -> inside :func:`hardnet_backbone`
  * ``:106-188``  hardnet.__init__ / forward                                -> :func:`hardnet_backbone`
Layer counts, strides and kernel sizes come from the state_dict (which layers exist, their weight shapes); the link rule
is restated here independently of the product (centerpose_b200/archs/hardnet.py).
Pinned by ``oracle/make_golden_hardnet.py`` against the reference module (``tests/golden/hardnet_*.npz``).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .dla_ref import _bn, keypoint_head

STRIDE2 = {"base.0", "base.2"}


def _conv_layer(sd, x, p, stride=1):
    w = sd[p + ".conv.weight"]
    return F.relu(_bn(sd, F.conv2d(x, w, None, stride=stride, padding=w.shape[2] // 2), p + ".norm"))


def _n_layers(sd, p):
    n = 0
    while f"{p}.layers.{n}.conv.weight" in sd:
        n += 1
    return n


def _block(sd, x, p):
    outs = [x]
    n = _n_layers(sd, p)
    for l in range(1, n + 1):
        src = [outs[l - 2 ** i] for i in range(l.bit_length()) if l % 2 ** i == 0]
        outs.append(_conv_layer(sd, torch.cat(src, 1) if len(src) > 1 else src[0], f"{p}.layers.{l - 1}"))
    return torch.cat([outs[l] for l in range(1, n + 1) if l % 2 == 1 or l == n], 1)


def hardnet_backbone(sd, x, p="backbone_model"):
    for i in range(4):
        x = _conv_layer(sd, x, f"{p}.base.{i}", 2 if f"base.{i}" in STRIDE2 else 1)
    skips = []
    i = 4
    while f"{p}.base.{i}.layers.0.conv.weight" in sd:
        blk = _block(sd, x, f"{p}.base.{i}")
        x = _conv_layer(sd, blk, f"{p}.base.{i + 1}")
        if f"{p}.base.{i + 3}.layers.0.conv.weight" in sd:             # a later stage follows: skip + AvgPool2d(2, 2)
            skips.append(blk)
            x = F.avg_pool2d(x, 2, 2)
        i += 3
    for u in range(len(skips)):
        skip = skips.pop()
        x = F.interpolate(x, size=skip.shape[2:], mode="bilinear", align_corners=True)
        x = _conv_layer(sd, torch.cat([x, skip], 1), f"{p}.conv1x1_up.{u}")
        x = _block(sd, x, f"{p}.denseBlocksUp.{u}")
    return x


@torch.no_grad()
def forward(sd, x):
    """state_dict + (B,3,H,W) fp32 -> [hm, wh, hps, reg, hm_hp, hp_offset] logits (NCHW), as ``dla_ref.forward``."""
    sd = {k: v.float() for k, v in sd.items() if v.dtype.is_floating_point}
    return keypoint_head(sd, hardnet_backbone(sd, x))
