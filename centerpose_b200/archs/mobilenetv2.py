"""MobileNetV2 + MobileNetUp (the reference's ``'mobilenetv2'`` arch, ``lib/models/backbones/mobilenet/mobilenetv2.py``):
parameter tree + lowering to fused ops.  Stride-4 output with 24 channels (``experiments/mobilenetv2_512x512.yaml``:
INTERMEDIATE_CHANNEL 24).

Network.  ``get_mobile_pose_netv2`` always builds ``mobilenetv2_5`` (width 0.5) whatever ``num_layers`` says
(``mobilenetv2.py:254-259``), and so does this module.  The stem is a 3x3 / stride-2 ConvBNReLU (conv -> BN -> ReLU6),
then 17 inverted residual blocks [1x1 expand ConvBNReLU (absent when t = 1) -> 3x3 depthwise ConvBNReLU (stride s) ->
1x1 projection + BN (+ the block input when stride 1 and in == out)].  The blocks are grouped into ``feature_1``,
``feature_2``, ``feature_4`` and ``feature_6`` (strides 4, 8, 16, 32; 16, 16, 48, 160 channels).  MobileNetUp: a 1x1
ConvBNReLU 160 -> 24 on the stride-32 map, then three IDAUp steps, each ``relu(bn(up(x))) + relu(bn(conv1x1(skip)))``
with a depthwise ConvTranspose2d(k 2, stride 2, pad 0), and a final 3x3 ConvBNReLU.  MobileNetUp's BatchNorms, except
``conv_last``'s, use eps 1e-3 (``mobilenetv2.py:167,172,189``).

Lowering.
  * Channels are zero-padded to the next multiple of 16, as in archs/mobilenet.py (8 -> 16, 24 -> 32): the padding's
    folded weights and biases are zero, so the padded channels stay exactly 0 through ReLU6, ReLU and the adds.  The
    8-channel projection of the first block thereby runs on the narrowest tensor-core tile.
  * ReLU6 is an epilogue activation (FLAG_RELU6) of the stem, the expand convs and the depthwise convs.
  * IDAUp: the 1x1 lateral conv (+BN+ReLU) writes the skip operand; the deconv + BN + ReLU + skip add is one
    DWDECONV_ADD op in its bias form (PlanBuilder.up_add with b, act, stride 2, pad 0).
"""
from __future__ import annotations

import torch
from torch import nn

from .common import StateView, attach, bn, conv
from ..plan import BN_EPS, PlanBuilder, Sym, fold_bn

WIDTH = 0.5                                   # mobilenetv2_5 (mobilenetv2.py:246-250)
# (t, c, n, s)   mobilenetv2.py:77-85
SETTING = [(1, 16, 1, 1), (6, 24, 2, 2), (6, 32, 3, 2), (6, 64, 4, 2), (6, 96, 3, 1), (6, 160, 3, 2), (6, 320, 1, 1)]
FEAT_ID = (1, 2, 4, 6)
OUT_DIM = 24
UP_EPS = 1e-3                                 # MobileNetUp.conv and IDAUp's BatchNorms


def make_divisible(v: float, divisor: int = 8) -> int:
    new_v = max(divisor, int(v + divisor / 2) // divisor * divisor)
    if new_v < 0.9 * v:
        new_v += divisor
    return new_v


STEM_C = make_divisible(32 * WIDTH)


def layout():
    """-> [(feature name, first index, [(in, hidden, out, stride, t), ...])] and the four features' channels.  feature_1
    holds the stem at index 0, so its blocks start at 1."""
    feats, chans, cur, c_in = [], [], [], STEM_C
    for sid, (t, c, n, s) in enumerate(SETTING):
        oup = make_divisible(c * WIDTH)
        for i in range(n):
            cur.append((c_in, int(round(c_in * t)), oup, s if i == 0 else 1, t))
            c_in = oup
        if sid in FEAT_ID:
            feats.append((f"feature_{sid}", 1 if not feats else 0, cur))
            chans.append(oup)
            cur = []
    return feats, chans


def feature_channels(cfg=None) -> int:
    return OUT_DIM


def padded(c: int) -> int:
    return (c + 15) // 16 * 16


def _bn_eps(c, eps):
    return nn.BatchNorm2d(c, eps=eps, momentum=0.1)


def build_params(cfg=None) -> nn.Module:
    root = nn.Module()
    attach(root, "base.feature_1.0.0", conv(3, STEM_C, 3, 2, 1)); attach(root, "base.feature_1.0.1", bn(STEM_C))
    feats, chans = layout()
    for name, j0, blocks in feats:
        for j, (inp, hid, oup, s, t) in enumerate(blocks, j0):
            p = f"base.{name}.{j}.conv"
            i = 0
            if t != 1:
                attach(root, f"{p}.0.0", conv(inp, hid, 1)); attach(root, f"{p}.0.1", bn(hid))
                i = 1
            attach(root, f"{p}.{i}.0", nn.Conv2d(hid, hid, 3, s, 1, groups=hid, bias=False))
            attach(root, f"{p}.{i}.1", bn(hid))
            attach(root, f"{p}.{i + 1}", conv(hid, oup, 1)); attach(root, f"{p}.{i + 2}", bn(oup))
    # MobileNetUp.__init__ (mobilenetv2.py:186-211): conv, conv_last, then up_0.. for the shallower features
    rev = chans[::-1]
    attach(root, "dla_up.conv.0", conv(rev[0], OUT_DIM, 1)); attach(root, "dla_up.conv.1", _bn_eps(OUT_DIM, UP_EPS))
    attach(root, "dla_up.conv_last.0", conv(OUT_DIM, OUT_DIM, 3, 1, 1)); attach(root, "dla_up.conv_last.1", bn(OUT_DIM))
    for i, c in enumerate(rev[1:]):
        attach(root, f"dla_up.up_{i}.up.0", nn.ConvTranspose2d(OUT_DIM, OUT_DIM, 2, stride=2, padding=0, groups=OUT_DIM,
                                                               bias=False))
        attach(root, f"dla_up.up_{i}.up.1", _bn_eps(OUT_DIM, UP_EPS))
        attach(root, f"dla_up.up_{i}.conv.0", conv(c, OUT_DIM, 1)); attach(root, f"dla_up.up_{i}.conv.1", _bn_eps(OUT_DIM, UP_EPS))
    with torch.no_grad():                                         # mobilenetv2.py:104-112, 199-211
        for m in root.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out")
            elif isinstance(m, nn.ConvTranspose2d):               # fill_up_weights for k = 2: the (0, 0) tap only
                m.weight.zero_()
                m.weight[:, 0, 0, 0] = 1.0
    return root


# ------------------------------------------------------------------------------------------ lowering
def _rows(t: torch.Tensor, n: int) -> torch.Tensor:
    """zero-pad dim 0 of a folded weight / bias to n rows"""
    if t.shape[0] == n:
        return t
    out = torch.zeros(n, *t.shape[1:], dtype=t.dtype, device=t.device)
    out[:t.shape[0]] = t
    return out


def _pconv(pb: PlanBuilder, P: StateView, x: Sym, ckey: str, bkey: str, co_p: int, act=None, res=None, eps=BN_EPS):
    """k x k conv (pad k // 2) + folded BN on zero-padded channels"""
    w, b = fold_bn(P(ckey + ".weight"), None, P.bn(bkey), eps=eps)
    if w.shape[1] < x.C:
        w = torch.nn.functional.pad(w, (0, 0, 0, 0, 0, x.C - w.shape[1]))
    k = w.shape[2]
    return pb.conv([x], _rows(w, co_p), _rows(b, co_p), stride=1, pad=k // 2, act=act, res=res)


def _inverted_residual(pb: PlanBuilder, P: StateView, x: Sym, p: str, inp: int, hid: int, oup: int, s: int, t: int) -> Sym:
    """InvertedResidual.forward (mobilenetv2.py:45-71)"""
    h, i = x, 0
    if t != 1:
        h = _pconv(pb, P, x, f"{p}.0.0", f"{p}.0.1", padded(hid), act="relu6")
        i = 1
    w, b = fold_bn(P(f"{p}.{i}.0.weight"), None, P.bn(f"{p}.{i}.1"))         # (hid, 1, 3, 3)
    h = pb.dwconv(h, _rows(w, h.C), _rows(b, h.C), stride=s, act="relu6")
    res = x if (s == 1 and inp == oup) else None
    return _pconv(pb, P, h, f"{p}.{i + 1}", f"{p}.{i + 2}", padded(oup), res=res)


def lower(pb: PlanBuilder, P: StateView, x: Sym) -> Sym:
    """MobileNetSeg.forward (mobilenetv2.py:221-224) -> MobileNetUp output (24 real channels in 32, stride 4)."""
    w, b = fold_bn(P("base.feature_1.0.0.weight"), None, P.bn("base.feature_1.0.1"))
    t = pb.stem(x, w, b, 3, 2, 1, act="relu6")
    feats = []
    for name, j0, blocks in layout()[0]:
        for j, (inp, hid, oup, s, tt) in enumerate(blocks, j0):
            t = _inverted_residual(pb, P, t, f"base.{name}.{j}.conv", inp, hid, oup, s, tt)
        feats.append(t)
    o_p = padded(OUT_DIM)
    y = _pconv(pb, P, feats[-1], "dla_up.conv.0", "dla_up.conv.1", o_p, act="relu", eps=UP_EPS)
    for i in range(len(feats) - 1):                               # MobileNetUp.forward (:213-219) -> IDAUp (:174-179)
        skip = _pconv(pb, P, feats[len(feats) - 2 - i], f"dla_up.up_{i}.conv.0", f"dla_up.up_{i}.conv.1", o_p, act="relu",
                      eps=UP_EPS)
        wu, bu = fold_bn(P(f"dla_up.up_{i}.up.0.weight"), None, P.bn(f"dla_up.up_{i}.up.1"), eps=UP_EPS)   # (24, 1, 2, 2)
        y = pb.up_add(y, skip, _rows(wu, o_p), b=_rows(bu, o_p), act="relu", stride=2, pad=0)
    return _pconv(pb, P, y, "dla_up.conv_last.0", "dla_up.conv_last.1", o_p, act="relu")
