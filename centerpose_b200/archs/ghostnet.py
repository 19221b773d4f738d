"""GhostNet (the reference's ``'ghostnet'`` arch, ``lib/models/backbones/ghost_net.py``): parameter tree + lowering to
fused ops.  160 channels, always resized to 128 x 128 (``experiments/ghost_net.yaml``: INTERMEDIATE_CHANNEL 160).

Network.  A 3x3 / stride-2 conv -> BN -> ReLU stem (16 channels), then 16 Ghost bottlenecks (``ghost_net.py:81-110``,
table ``:176-193``): GhostModule(in -> hidden, ReLU) -> [3x3 / 5x5 depthwise conv + BN, stride 2 blocks only] ->
[SELayer] -> GhostModule(hidden -> out, no activation), plus the shortcut: the input itself when stride 1 and
in == out, else a 3x3 depthwise conv + BN + ReLU (stride s) -> 1x1 conv + BN.  A GhostModule (``:51-78``) is a 1x1
conv + BN (+ReLU) giving ceil(out / 2) "primary" channels, a 3x3 depthwise conv + BN (+ReLU) of those giving as many
"cheap" channels, and the concatenation of both, cut to ``out`` channels.  SELayer (``:31-45``): global average pool ->
Linear (C -> C/4, bias) -> ReLU -> Linear (C/4 -> C, bias) -> clamp(0, 1) -> x * gate.  Only the stem and the first two
bottlenecks have stride 2, so the features are at stride 8; ``forward`` then resizes them (bilinear, align_corners) to a
FIXED 128 x 128 (``:154-156``), whatever the input size.  Only a 512 x 512 input gives a stride-4 map; at any other size
the heads see the same geometrically stretched map as in the reference, and the decoded coordinates are as meaningless
as the reference's.  This module reproduces that; it does not correct it.

Lowering.
  * A ghost module's concatenation is never materialised: its output is a list of two slabs ``(Sym, real channels)``,
    primary and cheap, each zero-padded to the next multiple of 16 (the counts are multiples of 4: 8, 12, 20, 36, 92 ...);
    a consumer conv's weight columns are scattered over the slabs (:func:`archs.common.scatter_columns`, as in
    archs/hardnet.py).  ``[:out]`` is a no-op for every entry of the table (out is even); :func:`ghost_module` asserts it.
  * Per-channel ops (the depthwise convs, the SE gate, the shortcut add, the resize) run on each slab.  A producer of
    ``out`` channels that the block output adds into (the shortcut's 1x1 conv) is split into one conv per slab, each
    with the ghost module's slab as its residual operand.  The identity shortcut is one add per slab (UPSAMPLE_ADD with factor 1).
  * SE: per-slab average pools feed the first FC as a two-input 1x1 conv on the 1x1 map (ReLU); the second FC is one
    1x1 conv per slab with the clamp as its epilogue activation (FLAG_CLIP01), and SCALE_ADD applies each gate.  The
    SE sits before the second ghost module, so no shortcut joins it.
"""
from __future__ import annotations

import math
from typing import List, Tuple

import torch
from torch import nn

from .common import StateView, attach, bn, conv, scatter_columns
from ..plan import PlanBuilder, Sym, fold_bn

# (kernel, expansion, out, SE, stride)   ghost_net.py:176-193
CFGS = [(3, 16, 16, 0, 2), (3, 48, 24, 0, 2), (3, 72, 24, 0, 1), (5, 72, 40, 1, 1), (5, 120, 40, 1, 1),
        (3, 240, 80, 0, 1), (3, 200, 80, 0, 1), (3, 184, 80, 0, 1), (3, 184, 80, 0, 1), (3, 480, 112, 1, 1),
        (3, 672, 112, 1, 1), (5, 672, 160, 1, 1), (5, 960, 160, 0, 1), (5, 960, 160, 1, 1), (5, 960, 160, 0, 1),
        (5, 960, 160, 1, 1)]
OUT_HW = (128, 128)                            # ghost_net.py:155

Slab = Tuple[Sym, int]                         # (zero-padded activation, real channels)


def make_divisible(v: float, divisor: int = 4) -> int:
    new_v = max(divisor, int(v + divisor / 2) // divisor * divisor)
    if new_v < 0.9 * v:
        new_v += divisor
    return new_v


STEM_C = make_divisible(16)


def blocks():
    """-> [(features index, kernel, in, hidden, out, SE, stride)] (width 1.0, ghost_net.py:124-129)"""
    out, c_in = [], STEM_C
    for i, (k, exp, c, se, s) in enumerate(CFGS, 1):
        oup = make_divisible(c)
        out.append((i, k, c_in, make_divisible(exp), oup, bool(se), s))
        c_in = oup
    return out


FEAT_C = blocks()[-1][4]


def feature_channels(cfg=None) -> int:
    return FEAT_C


def _dw(c, k, stride):
    return nn.Conv2d(c, c, k, stride, k // 2, groups=c, bias=False)


def _ghost_params(root, p, inp, oup):
    init = math.ceil(oup / 2)
    attach(root, p + ".primary_conv.0", conv(inp, init, 1)); attach(root, p + ".primary_conv.1", bn(init))
    attach(root, p + ".cheap_operation.0", _dw(init, 3, 1)); attach(root, p + ".cheap_operation.1", bn(init))


def build_params(cfg=None) -> nn.Module:
    root = nn.Module()
    attach(root, "features.0.0", conv(3, STEM_C, 3, 2, 1)); attach(root, "features.0.1", bn(STEM_C))
    for i, k, inp, hid, oup, se, s in blocks():
        p = f"features.{i}"
        _ghost_params(root, p + ".conv.0", inp, hid)
        if s == 2:
            attach(root, p + ".conv.1.0", _dw(hid, k, s)); attach(root, p + ".conv.1.1", bn(hid))
        if se:
            attach(root, p + ".conv.2.fc.0", nn.Linear(hid, hid // 4)); attach(root, p + ".conv.2.fc.2", nn.Linear(hid // 4, hid))
        _ghost_params(root, p + ".conv.3", hid, oup)
        if not (s == 1 and inp == oup):
            attach(root, p + ".shortcut.0.0", _dw(inp, 3, s)); attach(root, p + ".shortcut.0.1", bn(inp))
            attach(root, p + ".shortcut.1", conv(inp, oup, 1)); attach(root, p + ".shortcut.2", bn(oup))
    with torch.no_grad():                                         # GhostNet._initialize_weights (ghost_net.py:165-171)
        for m in root.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")
    return root


# ------------------------------------------------------------------------------------------ lowering
def _pad16(c: int) -> int:
    return (c + 15) // 16 * 16


def _rows(t: torch.Tensor, n: int) -> torch.Tensor:
    """zero-pad dim 0 of a weight / bias to n rows"""
    if t.shape[0] == n:
        return t
    out = torch.zeros(n, *t.shape[1:], dtype=t.dtype, device=t.device)
    out[:t.shape[0]] = t
    return out


def ghost_module(pb: PlanBuilder, P: StateView, p: str, x: List[Slab], oup: int, relu: bool) -> List[Slab]:
    """GhostModule.forward (ghost_net.py:74-78) -> [(primary, init), (cheap, new)]"""
    act = "relu" if relu else None
    w, b = fold_bn(P(p + ".primary_conv.0.weight"), None, P.bn(p + ".primary_conv.1"))
    init = w.shape[0]
    wc, bc = fold_bn(P(p + ".cheap_operation.0.weight"), None, P.bn(p + ".cheap_operation.1"))    # (new, 1, 3, 3)
    new = wc.shape[0]
    assert new == init and init + new == oup, (init, new, oup)     # ratio 2, and out[:, :oup] keeps every channel
    cp = _pad16(init)
    x1 = pb.conv([s for s, _ in x], _rows(scatter_columns(w, x), cp), _rows(b, cp), stride=1, pad=0, act=act)
    x2 = pb.dwconv(x1, _rows(wc, cp), _rows(bc, cp), stride=1, act=act)
    return [(x1, init), (x2, new)]


def dw_slabs(pb: PlanBuilder, P: StateView, p: str, x: List[Slab], stride: int, act=None) -> List[Slab]:
    """depthwise_conv (ghost_net.py:48-53) over a slab list: one depthwise op per slab"""
    w, b = fold_bn(P(p + ".0.weight"), None, P.bn(p + ".1"))
    out, off = [], 0
    for s, r in x:
        out.append((pb.dwconv(s, _rows(w[off:off + r], s.C), _rows(b[off:off + r], s.C), stride=stride, act=act), r))
        off += r
    return out


def se_layer(pb: PlanBuilder, P: StateView, p: str, x: List[Slab]) -> List[Slab]:
    """SELayer.forward (ghost_net.py:39-45)"""
    pooled = [(pb.avgpool(s), r) for s, r in x]
    w1, b1 = P(p + ".fc.0.weight").float(), P(p + ".fc.0.bias").float()           # Linear (C/4, C)
    mid = w1.shape[0]
    mp = _pad16(mid)
    g = pb.conv([s for s, _ in pooled], _rows(scatter_columns(w1[:, :, None, None], pooled), mp), _rows(b1, mp),
                stride=1, pad=0, act="relu")
    w2, b2 = P(p + ".fc.2.weight").float(), P(p + ".fc.2.bias").float()            # Linear (C, C/4)
    out, off = [], 0
    for s, r in x:
        wg = torch.zeros(s.C, mp, 1, 1, dtype=torch.float32, device=w2.device)
        wg[:r, :mid, 0, 0] = w2[off:off + r]
        gate = pb.conv([g], wg, _rows(b2[off:off + r], s.C), stride=1, pad=0, act="clip01")
        out.append((pb.scale_add(s, gate), r))
        off += r
    return out


def bottleneck(pb: PlanBuilder, P: StateView, p: str, x: List[Slab], k: int, inp: int, hid: int, oup: int, se: bool,
               s: int) -> List[Slab]:
    """GhostBottleneck.forward (ghost_net.py:109-110)"""
    h = ghost_module(pb, P, p + ".conv.0", x, hid, relu=True)
    if s == 2:
        h = dw_slabs(pb, P, p + ".conv.1", h, s)
    if se:
        h = se_layer(pb, P, p + ".conv.2", h)
    y = ghost_module(pb, P, p + ".conv.3", h, oup, relu=False)
    if s == 1 and inp == oup:
        return [(pb.upsample_add(a, c, 1), r) for (a, r), (c, _) in zip(y, x)]          # a plain add (factor 1)
    sc = dw_slabs(pb, P, p + ".shortcut.0", x, s, act="relu")
    w, b = fold_bn(P(p + ".shortcut.1.weight"), None, P.bn(p + ".shortcut.2"))
    w = scatter_columns(w, sc)
    out, off = [], 0
    for a, r in y:
        out.append((pb.conv([t for t, _ in sc], _rows(w[off:off + r], a.C), _rows(b[off:off + r], a.C), stride=1, pad=0,
                            res=a), r))
        off += r
    return out


def lower(pb: PlanBuilder, P: StateView, x: Sym) -> List[Slab]:
    """GhostNet.forward (ghost_net.py:153-158) -> the last bottleneck's two 80-channel slabs, resized to 128 x 128."""
    w, b = fold_bn(P("features.0.0.weight"), None, P.bn("features.0.1"))
    cur: List[Slab] = [(pb.stem(x, w, b, 3, 2, 1, relu=True), STEM_C)]
    for i, k, inp, hid, oup, se, s in blocks():
        cur = bottleneck(pb, P, f"features.{i}", cur, k, inp, hid, oup, se, s)
    return [(pb.resize_bilinear(t, *OUT_HW), r) for t, r in cur]
