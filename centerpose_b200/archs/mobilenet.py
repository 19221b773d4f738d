"""MobileNetV3-Large + DCN IDAUp (the reference's ``'mobilenetv3'`` arch,
``lib/models/backbones/mobilenet/mobilenetv3.py:159-233``): parameter tree + lowering to fused ops.

Channel padding.  The reference's channel counts (24, 40, 72, 120, 184, 200 ...) are not multiples of 16,
the K / N granularity of the wgmma kernels, and a DCN's gathered operand tile is 64 channels wide.  The
lowering therefore carries every activation with ZERO-PADDED channels (:func:`padded`: next multiple of 16;
24 / 40 / 160 -> 64 / 64 / 192 because those tensors feed the IDAUp DCNs) and zero-pads the folded weights
and biases to match.  Padded channels stay exactly zero through ReLU, h-swish, the SE gate (x * s) and the
shortcut adds, so the real channels are unchanged.

Per Block (``:114-147``): 1x1 expand (+BN+act, tensor cores) -> depthwise k x k (+BN+act, one HBM-bound
kernel) -> 1x1 project (+BN [+ shortcut when there is no SE]) -> [SE: global-avg-pool, two tiny 1x1 convs
(ReLU / h-sigmoid), then ONE pass that applies the gate and adds the shortcut].
"""
from __future__ import annotations

import torch
from torch import nn

from .common import DCNParams, StateView, attach, bilinear_up, bn, conv
from ..plan import PlanBuilder, Sym, fold_bn

# (group, kernel, in, expand, out, nonlinearity, SE, stride)   mobilenetv3.py:168-195
BLOCKS = [
    ("bneck0", 3, 16, 16, 16, "relu", False, 1), ("bneck0", 3, 16, 64, 24, "relu", False, 2),
    ("bneck0", 3, 24, 72, 24, "relu", False, 1),
    ("bneck1", 5, 24, 72, 40, "relu", True, 2), ("bneck1", 5, 40, 120, 40, "relu", True, 1),
    ("bneck1", 5, 40, 120, 40, "relu", True, 1),
    ("bneck2", 3, 40, 240, 80, "hswish", False, 2), ("bneck2", 3, 80, 200, 80, "hswish", False, 1),
    ("bneck2", 3, 80, 184, 80, "hswish", False, 1), ("bneck2", 3, 80, 184, 80, "hswish", False, 1),
    ("bneck2", 3, 80, 480, 112, "hswish", True, 1), ("bneck2", 3, 112, 672, 112, "hswish", True, 1),
    ("bneck2", 5, 112, 672, 160, "hswish", True, 1),
    ("bneck3", 5, 160, 672, 160, "hswish", True, 2), ("bneck3", 5, 160, 960, 160, "hswish", True, 1),
]
IDA_O = 24                                   # IDAUp(24, [24, 40, 160, 960], [1, 2, 4, 8])  (:199-200)
IDA_CH = [24, 40, 160, 960]
FEAT_PAD = 32                                # channels of the tensor handed to the heads (24 real)


def padded(c: int) -> int:
    return {24: 64, 40: 64, 160: 192}.get(c, (c + 15) // 16 * 16)


def feature_channels(cfg=None) -> int:
    return IDA_O


def build_params(cfg=None) -> nn.Module:
    root = nn.Module()
    attach(root, "conv1", conv(3, 16, 3, 2, 1)); attach(root, "bn1", bn_plain(16))
    idx = {}
    for group, k, cin, exp, cout, _nl, se, stride in BLOCKS:
        i = idx.get(group, 0); idx[group] = i + 1
        p = f"{group}.{i}"
        if se:                                                    # SeModule(out) (:96-109); registered first, as in Block.__init__
            attach(root, p + ".se.se.1", conv(cout, cout // 4, 1)); attach(root, p + ".se.se.2", bn_plain(cout // 4))
            attach(root, p + ".se.se.4", conv(cout // 4, cout, 1)); attach(root, p + ".se.se.5", bn_plain(cout))
        attach(root, p + ".conv1", conv(cin, exp, 1)); attach(root, p + ".bn1", bn_plain(exp))
        attach(root, p + ".conv2", nn.Conv2d(exp, exp, k, stride=stride, padding=k // 2, groups=exp, bias=False))
        attach(root, p + ".bn2", bn_plain(exp))
        attach(root, p + ".conv3", conv(exp, cout, 1)); attach(root, p + ".bn3", bn_plain(cout))
        if stride == 1 and cin != cout:
            attach(root, p + ".shortcut.0", conv(cin, cout, 1)); attach(root, p + ".shortcut.1", bn_plain(cout))
    attach(root, "conv2", conv(160, 960, 1)); attach(root, "bn2", bn_plain(960))
    for i in range(1, len(IDA_CH)):                               # IDAUp.__init__ (:47-60): proj, node, up registration order
        f = 2 ** i
        attach(root, f"ida_up.proj_{i}.actf.0", bn(IDA_O))
        attach(root, f"ida_up.proj_{i}.conv", DCNParams(IDA_CH[i], IDA_O))
        attach(root, f"ida_up.up_{i}", bilinear_up(IDA_O, f))
        attach(root, f"ida_up.node_{i}.actf.0", bn(IDA_O))
        attach(root, f"ida_up.node_{i}.conv", DCNParams(IDA_O, IDA_O))
    with torch.no_grad():                                         # init_params (:203-215)
        for m in root.modules():
            if isinstance(m, nn.Conv2d):                          # includes the DCNs' conv_offset_mask, as in the reference
                nn.init.kaiming_normal_(m.weight, mode="fan_out")
                if m.bias is not None:
                    nn.init.constant_(m.bias, 0)
    return root


def bn_plain(c):
    return nn.BatchNorm2d(c)                                      # default momentum (mobilenetv3.py uses nn.BatchNorm2d(c))


# ------------------------------------------------------------------------------------------ lowering
def _pw(w: torch.Tensor, co_p: int, ci_p: int) -> torch.Tensor:
    co, ci, kh, kw = w.shape
    if co == co_p and ci == ci_p:
        return w
    out = torch.zeros(co_p, ci_p, kh, kw, dtype=w.dtype, device=w.device)
    out[:co, :ci] = w
    return out


def _pv(b: torch.Tensor, n: int) -> torch.Tensor:
    if b.shape[0] == n:
        return b
    out = torch.zeros(n, dtype=b.dtype, device=b.device)
    out[:b.shape[0]] = b
    return out


def _pconv(pb, P, x, ckey, bkey, co_p, act=None, res=None):
    """1x1 conv + folded BN on zero-padded channels."""
    w, b = fold_bn(P(ckey + ".weight"), None, P.bn(bkey))
    return pb.conv([x], _pw(w, co_p, x.C), _pv(b, co_p), stride=1, pad=0, act=act, res=res)


def _block(pb: PlanBuilder, P: StateView, x: Sym, p: str, k: int, exp: int, cout: int, nl: str, stride: int) -> Sym:
    exp_p, out_p = padded(exp), padded(cout)
    t = _pconv(pb, P, x, p + ".conv1", p + ".bn1", exp_p, act=nl)
    w2, b2 = fold_bn(P(p + ".conv2.weight"), None, P.bn(p + ".bn2"))             # (exp, 1, k, k)
    w2p = torch.zeros(exp_p, 1, k, k, dtype=w2.dtype, device=w2.device); w2p[:exp] = w2
    t = pb.dwconv(t, w2p, _pv(b2, exp_p), stride=stride, act=nl)
    sc = None
    if stride == 1:
        sc = _pconv(pb, P, x, p + ".shortcut.0", p + ".shortcut.1", out_p) if P.has(p + ".shortcut.0.weight") else x
        assert sc.C == out_p
    if not P.has(p + ".se.se.1.weight"):
        return _pconv(pb, P, t, p + ".conv3", p + ".bn3", out_p, res=sc)
    u = _pconv(pb, P, t, p + ".conv3", p + ".bn3", out_p)
    g = pb.avgpool(u)
    g = _pconv(pb, P, g, p + ".se.se.1", p + ".se.se.2", padded(cout // 4), act="relu")
    g = _pconv(pb, P, g, p + ".se.se.4", p + ".se.se.5", out_p, act="hsigmoid")
    return pb.scale_add(u, g, sc)


def _deform(pb, P, x, p, co_p):
    """DeformConv (mobilenetv3.py:34-45): DCN + BN + ReLU with BN folded, on padded channels."""
    w, b = fold_bn(P(p + ".conv.weight"), P(p + ".conv.bias"), P.bn(p + ".actf.0"))
    om_w = P(p + ".conv.conv_offset_mask.weight").float()
    return pb.dcn(x, _pw(w, co_p, x.C), _pv(b, co_p), _pw(om_w, om_w.shape[0], x.C), P(p + ".conv.conv_offset_mask.bias"))


def lower(pb: PlanBuilder, P: StateView, x: Sym) -> Sym:
    """MobileNetV3.forward (mobilenetv3.py:217-233) -> IDAUp output (24 real channels in 32, stride 4)."""
    w, b = fold_bn(P("conv1.weight"), None, P.bn("bn1"))
    t = pb.stem(x, w, b, 3, 2, 1, act="hswish")
    feats = {}
    idx = {}
    for group, k, _cin, exp, cout, nl, _se, stride in BLOCKS:
        i = idx.get(group, 0); idx[group] = i + 1
        t = _block(pb, P, t, f"{group}.{i}", k, exp, cout, nl, stride)
        feats[group] = t
    out3 = _pconv(pb, P, feats["bneck3"], "conv2", "bn2", 960, act="hswish")
    layers = [feats["bneck0"], feats["bneck1"], feats["bneck2"], out3]
    o_p = padded(IDA_O)
    for i in range(1, len(layers)):                               # IDAUp.forward (:62-69)
        y = _deform(pb, P, layers[i], f"ida_up.proj_{i}", o_p)
        wu = P(f"ida_up.up_{i}.weight").float()                   # (24, 1, 2f, 2f)
        wup = torch.zeros(o_p, 1, wu.shape[2], wu.shape[3], dtype=wu.dtype, device=wu.device); wup[:wu.shape[0]] = wu
        y = pb.up_add(y, layers[i - 1], wup)
        layers[i] = _deform(pb, P, y, f"ida_up.node_{i}", o_p if i < len(layers) - 1 else FEAT_PAD)
    return layers[-1]
