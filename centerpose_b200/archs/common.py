"""Helpers shared by the backbone descriptions."""
from __future__ import annotations

import math

import torch
from torch import nn


def attach(root: nn.Module, path: str, leaf: nn.Module) -> nn.Module:
    """Register ``leaf`` under dotted ``path`` below ``root``, creating plain container modules
    on the way, so that ``root.state_dict()`` carries exactly the reference's key names."""
    parts = path.split(".")
    cur = root
    for p in parts[:-1]:
        nxt = cur._modules.get(p)
        if nxt is None:
            nxt = nn.Module()
            cur.add_module(p, nxt)
        cur = nxt
    cur.add_module(parts[-1], leaf)
    return leaf


def conv(ci, co, k, stride=1, pad=0, bias=False):
    return nn.Conv2d(ci, co, k, stride=stride, padding=pad, bias=bias)


def bn(c):
    return nn.BatchNorm2d(c, momentum=0.1)


class DCNParams(nn.Module):
    """Parameter holder with the reference ``DCN`` module's names and default init
    (``DCNv2/dcn_v2.py:57-115``): ``weight`` (Co,Ci,3,3) ~ U(+-1/sqrt(Ci*9)), ``bias`` 0,
    ``conv_offset_mask`` = Conv2d(Ci, 27, 3, pad 1) zero-initialised."""

    def __init__(self, ci, co):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(co, ci, 3, 3))
        self.bias = nn.Parameter(torch.zeros(co))
        self.conv_offset_mask = nn.Conv2d(ci, 27, 3, stride=1, padding=1, bias=True)
        stdv = 1.0 / math.sqrt(ci * 9)
        with torch.no_grad():
            self.weight.uniform_(-stdv, stdv)
            self.conv_offset_mask.weight.zero_()
            self.conv_offset_mask.bias.zero_()


def bilinear_up(c, f):
    """Depthwise ConvTranspose2d(c, c, 2f, stride f, pad f//2, groups c) initialised to bilinear
    interpolation (``pose_dla_dcn.py:324-333,361-364``); an ordinary parameter afterwards."""
    k = 2 * f
    m = nn.ConvTranspose2d(c, c, k, stride=f, padding=f // 2, output_padding=0, groups=c, bias=False)
    ff = math.ceil(k / 2)
    cc = (2 * ff - 1 - ff % 2) / (2.0 * ff)
    with torch.no_grad():
        for i in range(k):
            for j in range(k):
                m.weight[:, 0, i, j] = (1 - abs(i / ff - cc)) * (1 - abs(j / ff - cc))
    return m


def scatter_columns(w: torch.Tensor, slabs) -> torch.Tensor:
    """Input columns of a conv weight (Co, sum(real), kh, kw) laid out over a channel concatenation that is never
    materialised: ``slabs`` is a list of ``(Sym, real)`` pairs, each a zero-padded activation (``Sym.C`` channels, the
    first ``real`` of them live).  Returns (Co, sum(Sym.C), kh, kw) with every slab's columns at its padded offset and
    zeros in the gaps."""
    co, ci, kh, kw = w.shape
    assert ci == sum(r for _, r in slabs), (ci, [(s.C, r) for s, r in slabs])
    if all(s.C == r for s, r in slabs):
        return w
    out = torch.zeros(co, sum(s.C for s, _ in slabs), kh, kw, dtype=w.dtype, device=w.device)
    src = dst = 0
    for s, r in slabs:
        out[:, dst:dst + r] = w[:, src:src + r]
        src += r
        dst += s.C
    return out


class StateView:
    """Read access to a (prefix-stripped) state_dict on the target device."""

    def __init__(self, sd, prefix, device):
        self.sd, self.prefix, self.device = sd, prefix, device

    def __call__(self, key):
        return self.sd[self.prefix + key].detach().to(self.device)

    def has(self, key):
        return (self.prefix + key) in self.sd

    def bn(self, key):
        return {k: self(f"{key}.{k}") for k in ("weight", "bias", "running_mean", "running_var")}
