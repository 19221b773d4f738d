"""HarDNet (the reference's ``'hardnet'`` arch, ``lib/models/backbones/hardnet.py``): parameter tree + lowering to
fused ops.  Stride-4 output with 48 channels (``experiments/hardnet_512x512.yaml``: INTERMEDIATE_CHANNEL 48).

Network.  A stem of four ConvLayers (conv k x k, pad k//2, no bias -> BN -> ReLU; 3->16 stride 2, 16->24, 24->32
stride 2, 32->48), five stages of [harmonic dense block -> 1x1 ConvLayer (-> 2x2 average pool, first four stages)],
then four up stages of [bilinear resize (align_corners) to the skip's size -> concat with the skip -> 1x1 ConvLayer
halving the channels -> harmonic dense block].  The skips are the outputs of the first four down blocks.

Harmonic dense block with growth rate g and n layers: layer l (1-based) reads the channel concatenation of the earlier
outputs l - 2^i for every 2^i dividing l, nearest first (output 0 is the block input), and produces g * 1.7^t channels
rounded to an even count, t = the number of those links beyond the first.  The block's output is the concatenation of
the odd layers and the last one.

Lowering.
  * Padded slabs.  Every conv's output channels are zero-padded to the next multiple of 16 (10 -> 16, 18 -> 32, 28 -> 32,
    46 -> 48 ...): the folded weights and bias rows of the padding are zero, so the padded channels are exactly 0 after
    the ReLU (as in archs/mobilenet.py).  Stopping at the NEXT multiple of 16 keeps every K = 16 MMA step carrying real
    data, which the round-toward-zero compensation (plan.rz_compensation, linear in K steps) assumes.
  * A concatenation is never materialised: it is a list of slabs ``(Sym, real channels)``, each one conv input; the
    consumer's weight columns are scattered into the padded layout (:func:`archs.common.scatter_columns`).
  * A conv op reads at most four inputs.  A longer slab list (the 1x1 conv after an 8-layer block: 5 slabs; the up
    path's 1x1 convs: 6, 10, 8, 6) is split, in concatenation order, into chunks of <= 4 slabs, one conv each; every
    chunk after the first adds the previous chunk's result as its residual, and only the last one carries the folded
    bias and the ReLU.  The epilogue order is +bias, +residual, activation, so this is the same function.
"""
from __future__ import annotations

from typing import List, Tuple

import torch
from torch import nn

from .common import StateView, attach, bn, conv, scatter_columns
from ..plan import PlanBuilder, Sym, fold_bn

STEM_CH = [16, 24, 32, 48]                   # base.0 .. base.3 (base.0 and base.2 stride 2)
STAGE_CH = [64, 96, 160, 224, 320]           # 1x1 ConvLayer after each down block
GROWTH = [10, 16, 18, 24, 32]
N_LAYERS = [4, 4, 8, 8, 8]
GRMUL = 1.7
FEAT_C = 48

Slab = Tuple[Sym, int]                       # (zero-padded activation, real channels)


def links(l: int) -> List[int]:
    """Earlier outputs layer l (1-based) reads, in concatenation order: l - 1, l - 2, l - 4, ... while 2^i divides l."""
    out, d = [], 1
    while l % d == 0:
        out.append(l - d)
        d *= 2
    return out


def layer_width(l: int, growth: int) -> int:
    w = float(growth)
    for _ in links(l)[1:]:
        w *= GRMUL
    return 2 * (int(w + 1.0) // 2)


def block_widths(c_in: int, growth: int, n: int) -> List[int]:
    """channels of outputs 0..n of a block (output 0 = its input)."""
    return [c_in] + [layer_width(l, growth) for l in range(1, n + 1)]


def block_outputs(n: int) -> List[int]:
    """outputs that make up the block's result, in order: the odd layers and the last."""
    return [l for l in range(1, n + 1) if l % 2 == 1 or l == n]


def feature_channels(cfg=None) -> int:
    return FEAT_C


def _conv_layer(root, key, ci, co, k=3, stride=1):
    attach(root, key + ".conv", conv(ci, co, k, stride, k // 2))
    attach(root, key + ".norm", bn(co))


def _block_params(root, key, c_in, growth, n) -> int:
    w = block_widths(c_in, growth, n)
    for l in range(1, n + 1):
        _conv_layer(root, f"{key}.layers.{l - 1}", sum(w[j] for j in links(l)), w[l])
    return sum(w[j] for j in block_outputs(n))


def build_params(cfg=None) -> nn.Module:
    root = nn.Module()
    ci = 3
    for i, (co, stride) in enumerate(zip(STEM_CH, (2, 1, 2, 1))):
        _conv_layer(root, f"base.{i}", ci, co, 3, stride)
        ci = co
    skips, idx = [], 4
    for s in range(len(GROWTH)):
        c_blk = _block_params(root, f"base.{idx}", ci, GROWTH[s], N_LAYERS[s])
        _conv_layer(root, f"base.{idx + 1}", c_blk, STAGE_CH[s], 1)
        ci = STAGE_CH[s]
        if s < len(GROWTH) - 1:
            skips.append(c_blk)
            idx += 3                                         # block, 1x1 ConvLayer, AvgPool2d
    # up path; the reference registers every denseBlocksUp before any conv1x1_up, so the state_dict keeps that order
    ups = []
    for i, s in enumerate(range(len(skips) - 1, -1, -1)):
        c_cat = ci + skips[s]
        ups.append((c_cat, c_cat // 2))
        ci = sum(block_widths(c_cat // 2, GROWTH[s], N_LAYERS[s])[j] for j in block_outputs(N_LAYERS[s]))
    for i, s in enumerate(range(len(skips) - 1, -1, -1)):
        _block_params(root, f"denseBlocksUp.{i}", ups[i][1], GROWTH[s], N_LAYERS[s])
    for i, (c_cat, c_half) in enumerate(ups):
        _conv_layer(root, f"conv1x1_up.{i}", c_cat, c_half, 1)
    assert ci == FEAT_C, ci
    return root


# ------------------------------------------------------------------------------------------ lowering
def _pad16(c: int) -> int:
    return (c + 15) // 16 * 16


def conv_layer(pb: PlanBuilder, P: StateView, key: str, slabs: List[Slab], stride: int = 1) -> Slab:
    """ConvLayer over a slab list -> one zero-padded slab.  More than four slabs: chained chunk convs (module doc)."""
    w, b = fold_bn(P(key + ".conv.weight"), None, P.bn(key + ".norm"))
    co, _, k, _ = w.shape
    cop = _pad16(co)
    wp = torch.zeros(cop, sum(s.C for s, _ in slabs), k, k, dtype=torch.float32, device=w.device)
    wp[:co] = scatter_columns(w, slabs)
    bp = torch.zeros(cop, dtype=torch.float32, device=b.device)
    bp[:co] = b
    srcs = [s for s, _ in slabs]
    y, off = None, 0
    for j in range(0, len(srcs), 4):
        chunk = srcs[j:j + 4]
        c = sum(s.C for s in chunk)
        last = j + 4 >= len(srcs)
        y = pb.conv(chunk, wp[:, off:off + c], bp if last else torch.zeros_like(bp), stride=stride, pad=k // 2,
                    relu=last, res=y)
        off += c
    return y, co


def hard_block(pb: PlanBuilder, P: StateView, key: str, x: List[Slab], n: int) -> List[Slab]:
    outs = [x]
    for l in range(1, n + 1):
        outs.append([conv_layer(pb, P, f"{key}.layers.{l - 1}", [s for j in links(l) for s in outs[j]])])
    return [s for j in block_outputs(n) for s in outs[j]]


def lower(pb: PlanBuilder, P: StateView, x: Sym) -> List[Slab]:
    """hardnet.forward (hardnet.py:170-188) -> the last up block's slabs: layers 1, 3 and 4, 10 + 10 + 28 real channels
    in 16 + 16 + 32, stride 4."""
    w, b = fold_bn(P("base.0.conv.weight"), None, P.bn("base.0.norm"))
    cur: List[Slab] = [(pb.stem(x, w, b, 3, 2, 1, relu=True), STEM_CH[0])]
    cur = [conv_layer(pb, P, "base.1", cur)]
    cur = [conv_layer(pb, P, "base.2", cur, stride=2)]
    cur = [conv_layer(pb, P, "base.3", cur)]
    skips, idx = [], 4
    for s in range(len(GROWTH)):
        blk = hard_block(pb, P, f"base.{idx}", cur, N_LAYERS[s])
        cur = [conv_layer(pb, P, f"base.{idx + 1}", blk)]
        if s < len(GROWTH) - 1:
            skips.append(blk)
            cur = [(pb.avgpool2(cur[0][0]), cur[0][1])]
            idx += 3
    for i in range(len(skips)):                                     # TransitionUp -> conv1x1_up -> denseBlocksUp
        skip = skips.pop()
        H, W = skip[0][0].H, skip[0][0].W
        up = [(pb.resize_bilinear(s, H, W), r) for s, r in cur]
        cur = [conv_layer(pb, P, f"conv1x1_up.{i}", up + skip)]
        cur = hard_block(pb, P, f"denseBlocksUp.{i}", cur, N_LAYERS[len(skips)])
    return cur
