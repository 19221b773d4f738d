"""ORACLE (test infrastructure, not product): functional torch-CPU fp32 restatement of
the reference's DLA-34 + DCN-IDAUp backbone and the six-head KeypointHead, evaluated
directly from a reference-format ``state_dict`` (eval-mode BatchNorm, eps 1e-5).

Follows (``/root/reference/lib``):
  * ``models/backbones/pose_dla_dcn.py:284-290``  DLA.forward        -> :func:`_dla_base`
  * ``...pose_dla_dcn.py:43-57``                  BasicBlock.forward -> :func:`_block`
  * ``...pose_dla_dcn.py:155-163, 206-219``       Root / Tree.forward-> :func:`_tree`
  * ``...pose_dla_dcn.py:345-348``                DeformConv.forward -> :func:`_deform`
  * ``...pose_dla_dcn.py:371-377``                IDAUp.forward      -> :func:`_ida`
  * ``...pose_dla_dcn.py:398-404``                DLAUp.forward      -> :func:`_dla_up`
  * ``...pose_dla_dcn.py:437-447``                DLASeg.forward     -> :func:`dla34_backbone`
  * ``models/heads/keypoint.py:40-42``            KeypointHead.forward -> :func:`keypoint_head`
  * ``models/model.py:57-59``                     BackBoneWithHead.forward -> :func:`forward`

Pinned by ``oracle/make_golden.py`` against the reference's own modules executed in the
build container (golden head maps in ``tests/golden/``).
Only tests / smoke / bench's CPU-baseline legs import this module.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .dcn_ref import dcn_module_forward

EPS = 1e-5
HEADS = ("hm", "wh", "hps", "reg", "hm_hp", "hp_offset")


def _bn(sd, x, p):
    return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"],
                        sd[p + ".weight"], sd[p + ".bias"], False, 0.0, EPS)


def _conv(sd, x, p, stride=1, pad=0):
    return F.conv2d(x, sd[p + ".weight"], sd.get(p + ".bias"), stride=stride, padding=pad)


def _block(sd, x, p, stride, residual=None):
    if residual is None:
        residual = x
    out = F.relu(_bn(sd, _conv(sd, x, p + ".conv1", stride, 1), p + ".bn1"))
    out = _bn(sd, _conv(sd, out, p + ".conv2", 1, 1), p + ".bn2")
    return F.relu(out + residual)


def _tree(sd, x, p, levels, cin, cout, stride, level_root, children=None):
    children = [] if children is None else children
    bottom = F.max_pool2d(x, stride, stride) if stride > 1 else x
    if level_root:
        children.append(bottom)
    if levels == 1:
        if cin != cout:
            residual = _bn(sd, _conv(sd, bottom, p + ".project.0"), p + ".project.1")
        else:
            residual = bottom
        x1 = _block(sd, x, p + ".tree1", stride, residual)
        x2 = _block(sd, x1, p + ".tree2", 1)
        cat = torch.cat([x2, x1] + children, 1)
        return F.relu(_bn(sd, _conv(sd, cat, p + ".root.conv"), p + ".root.bn"))
    # levels > 1: the reference also evaluates self.project(bottom) here (:209) but the
    # sub-Tree it is passed to overwrites its `residual` argument — dead compute, skipped.
    x1 = _tree(sd, x, p + ".tree1", levels - 1, cin, cout, stride, False)
    children.append(x1)
    return _tree(sd, x1, p + ".tree2", levels - 1, cout, cout, 1, False, children)


def _dla_base(sd, x, p):
    ch = [16, 32, 64, 128, 256, 512]
    lv = [1, 1, 1, 2, 2, 1]
    x = F.relu(_bn(sd, _conv(sd, x, p + ".base_layer.0", 1, 3), p + ".base_layer.1"))
    ys = []
    x = F.relu(_bn(sd, _conv(sd, x, p + ".level0.0", 1, 1), p + ".level0.1")); ys.append(x)
    x = F.relu(_bn(sd, _conv(sd, x, p + ".level1.0", 2, 1), p + ".level1.1")); ys.append(x)
    for i in range(2, 6):
        x = _tree(sd, x, f"{p}.level{i}", lv[i], ch[i - 1], ch[i], 2, level_root=(i > 2))
        ys.append(x)
    return ys


def _deform(sd, x, p):
    y = dcn_module_forward(x, sd[p + ".conv.weight"], sd[p + ".conv.bias"],
                           sd[p + ".conv.conv_offset_mask.weight"],
                           sd[p + ".conv.conv_offset_mask.bias"])
    return F.relu(_bn(sd, y, p + ".actf.0"))


def _ida(sd, layers, p, startp, endp):
    for i in range(startp + 1, endp):
        k = i - startp
        w = sd[f"{p}.up_{k}.weight"]
        f = w.shape[2] // 2
        y = _deform(sd, layers[i], f"{p}.proj_{k}")
        y = F.conv_transpose2d(y, w, None, stride=f, padding=f // 2, groups=w.shape[0])
        layers[i] = _deform(sd, y + layers[i - 1], f"{p}.node_{k}")


def _dla_up(sd, layers, p, startp):
    out = [layers[-1]]
    for i in range(len(layers) - startp - 1):
        _ida(sd, layers, f"{p}.ida_{i}", len(layers) - i - 2, len(layers))
        out.insert(0, layers[-1])
    return out


def dla34_backbone(sd, x, p="backbone_model"):
    layers = _dla_base(sd, x, p + ".base")
    x = _dla_up(sd, list(layers), p + ".dla_up", 2)
    y = [t for t in x[:3]]
    _ida(sd, y, p + ".ida_up", 0, len(y))
    return y[-1]


def keypoint_head(sd, feat, p="head_model"):
    outs = []
    for h in HEADS:
        t = F.relu(_conv(sd, feat, f"{p}.{h}.0", 1, 1))
        outs.append(_conv(sd, t, f"{p}.{h}.2"))
    return outs


@torch.no_grad()
def forward(sd, x, arch="dla_34"):
    """state_dict + (B,3,H,W) -> [hm, wh, hps, reg, hm_hp, hp_offset] logits (NCHW), evaluated in the dtype and on the
    device of ``x`` (fp32 on the CPU pins the reference; float64 on the GPU is the network tests' oracle)."""
    sd = {k: v.to(x.device, x.dtype) for k, v in sd.items() if v.dtype.is_floating_point}
    if arch == "dla_34":
        feat = dla34_backbone(sd, x)
    elif arch == "res_50":
        from .resnet_ref import resnet50_backbone
        feat = resnet50_backbone(sd, x)
    elif arch == "mobilenetv3":
        from .mobilenet_ref import mobilenetv3_backbone
        feat = mobilenetv3_backbone(sd, x)
    elif arch == "hrnet":
        from .hrnet_ref import hrnet_backbone
        feat = hrnet_backbone(sd, x)
    else:
        raise ValueError(arch)
    return keypoint_head(sd, feat)
