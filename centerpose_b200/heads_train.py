"""The keypoint heads with their backward on the device: a drop-in for the reference's ``KeypointHead``
(lib/models/heads/keypoint.py) that trains without storing the heads' hidden maps.

    from centerpose_b200 import dcn, heads_train
    dcn.install_ext()
    from models import model
    model._head_factory["keypoint"] = heads_train.KeypointHead     # before create_model
    model = create_model("dla_34", head_conv, cfg)                  # its heads now run csrc/heads_train.cu

Each head is Conv2d(C, hc, 3) -> ReLU -> Conv2d(hc, c_h, 1).  Torch's autograd keeps every head's hc x H x W hidden
map until the backward (96 MiB per 128x128 image at hc = 256); here the forward keeps each tile in shared memory and
the backward recomputes it, so a training step saves only x and the weights.  The module keeps the reference's six
``nn.Sequential`` children as parameter holders: state_dict keys, ``named_parameters()`` order, init and ``.to()``
are the reference's; only ``forward`` changes.

Two precisions, both on every shape, as in ``centerpose_b200.dcn``:
  * ``"default"``: tensor cores (mma.sync tf32), each fp32 operand split into two tf32 parts, fp32 accumulation.
  * ``"fp32"``: CUDA-core fp32.
Every output and gradient is the same bits on every run.  CPU tensors raise ``RuntimeError``, tensors other than
float32 ``ValueError``, an input whose channels are not the heads' ``RuntimeError``.
"""
from __future__ import annotations

import torch
from torch import nn
from torch.autograd.function import once_differentiable

from .dcn import _check_tensors, _precision_code

HEADS = ("hm", "wh", "hps", "reg", "hm_hp", "hp_offset")
OUTPUTS = (1, 2, 34, 2, 17, 2)


def _check_input(what, x, w0):
    if x.dim() != 4:
        raise ValueError("%s: x must be 4-D (B, C, H, W), got %s" % (what, tuple(x.shape)))
    if x.shape[1] != w0.shape[1]:
        raise RuntimeError("%s: x has %d channels, the heads take %d" % (what, x.shape[1], w0.shape[1]))
    return tuple(int(v) for v in x.shape)


def _concat(params):
    """W0 (6*hc, C, 3, 3), b0, W2 (58, hc), b2 from the 24 parameters in named_parameters() order.  A per-call copy of
    a few MB (3.5 MB for DLA-34's heads), freed when the call returns."""
    w0 = torch.cat([params[4 * h] for h in range(6)])
    b0 = torch.cat([params[4 * h + 1] for h in range(6)])
    w2 = torch.cat([params[4 * h + 2].reshape(params[4 * h + 2].shape[0], -1) for h in range(6)])
    b2 = torch.cat([params[4 * h + 3] for h in range(6)])
    return [t.contiguous() for t in (w0, b0, w2, b2)]


def heads_forward(x, params, precision="default"):
    """The six maps [hm, wh, hps, reg, hm_hp, hp_offset] of ``x`` for the 24 head parameters (no autograd)."""
    from . import _lib
    code = _precision_code(precision)
    _check_tensors("heads_train_forward", [("x", x)] + [("head parameter %d" % i, p) for i, p in enumerate(params)])
    B, C, H, W = _check_input("heads_train_forward", x, params[0])
    w0, b0, w2, b2 = _concat(params)
    hc = w0.shape[0] // 6
    outs = [torch.empty((B, c, H, W), dtype=torch.float32, device=x.device) for c in OUTPUTS]
    _lib.launch("heads_train_forward", x.device, x.contiguous(), w0, b0, w2, b2,
                _lib.Heads(*(o.data_ptr() for o in outs)), B, C, H, W, hc, code)
    return outs


def heads_backward(x, params, grad_outputs, need_x=True, precision="default"):
    """(grad_x or None, [24 parameter gradients]) for ``grad_outputs`` (six maps, None for a head without a gradient,
    whose four parameter gradients are then None)."""
    from . import _lib
    code = _precision_code(precision)
    named = [("x", x)] + [("grad_output %s" % HEADS[h], g) for h, g in enumerate(grad_outputs) if g is not None]
    _check_tensors("heads_train_backward", named + [("head parameter %d" % i, p) for i, p in enumerate(params)])
    B, C, H, W = _check_input("heads_train_backward", x, params[0])
    dev = x.device
    w0, b0, w2, _ = _concat(params)
    hc = w0.shape[0] // 6
    gs = [None if g is None else g.contiguous() for g in grad_outputs]
    for h, g in enumerate(gs):
        if g is not None and tuple(g.shape) != (B, OUTPUTS[h], H, W):
            raise ValueError("heads_train_backward: grad_output %s has shape %s, expected %s"
                             % (HEADS[h], tuple(g.shape), (B, OUTPUTS[h], H, W)))
    gx = torch.empty((B, C, H, W), dtype=torch.float32, device=dev) if need_x else None
    gw0, gb0, gw2 = (torch.empty_like(t) for t in (w0, b0, w2))
    gb2 = torch.empty((sum(OUTPUTS),), dtype=torch.float32, device=dev)
    ws = torch.empty(_lib.lib().cpb200_heads_train_workspace_bytes(B, C, H, W, hc), dtype=torch.uint8, device=dev)
    _lib.launch("heads_train_backward", dev, x.contiguous(), w0, b0, w2,
                _lib.Heads(*(None if g is None else g.data_ptr() for g in gs)), gx, gw0, gb0, gw2, gb2,
                B, C, H, W, hc, code, ws, ws.numel())
    grads, o = [], 0
    for h, c in enumerate(OUTPUTS):
        if gs[h] is None:
            grads += [None] * 4
        else:
            grads += [gw0[h * hc:(h + 1) * hc].view_as(params[4 * h]), gb0[h * hc:(h + 1) * hc],
                      gw2[o:o + c].view_as(params[4 * h + 2]), gb2[o:o + c]]
        o += c
    return gx, grads


class _Heads(torch.autograd.Function):
    """Saves x and the 24 parameters (tensors autograd holds anyway), nothing else."""

    @staticmethod
    def forward(ctx, precision, x, *params):
        ctx.precision = precision
        ctx.set_materialize_grads(False)         # a head whose map gets no gradient keeps None, as in torch
        ctx.save_for_backward(x, *params)
        outs = heads_forward(x, params, precision)
        return tuple(outs)

    @staticmethod
    @once_differentiable
    def backward(ctx, *grad_outputs):
        x, *params = ctx.saved_tensors
        if all(g is None for g in grad_outputs):
            return (None,) * (2 + len(params))
        gx, grads = heads_backward(x, params, grad_outputs, need_x=ctx.needs_input_grad[1],
                                   precision=ctx.precision)
        grads = [g if need else None for g, need in zip(grads, ctx.needs_input_grad[2:])]
        return (None, gx, *grads)


class KeypointHead(nn.Module):
    """The reference's ``KeypointHead(intermediate_channel, head_conv)``, its forward and backward on the device."""

    def __init__(self, intermediate_channel, head_conv, precision="default"):
        super().__init__()
        _precision_code(precision)
        self.precision = precision
        for name, c in zip(HEADS, OUTPUTS):
            setattr(self, name, nn.Sequential(
                nn.Conv2d(intermediate_channel, head_conv, kernel_size=3, padding=1, bias=True),
                nn.ReLU(inplace=True),
                nn.Conv2d(head_conv, c, kernel_size=1, stride=1, padding=0)))
        self.init_weights()

    def init_weights(self):
        """The reference's: -2.19 output biases of hm and hm_hp, N(0, 0.001) weights and 0 biases of the rest."""
        self.hm[-1].bias.data.fill_(-2.19)
        self.hm_hp[-1].bias.data.fill_(-2.19)
        for name in ("wh", "hps", "reg", "hp_offset"):
            self.fill_fc_weights(getattr(self, name))

    def fill_fc_weights(self, layers):
        for m in layers.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.normal_(m.weight, std=0.001)
                if m.bias is not None:
                    nn.init.constant_(m.bias, 0)

    def head_parameters(self):
        """The 24 parameters in HEADS order: each head's 3x3 weight and bias, then its 1x1 weight and bias."""
        return [p for name in HEADS for i in (0, 2) for p in (getattr(self, name)[i].weight,
                                                              getattr(self, name)[i].bias)]

    def forward(self, x):
        params = self.head_parameters()
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in params)):
            return list(_Heads.apply(self.precision, x, *params))
        return heads_forward(x, params, self.precision)
