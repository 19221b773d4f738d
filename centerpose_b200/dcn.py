"""Modulated deformable convolution (DCNv2) with its backward on the device: a drop-in for the reference's ``_ext``
extension, so the models whose necks are built from ``DCN`` (DLA-34, MobileNetV3, ResNet-DCN) train on current torch.

    from centerpose_b200 import dcn
    dcn.install_ext()                                   # before the reference's model code is imported
    model = create_model("dla_34", heads, head_conv)    # its DCN layers now run csrc/dcn_train.cu

or use the modules directly: ``dcn.DCN(64, 64, kernel_size=3, stride=1, padding=1)`` takes the reference's
arguments and state_dict keys.

``dcn_v2_forward`` / ``dcn_v2_backward`` have the positional signatures and return values of
``DCNv2/src/dcn_v2.h:9-79``.  Only the configuration every reference backbone builds is supported: a 3x3 kernel,
stride 1, padding 1, dilation 1, one deformable group; anything else raises ``NotImplementedError`` naming the
parameter.  CPU tensors raise ``RuntimeError`` (the reference has no CPU path), tensors other than float32 raise
``ValueError``.

Two precisions, both on every shape:
  * ``"default"``: tensor cores (mma.sync tf32), each fp32 operand split into two tf32 parts, fp32 accumulation.
    tf32 has fp32's exponent range, so the result is fp32-faithful for values anywhere in fp32's normal range.
  * ``"fp32"``: CUDA-core fp32.
The output, grad_offset, grad_mask, grad_weight and grad_bias are the same bits on every run; grad_input is
accumulated with fp32 atomics, as in the reference.
"""
from __future__ import annotations

import math
import sys
import types

import torch
from torch import nn
from torch.autograd.function import once_differentiable
from torch.nn.modules.utils import _pair

PRECISIONS = {"default": 0, "fp32": 1}


def _precision_code(precision):
    if precision not in PRECISIONS:
        raise ValueError("dcn: precision must be one of %s, got %r" % (sorted(PRECISIONS), precision))
    return PRECISIONS[precision]


def _check_config(kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w, deformable_group):
    for name, got, want in (("kernel_size", (kernel_h, kernel_w), (3, 3)), ("stride", (stride_h, stride_w), (1, 1)),
                            ("padding", (pad_h, pad_w), (1, 1)), ("dilation", (dilation_h, dilation_w), (1, 1)),
                            ("deformable_groups", (deformable_group,), (1,))):
        if tuple(int(v) for v in got) != want:
            raise NotImplementedError("dcn: %s %s is not supported; only kernel_size 3, stride 1, padding 1, "
                                      "dilation 1 and deformable_groups 1 are" % (name, tuple(got)))


def _check_tensors(what, named):
    for name, t in named:
        if not isinstance(t, torch.Tensor):
            raise ValueError("%s: %s must be a tensor" % (what, name))
    for name, t in named:
        if not t.is_cuda:
            raise RuntimeError("%s: %s must be a CUDA tensor" % (what, name))
    for name, t in named:
        if t.dtype != torch.float32:
            raise ValueError("%s: %s must be float32, got %s" % (what, name, t.dtype))
    dev = named[0][1].device
    for name, t in named:
        if t.device != dev:
            raise RuntimeError("%s: %s is on %s, input on %s" % (what, name, t.device, dev))


def _check_shapes(what, input, weight, bias, offset, mask, kernel_h, kernel_w):
    if input.dim() != 4 or weight.dim() != 4:
        raise ValueError("%s: input and weight must be 4-D, got %s and %s" % (what, tuple(input.shape),
                                                                            tuple(weight.shape)))
    B, C, H, W = input.shape
    Co, Ck, kh, kw = weight.shape
    # dcn_v2_cuda.cu's AT_ASSERTMs
    if kh != kernel_h or kw != kernel_w:
        raise RuntimeError("%s: Input shape and kernel shape wont match: (%d x %d vs %d x %d)."
                           % (what, kernel_h, kernel_w, kh, kw))
    if C != Ck:
        raise RuntimeError("%s: Input shape and kernel channels wont match: (%d vs %d)." % (what, C, Ck))
    for name, t, want in (("bias", bias, (Co,)), ("offset", offset, (B, 2 * kh * kw, H, W)),
                          ("mask", mask, (B, kh * kw, H, W))):
        if tuple(t.shape) != want:
            raise ValueError("%s: %s has shape %s, expected %s" % (what, name, tuple(t.shape), want))
    return B, C, H, W, Co


def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


def dcn_v2_forward(input, weight, bias, offset, mask, kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w,
                   dilation_h, dilation_w, deformable_group, *, precision="default"):
    """``_ext.dcn_v2_forward``: the (B, Co, H, W) output of the modulated deformable conv."""
    from . import _lib
    code = _precision_code(precision)
    _check_tensors("dcn_v2_forward", [("input", input), ("weight", weight), ("bias", bias), ("offset", offset),
                                      ("mask", mask)])
    B, C, H, W, Co = _check_shapes("dcn_v2_forward", input, weight, bias, offset, mask, kernel_h, kernel_w)
    _check_config(kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w, deformable_group)
    dev = input.device
    x, w, b, o, m = (t.contiguous() for t in (input, weight, bias, offset, mask))
    out = torch.empty((B, Co, H, W), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        st = _lib.lib().cpb200_dcn_train_forward(x.data_ptr(), w.data_ptr(), b.data_ptr(), o.data_ptr(),
                                                 m.data_ptr(), out.data_ptr(), B, C, H, W, Co, code, _stream(dev))
    _lib.check(st, "dcn_v2_forward")
    return out


def dcn_v2_backward(input, weight, bias, offset, mask, grad_output, kernel_h, kernel_w, stride_h, stride_w, pad_h,
                    pad_w, dilation_h, dilation_w, deformable_group, *, precision="default"):
    """``_ext.dcn_v2_backward``: ``[grad_input, grad_offset, grad_mask, grad_weight, grad_bias]``."""
    from . import _lib
    code = _precision_code(precision)
    _check_tensors("dcn_v2_backward", [("input", input), ("weight", weight), ("bias", bias), ("offset", offset),
                                       ("mask", mask), ("grad_output", grad_output)])
    B, C, H, W, Co = _check_shapes("dcn_v2_backward", input, weight, bias, offset, mask, kernel_h, kernel_w)
    _check_config(kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w, dilation_h, dilation_w, deformable_group)
    if tuple(grad_output.shape) != (B, Co, H, W):
        raise ValueError("dcn_v2_backward: grad_output has shape %s, expected %s"
                         % (tuple(grad_output.shape), (B, Co, H, W)))
    dev = input.device
    x, w, o, m, g = (t.contiguous() for t in (input, weight, offset, mask, grad_output))
    grads = [torch.empty_like(x), torch.empty_like(o), torch.empty_like(m), torch.empty_like(w),
             torch.empty((Co,), dtype=torch.float32, device=dev)]
    L = _lib.lib()
    ws = torch.empty(L.cpb200_dcn_train_workspace_bytes(B, C, H, W, Co), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        st = L.cpb200_dcn_train_backward(x.data_ptr(), w.data_ptr(), o.data_ptr(), m.data_ptr(), g.data_ptr(),
                                         *[t.data_ptr() for t in grads], B, C, H, W, Co, code, ws.data_ptr(),
                                         ws.numel(), _stream(dev))
    _lib.check(st, "dcn_v2_backward")
    return grads


class _DCNv2(torch.autograd.Function):
    @staticmethod
    def forward(ctx, input, offset, mask, weight, bias, stride, padding, dilation, deformable_groups,
                precision="default"):
        ctx.stride, ctx.padding, ctx.dilation = _pair(stride), _pair(padding), _pair(dilation)
        ctx.kernel_size = _pair(weight.shape[2:4])
        ctx.deformable_groups, ctx.precision = deformable_groups, precision
        out = dcn_v2_forward(input, weight, bias, offset, mask, *ctx.kernel_size, *ctx.stride, *ctx.padding,
                             *ctx.dilation, deformable_groups, precision=precision)
        ctx.save_for_backward(input, offset, mask, weight, bias)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        input, offset, mask, weight, bias = ctx.saved_tensors
        gi, go, gm, gw, gb = dcn_v2_backward(input, weight, bias, offset, mask, grad_output, *ctx.kernel_size,
                                             *ctx.stride, *ctx.padding, *ctx.dilation, ctx.deformable_groups,
                                             precision=ctx.precision)
        return gi, go, gm, gw, gb, None, None, None, None, None


def dcn_v2_conv(input, offset, mask, weight, bias, stride, padding, dilation, deformable_groups,
                precision="default"):
    """``dcn_v2.py``'s ``dcn_v2_conv``, in the reference's argument order; once differentiable."""
    return _DCNv2.apply(input, offset, mask, weight, bias, stride, padding, dilation, deformable_groups, precision)


class DCNv2(nn.Module):
    """The reference's ``DCNv2`` module: parameters ``weight`` (Co, C, kh, kw) and ``bias`` (Co); forward takes the
    offset and mask (probabilities) from the caller."""

    def __init__(self, in_channels, out_channels, kernel_size, stride, padding, dilation=1, deformable_groups=1,
                 precision="default"):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size, self.stride = _pair(kernel_size), _pair(stride)
        self.padding, self.dilation = _pair(padding), _pair(dilation)
        self.deformable_groups = deformable_groups
        self.precision = precision
        self.weight = nn.Parameter(torch.empty(out_channels, in_channels, *self.kernel_size))
        self.bias = nn.Parameter(torch.empty(out_channels))
        self.reset_parameters()

    def reset_parameters(self):
        """weight ~ U(-1/sqrt(fan_in), 1/sqrt(fan_in)) with fan_in = C * kh * kw; bias = 0."""
        stdv = 1.0 / math.sqrt(self.in_channels * self.kernel_size[0] * self.kernel_size[1])
        self.weight.data.uniform_(-stdv, stdv)
        self.bias.data.zero_()

    def forward(self, input, offset, mask):
        taps = self.deformable_groups * self.kernel_size[0] * self.kernel_size[1]
        assert offset.shape[1] == 2 * taps and mask.shape[1] == taps
        return dcn_v2_conv(input, offset, mask, self.weight, self.bias, self.stride, self.padding, self.dilation,
                           self.deformable_groups, self.precision)


class DCN(DCNv2):
    """The reference's ``DCN``: ``DCNv2`` with its own offset / mask conv ``conv_offset_mask`` (3 * groups * kh * kw
    outputs, zero-initialised); the mask is the sigmoid of the last third."""

    def __init__(self, in_channels, out_channels, kernel_size, stride, padding, dilation=1, deformable_groups=1,
                 precision="default"):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, dilation, deformable_groups,
                         precision)
        self.conv_offset_mask = nn.Conv2d(self.in_channels, 3 * self.deformable_groups * self.kernel_size[0] *
                                          self.kernel_size[1], kernel_size=self.kernel_size, stride=self.stride,
                                          padding=self.padding, bias=True)
        self.init_offset()

    def init_offset(self):
        self.conv_offset_mask.weight.data.zero_()
        self.conv_offset_mask.bias.data.zero_()

    def forward(self, input):
        o1, o2, mask = torch.chunk(self.conv_offset_mask(input), 3, dim=1)
        return dcn_v2_conv(input, torch.cat((o1, o2), dim=1), torch.sigmoid(mask), self.weight, self.bias,
                           self.stride, self.padding, self.dilation, self.deformable_groups, self.precision)


def _psroi_unsupported(*args, **kwargs):
    raise NotImplementedError("dcn: DCNv2 position-sensitive RoI pooling is not implemented (no pose model uses it)")


def install_ext(precision="default"):
    """Register ``sys.modules["_ext"]`` with ``dcn_v2_forward`` / ``dcn_v2_backward`` at ``precision`` and the two
    psroi-pooling entry points (which raise ``NotImplementedError``).  Call it before the reference's ``dcn_v2.py``
    is imported: that module binds ``_ext`` once, at import.  Returns the module."""
    _precision_code(precision)          # an unknown precision is refused here, not at the first forward
    ext =types.ModuleType("_ext")
    ext.__doc__ = "centerpose_b200's DCNv2 (csrc/dcn_train.cu) at precision %r" % precision

    def fwd(input, weight, bias, offset, mask, kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w, dilation_h,
            dilation_w, deformable_group):
        return dcn_v2_forward(input, weight, bias, offset, mask, kernel_h, kernel_w, stride_h, stride_w, pad_h,
                              pad_w, dilation_h, dilation_w, deformable_group, precision=precision)

    def bwd(input, weight, bias, offset, mask, grad_output, kernel_h, kernel_w, stride_h, stride_w, pad_h, pad_w,
            dilation_h, dilation_w, deformable_group):
        return dcn_v2_backward(input, weight, bias, offset, mask, grad_output, kernel_h, kernel_w, stride_h,
                               stride_w, pad_h, pad_w, dilation_h, dilation_w, deformable_group, precision=precision)

    ext.dcn_v2_forward = fwd
    ext.dcn_v2_backward = bwd
    ext.dcn_v2_psroi_pooling_forward = _psroi_unsupported
    ext.dcn_v2_psroi_pooling_backward = _psroi_unsupported
    sys.modules["_ext"] = ext
    return ext
