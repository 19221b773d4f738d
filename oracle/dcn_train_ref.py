"""ORACLE (test infrastructure, not product): CPU restatements of the reference's modulated deformable convolution
(DCNv2) backward, ``dcn_v2_cuda_backward`` (``DCNv2/src/cuda/dcn_v2_cuda.cu:206-330``).  The forward is
``oracle/dcn_ref.py``.

The reference's backward cannot be built anywhere (its CUDA sources use the removed THC API, its CPU entry point is
``AT_ERROR``), so these restatements are the reference for its values.  Two forms:

  * :func:`dcn_v2_backward_loops` -- literal float64 loops over ``dcn_v2_im2col_cuda.cu:56-123``
    (``dmcn_get_gradient_weight``, ``dmcn_get_coordinate_weight``), ``:197-254`` (col2im: ``(int)`` truncation, 5x5
    window, ``|delta| < 1``) and ``:256-327`` (col2im_coord), with the three GEMMs of ``dcn_v2_cuda.cu:273-329`` as
    matrix products.  Small cases only.
  * :func:`dcn_v2_backward` -- autograd through the vectorised ``dcn_ref.dcn_v2_forward``, in the tensors' own dtype
    and device (float64 for a reference).

``oracle/make_golden_dcn_train.py`` checks the two against each other and against torchvision's float64
``deform_conv2d`` backward.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import dcn_ref


def _gradient_weight_loops(ah, aw, h, w, H, W):
    """dcn_v2_im2col_cuda.cu:56-80."""
    if ah <= -1 or ah >= H or aw <= -1 or aw >= W:
        return 0.0
    hl = int(np.floor(ah)); wl = int(np.floor(aw))
    hh_ = hl + 1; wh_ = wl + 1
    weight = 0.0
    if h == hl and w == wl:
        weight = (h + 1 - ah) * (w + 1 - aw)
    if h == hl and w == wh_:
        weight = (h + 1 - ah) * (aw + 1 - w)
    if h == hh_ and w == wl:
        weight = (ah + 1 - h) * (w + 1 - aw)
    if h == hh_ and w == wh_:
        weight = (ah + 1 - h) * (aw + 1 - w)
    return weight


def _coordinate_weight_loops(ah, aw, H, W, im, bp_dir):
    """dcn_v2_im2col_cuda.cu:82-123 (im is one (H,W) channel plane)."""
    if ah <= -1 or ah >= H or aw <= -1 or aw >= W:
        return 0.0
    hl = int(np.floor(ah)); wl = int(np.floor(aw))
    hh_ = hl + 1; wh_ = wl + 1
    weight = 0.0
    if bp_dir == 0:
        if hl >= 0 and wl >= 0:
            weight += -1 * (wl + 1 - aw) * im[hl, wl]
        if hl >= 0 and wh_ <= W - 1:
            weight += -1 * (aw - wl) * im[hl, wh_]
        if hh_ <= H - 1 and wl >= 0:
            weight += (wl + 1 - aw) * im[hh_, wl]
        if hh_ <= H - 1 and wh_ <= W - 1:
            weight += (aw - wl) * im[hh_, wh_]
    else:
        if hl >= 0 and wl >= 0:
            weight += -1 * (hl + 1 - ah) * im[hl, wl]
        if hl >= 0 and wh_ <= W - 1:
            weight += (hl + 1 - ah) * im[hl, wh_]
        if hh_ <= H - 1 and wl >= 0:
            weight += -1 * (ah - hl) * im[hh_, wl]
        if hh_ <= H - 1 and wh_ <= W - 1:
            weight += (ah - hl) * im[hh_, wh_]
    return weight


def dcn_v2_backward_loops(inp, weight, bias, offset, mask, grad_out, stride=1, pad=1, dil=1):
    """Literal float64 restatement of dcn_v2_cuda_backward for one deformable group.  Returns
    (grad_input, grad_offset, grad_mask, grad_weight, grad_bias) as numpy arrays."""
    inp, weight, bias, offset, mask, grad_out = (np.asarray(a, np.float64) for a in
                                                 (inp, weight, bias, offset, mask, grad_out))
    B, C, H, W = inp.shape
    Co, _, kh, kw = weight.shape
    Ho = (H + 2 * pad - (dil * (kh - 1) + 1)) // stride + 1
    Wo = (W + 2 * pad - (dil * (kw - 1) + 1)) // stride + 1
    grad_input = np.zeros_like(inp); grad_offset = np.zeros_like(offset); grad_mask = np.zeros_like(mask)
    grad_weight = np.zeros_like(weight); grad_bias = np.zeros_like(bias)
    wmat = weight.reshape(Co, C * kh * kw)
    for b in range(B):
        gout = grad_out[b].reshape(Co, Ho * Wo)
        columns = (wmat.T @ gout).reshape(C * kh * kw, Ho, Wo)          # dcn_v2_cuda.cu:273-276
        # col2im_coord (:256-327): one (offset channel, ho, wo) per index
        for oc in range(2 * kh * kw):
            for h in range(Ho):
                for w in range(Wo):
                    val = 0.0; mval = 0.0
                    tap = oc // 2; bp_dir = oc % 2
                    i = tap // kw; j = tap % kw
                    for cnt in range(C):
                        col = columns[cnt * kh * kw + tap, h, w]
                        h_in = h * stride - pad; w_in = w * stride - pad
                        off_h = offset[b, 2 * tap, h, w]; off_w = offset[b, 2 * tap + 1, h, w]
                        m = mask[b, tap, h, w]
                        inv_h = h_in + i * dil + off_h; inv_w = w_in + j * dil + off_w
                        if inv_h <= -1 or inv_w <= -1 or inv_h >= H or inv_w >= W:
                            inv_h = inv_w = -2
                        else:
                            mval += col * dcn_ref._bilinear_loops(inp[b, cnt], H, W, inv_h, inv_w)
                        cw = _coordinate_weight_loops(inv_h, inv_w, H, W, inp[b, cnt], bp_dir)
                        val += cw * col * m
                    grad_offset[b, oc, h, w] = val
                    if oc % 2 == 0:
                        grad_mask[b, tap, h, w] = mval
        # col2im (:197-254): one (c, tap, ho, wo) per index
        for c in range(C):
            for i in range(kh):
                for j in range(kw):
                    tap = i * kw + j
                    for h_out in range(Ho):
                        for w_out in range(Wo):
                            h_in = h_out * stride - pad; w_in = w_out * stride - pad
                            off_h = offset[b, 2 * tap, h_out, w_out]; off_w = offset[b, 2 * tap + 1, h_out, w_out]
                            m = mask[b, tap, h_out, w_out]
                            cur_h_f = h_in + i * dil + off_h; cur_w_f = w_in + j * dil + off_w
                            top = columns[c * kh * kw + tap, h_out, w_out] * m
                            cur_h = int(cur_h_f); cur_w = int(cur_w_f)          # (int): truncation toward zero
                            for dy in range(-2, 3):
                                for dx in range(-2, 3):
                                    if (0 <= cur_h + dy < H and 0 <= cur_w + dx < W and
                                            abs(cur_h_f - (cur_h + dy)) < 1 and abs(cur_w_f - (cur_w + dx)) < 1):
                                        wgt = _gradient_weight_loops(cur_h_f, cur_w_f, cur_h + dy, cur_w + dx, H, W)
                                        grad_input[b, c, cur_h + dy, cur_w + dx] += wgt * top
        # im2col, then grad_weight += grad_out . columns^T and grad_bias += grad_out . ones (:302-329)
        col = np.zeros((C * kh * kw, Ho * Wo))
        for c in range(C):
            for h in range(Ho):
                for w in range(Wo):
                    for i in range(kh):
                        for j in range(kw):
                            tap = i * kw + j
                            h_im = h * stride - pad + i * dil + offset[b, 2 * tap, h, w]
                            w_im = w * stride - pad + j * dil + offset[b, 2 * tap + 1, h, w]
                            val = 0.0
                            if h_im > -1 and w_im > -1 and h_im < H and w_im < W:
                                val = dcn_ref._bilinear_loops(inp[b, c], H, W, h_im, w_im)
                            col[c * kh * kw + tap, h * Wo + w] = val * mask[b, tap, h, w]
        grad_weight += (gout @ col.T).reshape(weight.shape)
        grad_bias += gout.sum(axis=1)
    return grad_input, grad_offset, grad_mask, grad_weight, grad_bias


def dcn_v2_backward(inp, weight, bias, offset, mask, grad_out, stride=1, pad=1, dil=1):
    """Autograd through ``dcn_ref.dcn_v2_forward`` in the tensors' own dtype and device (float64 for a reference).
    Returns (grad_input, grad_offset, grad_mask, grad_weight, grad_bias)."""
    leaves = [t.detach().clone().requires_grad_(True) for t in (inp, offset, mask, weight, bias)]
    x, o, m, w, b = leaves
    out = dcn_ref.dcn_v2_forward(x, w, b, o, m, stride, pad, dil)
    gi, go, gm, gw, gb = torch.autograd.grad(out, leaves, grad_out)
    return gi, go, gm, gw, gb
