"""Conditioned, seeded weight initialisation and synthetic inputs shared by bench.py, the oracle and the tests
(``oracle/init_recipe.py`` re-exports this module).

BENCH / TEST INFRASTRUCTURE, not on the inference path.  Operates on a reference-format ``state_dict`` (key names of
``lib/models/model.py:44-59`` modules) so the very same tensors can be loaded into the
reference model (via its ``load_model``) and into ``centerpose_b200.create_model``.

Why: with the reference's own initialisers "random-init weights" is numerically degenerate
(SURVEY.md §7 hard part 1): head weights are ``normal(std=0.001)`` (``heads/keypoint.py:52-57``)
and DCN ``conv_offset_mask`` is zero-initialised (``DCNv2/dcn_v2.py:113-115``), so the
heat-map is constant to ~1e-6 (every cell ties) and the deformable sampling path is never
exercised.  This recipe keeps the architecture and shapes and only changes the VALUES:

  * every 4-D conv weight        ~ N(0, gain/sqrt(fan_in)), gain sqrt(2) (ReLU-preserving)
  * depthwise deconv ``up_*``    bilinear kernel (``pose_dla_dcn.py:324-333`` formula) x U(0.8,1.2); a 2x2 kernel
                                 (stride 2: no overlap) is all ones x U(0.8,1.2)
  * ``nn.Linear`` weight         ~ N(0, 2/fan_in)
  * ``conv_offset_mask``         weight ~ N(0, 0.05/sqrt(fan_in)), bias ~ N(0, 0.5): every tap samples at a
                                 fractional position (|offset| ~ 0.5 px from the bias, mask != 0.5) with a small
                                 data-dependent part.  Measured (float64 oracle): with weight gain 0.7 the
                                 16 chained DCNs on spatially white random features amplify a 1e-7 input
                                 perturbation x150 and merely rounding the INPUT to bf16 moves the heads by
                                 28 % — any bf16 parity statement would be meaningless; with 0.05 the
                                 amplification is 1.7 and fp32-vs-fp64 noise is 2e-6.  Large data-dependent
                                 offsets (gain 1.5, many samples out of bounds) are covered at op level
                                 (tests/test_net_gpu.py::test_dcn_op_matches_oracle).
  * BatchNorm                    weight ~ U(0.5,1.5) (U(0.1,0.3) for a bottleneck's last ``bn3``, an HRNet branch
                                 block's last ``bn2`` and a Ghost bottleneck's second ghost module; U(0.2,0.6) inside HRNet ``fuse_layers``; U(0.4,0.8) for a
                                 MobileNetV3 block's projection ``bn3``), bias ~ N(0,0.1),
                                 mean ~ N(0,0.1), var ~ U(0.5,1.5)
  * conv / DCN biases            ~ N(0, 0.1)
  * head final 1x1 (``.2``)      per-head gain so logits/regressions have realistic spread;
                                 hm / hm_hp bias stays -2.19 (``heads/keypoint.py:45-46``)

Tensors are drawn in sorted-key order from one ``torch.Generator(seed)``; seed 317 is the
reference's ``SEED`` (``experiments/*.yaml:6``).
"""
from __future__ import annotations

import math
from collections import OrderedDict

import torch

OFFSET_GAIN = 0.05
HEAD_GAIN = {"hm": 0.09, "hm_hp": 0.055, "wh": 0.5, "hps": 0.65, "reg": 0.027, "hp_offset": 0.013}
HEAD_BIAS = {"hm": -2.19, "hm_hp": -2.19, "wh": 12.0, "hps": 0.0, "reg": 0.5, "hp_offset": 0.5}


def _bilinear_kernel(k: int) -> torch.Tensor:
    f = math.ceil(k / 2)
    c = (2 * f - 1 - f % 2) / (2.0 * f)
    w = torch.zeros(k, k)
    for i in range(k):
        for j in range(k):
            w[i, j] = (1 - abs(i / f - c)) * (1 - abs(j / f - c))
    return w


def conditioned_state_dict(template: "OrderedDict[str, torch.Tensor]", seed: int = 317):
    """template: any state_dict with the target keys/shapes.  Returns a new fp32 state_dict."""
    g = torch.Generator().manual_seed(seed)
    out = OrderedDict()

    def randn(shape): return torch.randn(shape, generator=g)
    def rand(shape, lo, hi): return torch.rand(shape, generator=g) * (hi - lo) + lo

    new = {}
    for k in sorted(template.keys()):
        v = template[k]
        shape = tuple(v.shape)
        if k.endswith("num_batches_tracked"):
            new[k] = torch.zeros((), dtype=torch.long)
            continue
        leaf = k.rsplit(".", 1)[1]
        is_bn = (k.rsplit(".", 1)[0] + ".running_mean") in template
        if is_bn:
            if leaf == "weight":
                # the last BN of a bottleneck residual branch is damped (cf. zero-gamma init) so that 16
                # stacked blocks keep activations O(1..10) instead of growing by ~sqrt(2) per block
                if ".bneck" in k:
                    # MobileNetV3 blocks: bn3 is the linear-bottleneck projection, not a damped residual branch;
                    # U(0.4,0.8) keeps the 15 blocks' activations O(1..25) (0.3-0.6 decays to 1e-1, 0.5-1.0 explodes)
                    new[k] = rand(shape, 0.4, 0.8) if k.endswith(".bn3.weight") else rand(shape, 0.5, 1.5)
                elif k.endswith(".bn3.weight") or (".branches." in k and k.endswith(".bn2.weight")) \
                        or ".conv.3.primary_conv.1." in k or ".conv.3.cheap_operation.1." in k:
                    # (GhostNet: the residual branch ends in a ghost module's two BNs; undamped, the 16 bottlenecks
                    # grow the features to ~1e7)
                    new[k] = rand(shape, 0.1, 0.3)
                elif ".fuse_layers." in k:                         # HRNet cross-resolution terms: y_i = sum_j f_ij(x_j)
                    new[k] = rand(shape, 0.2, 0.6)
                else:
                    new[k] = rand(shape, 0.5, 1.5)
            elif leaf == "bias": new[k] = 0.1 * randn(shape)
            elif leaf == "running_mean": new[k] = 0.1 * randn(shape)
            elif leaf == "running_var": new[k] = rand(shape, 0.5, 1.5)
            else: raise KeyError(k)
            continue
        if v.dim() == 4:
            if ".up_" in k and shape[1] == 1:                     # depthwise ConvTranspose2d
                # k = 2 (stride 2, MobileNetV2's IDAUp): every output reads one tap, so every tap carries weight (the
                # bilinear formula would give the (0, 0) tap only)
                base = (torch.ones(shape[2], shape[3]) if shape[2] == 2 else _bilinear_kernel(shape[2])).view(1, 1, shape[2], shape[3])
                new[k] = base * rand(shape, 0.8, 1.2)
                continue
            if "deconv_layers" in k:                              # dense ConvTranspose2d (Cin,Cout,k,k)
                fan_in = shape[0] * shape[2] * shape[3] / 4.0     # stride-2: ~k*k/4 taps hit each output
            else:
                fan_in = shape[1] * shape[2] * shape[3]
            if "conv_offset_mask" in k:
                new[k] = randn(shape) * (OFFSET_GAIN / math.sqrt(fan_in))
            elif k.startswith("head_model.") and k.endswith(".2.weight"):
                head = k.split(".")[1]
                new[k] = randn(shape) * (HEAD_GAIN[head] / math.sqrt(fan_in))
            else:
                new[k] = randn(shape) * math.sqrt(2.0 / fan_in)
            continue
        if v.dim() == 2:                                          # nn.Linear (GhostNet's SE): ReLU-preserving gain
            new[k] = randn(shape) * math.sqrt(2.0 / shape[1])
            continue
        if v.dim() == 1:                                          # conv / DCN / Linear bias
            if "conv_offset_mask" in k:
                new[k] = 0.5 * randn(shape)
            elif k.startswith("head_model.") and k.endswith(".2.bias"):
                head = k.split(".")[1]
                new[k] = torch.full(shape, HEAD_BIAS[head]) + (0.0 if head in ("hm", "hm_hp") else 1.0) * 0.05 * randn(shape)
            else:
                new[k] = 0.1 * randn(shape)
            continue
        raise KeyError(f"unhandled parameter {k} {shape}")
    for k in template.keys():                                      # preserve template order
        out[k] = new[k].to(torch.float32) if new[k].is_floating_point() else new[k]
    return out


def synth_images(B: int, H: int = 512, W: int = 512, seed: int = 317) -> torch.Tensor:
    """Already-normalised synthetic images (SURVEY.md §8d): N(0,1), fp32 NCHW."""
    g = torch.Generator().manual_seed(seed)
    return torch.randn(B, 3, H, W, generator=g)
