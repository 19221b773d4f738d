"""Host-side mirror of the reference's model factory (``lib/models/model.py``).

``create_model(arch, head_conv, cfg)`` returns an ``nn.Module`` whose ``state_dict()`` has the
reference's key names and shapes (``backbone_model.*`` / ``head_model.<head>.{0,2}.*``) so
reference checkpoints load unchanged, and whose ``forward`` returns the same six fp32 NCHW
logit maps ``[hm, wh, hps, reg, hm_hp, hp_offset]`` (``lib/models/heads/keypoint.py:40-42``) —
computed by the fused CUDA op program instead of torch modules.  CUDA tensors only: the
product has no CPU path and raises if the CUDA library is missing.
"""
from __future__ import annotations

import torch
from torch import nn

from .archs import dla as _dla
from .archs.common import StateView, attach, conv, scatter_columns
from .plan import PlanBuilder

HEADS = (("hm", 1), ("wh", 2), ("hps", 34), ("reg", 2), ("hm_hp", 17), ("hp_offset", 2))


def _res_arch():
    from .archs import resnet as _res
    return _res


def _mobilenet_arch():
    from .archs import mobilenet as _mb
    return _mb


def _hrnet_arch():
    from .archs import hrnet as _hr
    return _hr


def _hardnet_arch():
    from .archs import hardnet as _hd
    return _hd


def _mobilenetv2_arch():
    from .archs import mobilenetv2 as _mb2
    return _mb2


def _ghostnet_arch():
    from .archs import ghostnet as _gh
    return _gh


_backbone_factory = {
    # arch name -> (module with build_params(cfg)/lower(), feature channels or None = ask the module)   model.py:24-38
    "dla": lambda n: (_dla, 64) if n == 34 else None,
    "res": lambda n: (_res_arch(), 256) if n == 50 else None,
    "hrnet": lambda n: (_hrnet_arch(), None),
    "mobilenetv3": lambda n: (_mobilenet_arch(), 24),
    "hardnet": lambda n: (_hardnet_arch(), 48) if n == 0 else None,
    # both ignore the _N suffix, as the reference does (mobilenetv2.py:256 always builds width 0.5, ghost_net.py:198-200)
    "mobilenetv2": lambda n: (_mobilenetv2_arch(), 24),
    "ghostnet": lambda n: (_ghostnet_arch(), 160),
}


def _build_head(intermediate_channel: int, head_conv: int) -> nn.Module:
    """KeypointHead parameters and init (heads/keypoint.py:14-58)."""
    root = nn.Module()
    for name, c in HEADS:
        attach(root, f"{name}.0", conv(intermediate_channel, head_conv, 3, 1, 1, bias=True))
        attach(root, f"{name}.2", conv(head_conv, c, 1, 1, 0, bias=True))
    with torch.no_grad():
        root.hm._modules["2"].bias.fill_(-2.19)
        root.hm_hp._modules["2"].bias.fill_(-2.19)
        for name in ("wh", "hps", "reg", "hp_offset"):
            for m in getattr(root, name)._modules.values():
                nn.init.normal_(m.weight, std=0.001)
                nn.init.constant_(m.bias, 0)
    return root


class BackBoneWithHead(nn.Module):
    """Same constructor contract as ``lib/models/model.py:44-59``."""

    def __init__(self, arch, head_conv, cfg):
        super().__init__()
        num_layers = int(arch[arch.find("_") + 1:]) if "_" in arch else 0
        arch_name = arch[:arch.find("_")] if "_" in arch else arch
        if arch_name not in _backbone_factory or _backbone_factory[arch_name](num_layers) is None:
            raise KeyError(f"centerpose_b200: backbone {arch!r} is not implemented "
                           f"(available: dla_34, res_50, hrnet, mobilenetv3, hardnet, mobilenetv2, ghostnet)")
        self._arch_mod, feat_c = _backbone_factory[arch_name](num_layers)
        if feat_c is None:
            feat_c = self._arch_mod.feature_channels(cfg)
        self.arch = arch
        self.backbone_model = self._arch_mod.build_params(cfg)
        inter = int(getattr(cfg.MODEL, "INTERMEDIATE_CHANNEL", feat_c))
        if inter != feat_c:
            raise ValueError(f"MODEL.INTERMEDIATE_CHANNEL={inter} but {arch} produces {feat_c} channels")
        self.head_conv = int(cfg.MODEL.HEAD_CONV)
        self.head_model = _build_head(inter, self.head_conv)
        b200 = cfg.get("B200", None) if hasattr(cfg, "get") else getattr(cfg, "B200", None)
        self.precision = (b200 or {}).get("PRECISION", "fp16x2") if isinstance(b200, dict) else "fp16x2"
        self._plans = {}
        self.tc = None
        self.eval()

    # -- weight changes invalidate packed plans
    def load_state_dict(self, *a, **k):
        r = super().load_state_dict(*a, **k)
        self.invalidate()
        return r

    def _apply(self, fn, *a, **k):
        r = super()._apply(fn, *a, **k)
        self.invalidate()
        return r

    def invalidate(self):
        self._plans = {}

    def set_precision(self, precision: str, tc=None):
        """Arithmetic of the forward pass (the reference is fp32 end to end):
          'fp16x2'  wgmma tensor cores on split operands — every activation / weight is a pair of fp16 planes
                    (hi + lo, 22 significand bits), a*b = a_hi*b_hi + a_hi*b_lo + a_lo*b_hi with fp32 accumulation:
                    fp32-faithful (DLA-34 512x512 head maps within 1.8e-5 relative L2 of the reference's fp32 result) at tensor-core
                    speed; activations must stay within the fp16 range (|v| <= 65504, saturating);
          'bf16x2'  same with bf16 planes: full fp32 range, 16 significand bits;
          'bf16'    plain bf16 operands (fastest; ~2e-2 relative L2 through the ~100 layers);
          'fp32'    CUDA-core kernels, fp32 activations (reference arithmetic up to summation order; slow).
        tc=False keeps bf16 activations but forces the CUDA-core kernels — a debugging aid."""
        from .plan import PRECISIONS
        if precision not in PRECISIONS:
            raise ValueError(precision)
        self.precision = precision
        self.tc = tc
        self.invalidate()
        return self

    def _plan(self, B, H, W, device):
        key = (B, H, W, self.precision, self.tc, device.index)
        plan = self._plans.get(key)
        if plan is None:
            pb = PlanBuilder(B, H, W, self.precision, device, tc=self.tc)
            # BatchNorm folding, re-layout and hi/lo splitting of the weights run on the HOST (one-time, a few ms): the
            # device only ever sees the packed operands, and the process launches no torch kernels before its own
            host = torch.device("cpu")
            sd = {k: v.detach().to(host) for k, v in self.state_dict().items()}
            x = pb.input(3)
            feat = self._arch_mod.lower(pb, StateView(sd, "backbone_model.", host), x)
            P = StateView(sd, "head_model.", host)
            # lower() returns one activation, or a list of (activation, real channels) slabs standing for their channel
            # concatenation (archs/hardnet.py): the head's 3x3 convs then take the slabs as their inputs
            slabs = list(feat) if isinstance(feat, (list, tuple)) else None
            srcs = [s for s, _ in slabs] if slabs is not None else [feat]
            fmap = srcs[0]

            def w0_of(name):
                w0 = P(f"{name}.0.weight").float()
                if slabs is not None:
                    return scatter_columns(w0, slabs)
                if feat.C > w0.shape[1]:                 # backbone carries zero-padded channels (archs/mobilenet.py)
                    w0 = torch.nn.functional.pad(w0, (0, 0, 0, 0, 0, feat.C - w0.shape[1]))
                return w0

            hc = self.head_conv
            fuse = pb.use_tc and hc % 16 == 0 and hc <= 128
            if fuse:
                # Narrow heads (ResNet-50 / HRNet: head_conv 64): ONE 3x3 conv produces all six hidden maps: wide N tiles
                # issue fewer MMA instructions per output than six N=64 convs, and the feature map is read once instead of
                # six times.
                w_cat = torch.cat([w0_of(name) for name, _ in HEADS], dim=0)
                b_cat = torch.cat([P(f"{name}.0.bias").float() for name, _ in HEADS], dim=0)
                hid = pb.conv(srcs, w_cat, b_cat, stride=1, pad=1, relu=True)
            for i, (name, c) in enumerate(HEADS):
                dst = pb.output(c, fmap.H, fmap.W, name)
                if fuse:
                    t = pb.channel_slice(hid, i * hc, hc)
                else:
                    t = pb.conv(srcs, w0_of(name), P(f"{name}.0.bias").float(), stride=1, pad=1, relu=True)
                pb.conv([t], P(f"{name}.2.weight").float(), P(f"{name}.2.bias").float(),
                        stride=1, pad=0, relu=False, out="nchw", dst=dst)
            plan = pb.build()
            plan.out_shape = (fmap.H, fmap.W)
            if len(self._plans) > 8:
                self._plans.clear()
            self._plans[key] = plan
        return plan

    @torch.no_grad()
    def forward(self, x):
        if self.training:
            raise RuntimeError("centerpose_b200 implements the inference path only; call .eval()")
        if not x.is_cuda:
            raise RuntimeError("centerpose_b200: forward needs a CUDA tensor (no CPU path in the product)")
        if x.dim() != 4 or x.shape[1] != 3:
            raise RuntimeError("expected input (B,3,H,W)")
        x = x.float().contiguous()
        B, _, H, W = x.shape
        if H % 32 or W % 32:
            raise RuntimeError("input height/width must be multiples of 32 (reference pads with (x|31)+1)")
        plan = self._plan(B, H, W, x.device)
        Ho, Wo = plan.out_shape
        outs = {name: torch.empty((B, c, Ho, Wo), dtype=torch.float32, device=x.device) for name, c in HEADS}
        plan.bind(x, outs)
        plan.run()
        return [outs[name] for name, _ in HEADS]


def create_model(arch, head_conv, cfg):
    """``lib/models/model.py:63-65``."""
    return BackBoneWithHead(arch, head_conv, cfg)


def load_model(model, model_path, optimizer=None, resume=False, lr=None, lr_step=None):
    """``lib/models/model.py:67-120`` — tolerant checkpoint load (strips the DataParallel
    ``module.`` prefix, keeps the model's tensor on shape mismatch, reports missing keys)."""
    checkpoint = torch.load(model_path, map_location="cpu", weights_only=False)
    print("loaded {}, epoch {}".format(model_path, checkpoint["epoch"]))
    src = checkpoint["state_dict"]
    incoming = {}
    for k, v in src.items():
        incoming[k[7:] if k.startswith("module") and not k.startswith("module_list") else k] = v
    own = model.state_dict()
    hint = ("If you see this, your model does not fully load the pre-trained weight. Please make sure "
            "you have correctly specified --arch xxx or set the correct --num_classes for your own dataset.")
    for k in list(incoming):
        if k in own:
            if incoming[k].shape != own[k].shape:
                print("Skip loading parameter {}, required shape{}, loaded shape{}. {}".format(
                    k, own[k].shape, incoming[k].shape, hint))
                incoming[k] = own[k]
        else:
            print("Drop parameter {}.".format(k) + hint)
    for k in own:
        if k not in incoming:
            print("No param {}.".format(k) + hint)
            incoming[k] = own[k]
    model.load_state_dict(incoming, strict=False)
    if optimizer is not None and resume:
        start_epoch = 0
        if "optimizer" in checkpoint:
            optimizer.load_state_dict(checkpoint["optimizer"])
            start_epoch = checkpoint["epoch"]
            start_lr = lr
            for step in lr_step:
                if start_epoch >= step:
                    start_lr *= 0.1
            for group in optimizer.param_groups:
                group["lr"] = start_lr
            print("Resumed optimizer with start lr", start_lr)
        else:
            print("No optimizer parameters in checkpoint.")
        return model, optimizer, start_epoch
    if optimizer is not None:
        return model, optimizer, 0
    return model


def save_model(path, epoch, model, optimizer=None):
    """``lib/models/model.py:122-131`` — ``{'epoch', 'state_dict'[, 'optimizer']}``."""
    state_dict = model.module.state_dict() if isinstance(model, torch.nn.DataParallel) else model.state_dict()
    data = {"epoch": epoch, "state_dict": state_dict}
    if optimizer is not None:
        data["optimizer"] = optimizer.state_dict()
    torch.save(data, path)
