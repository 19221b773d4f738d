"""The training step's ``MultiPoseLoss`` (lib/trains/multi_pose.py) on the device, with its gradient: a drop-in for the
reference trainer's loss module.

    trainer.loss = MultiPoseLoss(cfg, local_rank)       # instead of the reference's MultiPoseLoss
    loss, loss_stats = trainer.loss(outputs, batch)     # outputs: the six head maps, batch: TrainData.batch or the
    loss.backward()                                     #   reference's DataLoader batch moved to the GPU

The forward is two launches (csrc/targets.cu ``cpb200_multi_pose_loss_train_batch``): the focal loss's per-(image,
channel) partials, then one CTA that combines them over the batch in a fixed order with the four regression losses.
The backward is two more (``cpb200_multi_pose_loss_train_backward``): one dense pass writes d loss / d logit of hm and
hm_hp and zero-fills the regression gradients, and one sparse pass writes the gathered entries' gradients.  Nothing of
the reference's graph is kept for the backward: only the inputs and a workspace of ``B * 18 * 3`` doubles.

One departure from the reference: its ``_sigmoid`` calls ``x.sigmoid_()``, so after its forward the model's hm and
hm_hp outputs hold probabilities.  Here the head maps are left as they are, logits.
"""
from __future__ import annotations

import ctypes

import torch

from . import val

REG_KEYS = ("hm", "reg_mask", "ind", "wh", "hps", "hps_mask")


def target_keys(cfg):
    """The batch keys the loss reads under ``cfg``'s LOSS gates: the ones ``TrainData.batch`` returns."""
    c = cfg.LOSS
    return REG_KEYS + (("reg",) if c.REG_OFFSET else ()) + (("hm_hp",) if c.HM_HP else ()) + \
        (("hp_offset", "hp_ind", "hp_mask") if c.REG_HP_OFFSET else ())


def head_gates(cfg):
    """Per head map (hm, wh, hps, reg, hm_hp, hp_offset), whether the loss depends on it; the reference's autograd
    leaves the others' ``.grad`` as None."""
    c = cfg.LOSS
    return (True, c.WH_WEIGHT > 0, True, bool(c.REG_OFFSET) and c.OFF_WEIGHT > 0,
            bool(c.HM_HP) and c.HM_HP_WEIGHT > 0, bool(c.REG_HP_OFFSET) and c.OFF_WEIGHT > 0)


class _Loss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, loss_cfg, gates, batch, hm, wh, hps, reg, hm_hp, hp_offset):
        from . import _lib
        heads = (hm, wh, hps, reg, hm_hp, hp_offset)
        B, R, dev = hm.shape[0], hm.shape[-1], hm.device
        ws = torch.empty(_lib.lib().cpb200_multi_pose_loss_train_workspace_bytes(B), dtype=torch.uint8, device=dev)
        stats = torch.empty(len(val.STATS), dtype=torch.float32, device=dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        _lib.launch("multi_pose_loss_train_batch", dev, _lib.Heads(*[h.data_ptr() for h in heads]),
                    val.targets_struct(batch), B, R, ctypes.byref(loss_cfg), stats, loss, ws)
        ctx.save_for_backward(*heads)
        ctx.loss_cfg, ctx.gates, ctx.batch, ctx.ws = loss_cfg, gates, batch, ws
        ctx.mark_non_differentiable(stats)
        return loss, stats

    @staticmethod
    def backward(ctx, grad_loss, _grad_stats):
        from . import _lib
        heads = ctx.saved_tensors
        hm = heads[0]
        B, R, dev = hm.shape[0], hm.shape[-1], hm.device
        g = grad_loss.to(device=dev, dtype=torch.float32).contiguous()
        grads = [torch.empty_like(h) if on else None for h, on in zip(heads, ctx.gates)]
        _lib.launch("multi_pose_loss_train_backward", dev, _lib.Heads(*[h.data_ptr() for h in heads]),
                    val.targets_struct(ctx.batch), B, R, ctypes.byref(ctx.loss_cfg), g, ctx.ws,
                    _lib.Heads(*[x.data_ptr() if x is not None else None for x in grads]))
        return (None, None, None) + tuple(grads)


class MultiPoseLoss(torch.nn.Module):
    """``MultiPoseLoss(cfg, local_rank)`` of lib/trains/multi_pose.py, normalised over the batch as the trainer calls
    it.  ``forward(outputs, batch)`` takes the six CUDA float32 head maps ``(hm, wh, hps, reg, hm_hp, hp_offset)``
    (hm and hm_hp as logits; they are not modified) and the batch dict, and returns ``(loss, loss_stats)``: ``loss`` a
    0-dim tensor with a ``grad_fn``, ``loss_stats`` the reference's seven keys as 0-dim device tensors.  Refuses the
    settings ``val.check_cfg`` refuses (MSE loss, dense keypoints, non-L1 regression, stacked networks, the oracle
    ablations).  The module has no parameters."""

    def __init__(self, cfg, local_rank=0):
        super().__init__()
        val.check_cfg(cfg)
        self.cfg = cfg
        self.local_rank = local_rank
        self._keys = target_keys(cfg)
        self._gates = head_gates(cfg)
        self._loss_cfg = val.loss_cfg(cfg)

    def forward(self, outputs, batch):
        if len(outputs) != 6:
            raise ValueError("MultiPoseLoss: expected the six head maps (hm, wh, hps, reg, hm_hp, hp_offset), got %d"
                             % len(outputs))
        heads = val.check_loss_inputs(outputs, batch, "MultiPoseLoss", self._keys)
        tg = {k: batch[k] for k in self._keys}
        loss, stats = _Loss.apply(self._loss_cfg, self._gates, tg, *heads)
        loss_stats = {k: stats[i] for i, k in enumerate(val.STATS)}
        loss_stats["loss"] = loss
        return loss, loss_stats
