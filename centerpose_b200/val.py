"""The reference's validation pass on the device (``tools/train.py``'s ``trainer.val``): the val split's training
targets (``MultiPoseDataset.__getitem__``, csrc/targets.cu ``cpb200_multi_pose_targets_batch``) and
``MultiPoseLoss.forward``'s seven stats (``cpb200_multi_pose_loss_batch``).

    ev = KeypointEval("person_keypoints_val2017.json")   # the ground truth, parsed and uploaded once
    tg = targets(ev, image_ids, shapes, cfg)              # {'hm', 'hm_hp', 'wh', 'reg', 'ind', ...} CUDA tensors
    stats = loss(model(inputs), tg, cfg)                  # (B, 7) float32, in STATS order

``MultiPoseDetector.run_val`` chains the image loading, the dataset's input warp, the forward, these two steps and the
decode of the predictions.  The targets are built from ``KeypointEval``'s ground-truth table, so the annotations are
parsed once for both the loss and the AP.
"""
from __future__ import annotations

import ctypes

import numpy as np
import torch

from .image import get_affine_transform

J = 17
MAX_OBJS = 32
STATS = ["loss", "hm_loss", "hp_loss", "hm_hp_loss", "hp_offset_loss", "wh_loss", "off_loss"]

# one entry of cpb200_multi_pose_targets_batch's device table (struct cpb200_val_image, include/centerpose_b200.h)
VAL_IMAGE = np.dtype([("gt_begin", "<i4"), ("gt_count", "<i4"), ("pad", "<i4", (2,)), ("trans_output", "<f8", (6,))])
assert VAL_IMAGE.itemsize == 64

# name, dtype and per-image shape (R the output resolution) of every target, in cpb200_multi_pose_targets order
TARGETS = [("hm", torch.float32, lambda R: (1, R, R)), ("hm_hp", torch.float32, lambda R: (J, R, R)),
           ("wh", torch.float32, lambda R: (MAX_OBJS, 2)), ("reg", torch.float32, lambda R: (MAX_OBJS, 2)),
           ("ind", torch.int64, lambda R: (MAX_OBJS,)), ("reg_mask", torch.uint8, lambda R: (MAX_OBJS,)),
           ("hps", torch.float32, lambda R: (MAX_OBJS, 2 * J)), ("hps_mask", torch.uint8, lambda R: (MAX_OBJS, 2 * J)),
           ("hp_offset", torch.float32, lambda R: (MAX_OBJS * J, 2)), ("hp_ind", torch.int64, lambda R: (MAX_OBJS * J,)),
           ("hp_mask", torch.int64, lambda R: (MAX_OBJS * J,))]


def center_scale(height, width):
    """The val split's ``c`` and ``s`` of an image (multi_pose.py: no augmentation)."""
    return np.array([width / 2., height / 2.], dtype=np.float32), max(height, width) * 1.0


def check_cfg(cfg, ev=None):
    """Raises ``NotImplementedError`` for the settings the device validation does not cover."""
    loss, model = cfg.LOSS, cfg.MODEL
    if loss.MSE_LOSS:
        raise NotImplementedError("validation with LOSS.MSE_LOSS (the reference needs cfg.hm_gauss, which it lacks)")
    if loss.DENSE_HP:
        raise NotImplementedError("validation with LOSS.DENSE_HP")
    if loss.REG_LOSS != "l1":
        raise NotImplementedError("validation with LOSS.REG_LOSS %r (only 'l1')" % (loss.REG_LOSS,))
    if int(model.NUM_STACKS) != 1:
        raise NotImplementedError("validation with MODEL.NUM_STACKS %r (only 1)" % (model.NUM_STACKS,))
    oracle = sorted(k for k, v in cfg.TEST.items() if k.startswith("EVAL_ORACLE_") and v)
    if oracle:
        raise NotImplementedError("validation with TEST.%s" % ", ".join(oracle))
    if int(model.OUTPUT_RES) * int(model.DOWN_RATIO) != int(model.INPUT_RES):
        raise NotImplementedError("validation with MODEL.OUTPUT_RES %d != INPUT_RES %d / DOWN_RATIO %d (the targets "
                                  "would index another grid than the head maps)"
                                  % (model.OUTPUT_RES, model.INPUT_RES, model.DOWN_RATIO))
    if ev is not None and ev.cat_id != 1:
        raise NotImplementedError("validation with ground-truth category id %r (the dataset's only id is 1)"
                                  % (ev.cat_id,))


def image_table(ev, image_ids, shapes, R):
    """The ``cpb200_val_image`` rows of images ``image_ids`` of sizes ``shapes`` (h, w) against ``ev``'s table."""
    if len(image_ids) != len(shapes):
        raise ValueError("val: %d image ids for %d shapes" % (len(image_ids), len(shapes)))
    t = np.zeros(len(image_ids), VAL_IMAGE)
    for n, (i, (h, w)) in enumerate(zip(image_ids, shapes)):
        if i not in ev.gt_range:
            raise ValueError("val: image id %r is not in the ground truth" % (i,))
        c, s = center_scale(h, w)
        t[n]["gt_begin"], t[n]["gt_count"] = ev.gt_range[i]
        t[n]["trans_output"] = np.asarray(get_affine_transform(c, s, 0, [R, R]), np.float64).reshape(6)
    return t


def targets_struct(tensors):
    """The ``cpb200_multi_pose_targets`` of the dict ``tensors`` under :data:`TARGETS`' names; a name it lacks is
    NULL."""
    from . import _lib
    return _lib.Targets(*[tensors[n].data_ptr() if n in tensors else None for n, _, _ in TARGETS])


def targets(ev, image_ids, shapes, cfg):
    """The val split's targets of images ``image_ids`` (of sizes ``shapes``, (h, w)) against the ground truth of the
    ``KeypointEval`` ``ev``: a dict of CUDA tensors on ``ev.device`` under the reference's batch keys, each with a
    leading batch dimension."""
    from . import _lib
    R = int(cfg.MODEL.OUTPUT_RES)
    table = image_table(ev, list(image_ids), list(shapes), R)
    B = len(table)
    out = {name: torch.empty((B,) + shape(R), dtype=dt, device=ev.device) for name, dt, shape in TARGETS}
    if B == 0:
        return out
    up = torch.from_numpy(table.view(np.uint8).reshape(-1).copy()).pin_memory().to(ev.device, non_blocking=True)
    _lib.launch("multi_pose_targets_batch", ev.device, up, B, ev.gts, R, targets_struct(out))
    return out


def loss_cfg(cfg):
    from . import _lib
    c = cfg.LOSS
    return _lib.LossCfg(float(c.HM_WEIGHT), float(c.WH_WEIGHT), float(c.OFF_WEIGHT), float(c.HP_WEIGHT),
                        float(c.HM_HP_WEIGHT), int(bool(c.HM_HP)), int(bool(c.REG_OFFSET)), int(bool(c.REG_HP_OFFSET)))


def check_loss_inputs(outputs, targets, what, names=None):
    """The six head maps ``outputs`` as contiguous tensors, after checking that they are CUDA float32 (B, C, R, R) on
    one device and that the ``targets`` named ``names`` (default: all of :data:`TARGETS`) are contiguous tensors of
    the dataset's dtypes and shapes on that device.  Raises ``ValueError`` naming ``what`` otherwise."""
    heads = [o.contiguous() for o in outputs]
    hm = heads[0]
    B, R = hm.shape[0], hm.shape[-1]
    for h, c in zip(heads, (1, 2, 2 * J, 2, J, 2)):
        if not h.is_cuda or h.dtype != torch.float32 or tuple(h.shape) != (B, c, R, R) or h.device != hm.device:
            raise ValueError("%s: head maps must be CUDA float32 (B, C, R, R) with C = 1, 2, 34, 2, 17, 2 on one "
                             "device; got %s" % (what, [(tuple(x.shape), x.dtype) for x in heads]))
    for name, dt, shape in TARGETS:
        if names is not None and name not in names:
            continue
        if name not in targets:
            raise ValueError("%s: the batch has no target %r" % (what, name))
        t = targets[name]
        if t.dtype != dt or tuple(t.shape) != (B,) + shape(R) or t.device != hm.device or not t.is_contiguous():
            raise ValueError("%s: target %r is %s %s, expected %s %s on %s"
                             % (what, name, t.dtype, tuple(t.shape), dt, (B,) + shape(R), hm.device))
    return heads


def loss(outputs, targets, cfg):
    """``MultiPoseLoss.forward`` per image on the forward's six head maps ``outputs`` (hm and hm_hp as logits; they
    are not modified) and ``targets`` (:func:`targets`).  Returns a (B, 7) float32 CUDA tensor, the stats in
    :data:`STATS` order, as each image's ``loss_stats[l].mean().item()`` would be in a batch of one."""
    from . import _lib
    heads = check_loss_inputs(outputs, targets, "val.loss")
    hm = heads[0]
    B, R = hm.shape[0], hm.shape[-1]
    stats = torch.empty((B, len(STATS)), dtype=torch.float32, device=hm.device)
    ws = torch.empty(max(_lib.lib().cpb200_multi_pose_loss_workspace_bytes(B), 1), dtype=torch.uint8, device=hm.device)
    cfg_c = loss_cfg(cfg)
    _lib.launch("multi_pose_loss_batch", hm.device, _lib.Heads(*[h.data_ptr() for h in heads]), targets_struct(targets),
                B, R, ctypes.byref(cfg_c), stats, ws)
    return stats
