"""Restatements of the trainer's MultiPoseLoss (lib/trains/multi_pose.py) over a batch, and of its gradient, for
``centerpose_b200.train_loss``'s tests.

* :func:`loss_torch`: the loss as torch ops with autograd, on the CPU or the device: ``sigmoid`` (out of place), the
  clamp, CornerNet's focal loss normalised over the whole batch, and the L1 terms of the gathered entries divided by
  the batch's mask count + 1e-4.  ``backward()`` through it is the op sequence the reference's autograd runs.
* :func:`stats64`: the seven stats with float64 sums (``val_ref.loss`` on the batch laid out as one image).
* :func:`focal_grad64`: d loss / d logit of a focal map as the float64 evaluation of the float32 op chain the device
  runs, with a first-order bound on the float32 chain's error for every element.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import val_ref

J = 17
HEADS = ("hm", "wh", "hps", "reg", "hm_hp", "hp_offset")
STATS = val_ref.STATS
LO, HI = float(np.float32(1e-4)), float(np.float32(1 - 1e-4))


def _focal(logits, gt):
    p = torch.clamp(torch.sigmoid(logits), min=1e-4, max=1 - 1e-4)
    pos = gt.eq(1).float()
    neg = gt.lt(1).float()
    pos_sum = (torch.log(p) * torch.pow(1 - p, 2) * pos).sum()
    neg_sum = (torch.log(1 - p) * torch.pow(p, 2) * torch.pow(1 - gt, 4) * neg).sum()
    npos = pos.sum()
    return -neg_sum if npos == 0 else -(pos_sum + neg_sum) / npos


def _l1(head, mask, ind, target, per_value):
    B, C = head.shape[:2]
    pred = head.permute(0, 2, 3, 1).reshape(B, -1, C).gather(1, ind[:, :, None].expand(-1, -1, C))
    m = mask.float() if per_value else mask[:, :, None].expand_as(pred).float()
    return torch.nn.functional.l1_loss(pred * m, target * m, reduction="sum") / (m.sum() + 1e-4)


def loss_torch(heads, batch, loss_cfg):
    """``(loss, stats)`` of the six (B, C, R, R) head maps ``heads`` (hm and hm_hp as logits) and the batch dict
    ``batch``, ``loss_cfg`` the cfg's LOSS section; ``stats`` maps :data:`STATS` to 0-dim tensors (0. for a term the
    gates leave out).  The gradient flows to the heads the loss reads."""
    hm, wh, hps, reg, hm_hp, hp_offset = heads
    c = loss_cfg
    z = torch.zeros((), device=hm.device)
    st = {k: z for k in STATS}
    st["hm_loss"] = _focal(hm, batch["hm"])
    st["hp_loss"] = _l1(hps, batch["hps_mask"], batch["ind"], batch["hps"], True)
    if c["WH_WEIGHT"] > 0:
        st["wh_loss"] = _l1(wh, batch["reg_mask"], batch["ind"], batch["wh"], False)
    if c["REG_OFFSET"] and c["OFF_WEIGHT"] > 0:
        st["off_loss"] = _l1(reg, batch["reg_mask"], batch["ind"], batch["reg"], False)
    if c["REG_HP_OFFSET"] and c["OFF_WEIGHT"] > 0:
        st["hp_offset_loss"] = _l1(hp_offset, batch["hp_mask"], batch["hp_ind"], batch["hp_offset"], False)
    if c["HM_HP"] and c["HM_HP_WEIGHT"] > 0:
        st["hm_hp_loss"] = _focal(hm_hp, batch["hm_hp"])
    loss = c["HM_WEIGHT"] * st["hm_loss"] + c["WH_WEIGHT"] * st["wh_loss"] + c["OFF_WEIGHT"] * st["off_loss"] + \
        c["HP_WEIGHT"] * st["hp_loss"] + c["HM_HP_WEIGHT"] * st["hm_hp_loss"] + c["OFF_WEIGHT"] * st["hp_offset_loss"]
    st["loss"] = loss
    return loss, st


def stats64(heads, batch, loss_cfg):
    """The seven float32 stats in :data:`STATS` order with float64 sums: the batch is laid out as one image whose
    planes hold every image's plane side by side, so ``val_ref.loss`` normalises over the whole batch."""
    heads = [np.asarray(h, np.float32) for h in heads]
    B, _, R, _ = heads[0].shape
    one = [h.transpose(1, 0, 2, 3).reshape(h.shape[1], B * R, R) for h in heads]
    off = (np.arange(B, dtype=np.int64) * R * R)[:, None]
    tg = {}
    for k in ("hm", "hm_hp"):
        if k in batch:
            tg[k] = np.asarray(batch[k]).transpose(1, 0, 2, 3).reshape(-1, B * R, R)
    for k in ("wh", "reg", "hps", "hps_mask", "hp_offset", "reg_mask", "hp_mask"):
        if k in batch:
            a = np.asarray(batch[k])
            tg[k] = a.reshape((-1,) + a.shape[2:])
    tg["ind"] = (np.asarray(batch["ind"]) + off).reshape(-1)
    if "hp_ind" in batch:
        tg["hp_ind"] = (np.asarray(batch["hp_ind"]) + off).reshape(-1)
    return val_ref.loss(one, tg, loss_cfg)


U = 2.0 ** -24          # unit roundoff of float32: a rounded result is within U * |x| (normal range)
TINY = 2.0 ** -149      # and within this absolutely below it


def _r(v):
    return U * np.abs(v) + TINY


def focal_grad64(logits, gt, grad_loss, weight, npos):
    """d (grad_loss * weight * focal loss) / d logits as the device evaluates it (csrc/targets.cu ``focal_grad``), in
    float64: ``(value, bound, edge)``.  ``bound`` bounds |float32 result - value| to first order: every float32 op
    adds its rounding (half an ulp, at most U * |result|) to the propagated error of its operands, ``expf`` adds 2 ulp
    and ``logf`` 1 ulp (CUDA's stated maximum errors; torch's CPU exp and log are within them).  ``edge`` marks the
    elements whose logistic lies within its error of a clamp bound: there the float32 chain may take either side of
    the clamp, so the bound does not hold and the side is compared with the reference instead."""
    x = np.asarray(logits, np.float64)
    gt = np.asarray(gt, np.float64)
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        e = np.exp(-x)
        ee = 4 * U * e
        a = 1 + e
        ea = ee + _r(a)
        s = 1 / a
        es = ea / (a * a) + _r(s)
        inside = (s >= LO) & (s <= HI)
        edge = (np.abs(s - LO) <= es) | (np.abs(s - HI) <= es)
        p = np.clip(s, LO, HI)
        ep = np.where(inside, es, 0.)
        G = -(float(grad_loss) * float(weight))
        g = G / npos if npos else G
        eg = 2 * _r(g)
        pi, ni = (gt == 1).astype(np.float64), (gt < 1).astype(np.float64)
        q = 1 - p
        eq = ep + _r(q)
        w = 1 - gt
        ew = _r(w)
        w2 = w * w
        ew2 = 2 * np.abs(w) * ew + _r(w2)
        nw = w2 * w2
        enw = 2 * np.abs(w2) * ew2 + _r(nw)
        h = g * ni * nw
        eh = np.abs(nw) * eg * ni + np.abs(g * ni) * enw + _r(h)
        p2 = p * p
        ep2 = 2 * p * ep + _r(p2)
        t3n = h * p2
        et3n = p2 * eh + np.abs(h) * ep2 + _r(t3n)
        t3 = t3n / q
        et3 = et3n / q + np.abs(t3) * eq / q + _r(t3)
        L = np.log(q)
        eL = eq / q + 2 * U * np.abs(L) + TINY
        hL = h * L
        ehL = np.abs(L) * eh + np.abs(h) * eL + _r(hL)
        t4 = hL * 2 * p
        et4 = 2 * p * ehL + np.abs(hL) * 2 * ep + _r(t4)
        d = -t3 + t4
        ed = et3 + et4 + _r(d)
        if npos:
            gp = g * pi
            egp = eg * pi
            qq = q * q
            eqq = 2 * q * eq + _r(qq)
            t1n = gp * qq
            et1n = qq * egp + np.abs(gp) * eqq + _r(t1n)
            t1 = t1n / p
            et1 = et1n / p + np.abs(t1) * ep / p + _r(t1)
            A = np.log(p)
            eA = ep / p + 2 * U * np.abs(A) + TINY
            gA = gp * A
            egA = np.abs(A) * egp + np.abs(gp) * eA + _r(gA)
            t2 = gA * 2 * q
            et2 = 2 * q * egA + np.abs(gA) * 2 * eq + _r(t2)
            pos = t1 - t2
            epos = et1 + et2 + _r(pos)
            d = pos + d
            ed = epos + ed + _r(d)
        ds = np.where(inside, d, 0.)
        eds = np.where(inside, ed, 0.)
        oms = 1 - s
        eoms = es + _r(oms)
        r1 = ds * oms
        er1 = np.abs(oms) * eds + np.abs(ds) * eoms + _r(r1)
        out = r1 * s
        eout = np.abs(s) * er1 + np.abs(r1) * es + _r(out)
    # second-order terms: every relative error above is far below 1e-3
    return out, eout * (1 + 1e-3), edge
