"""Generate ``tests/golden/train_loss.npz`` from the UNMODIFIED reference's ``MultiPoseLoss`` (lib/trains/multi_pose.py)
and ``.backward()`` on the CPU, and pin the restatement (``oracle/train_loss_ref.py``) against it before anything is
written.

Run:  python -m oracle.make_golden_train_loss      (from the repo root; needs /root/reference)

The cases are ``tests/train_loss_cases.NAMES``.  The reference's ``_sigmoid`` works in place, so each head map is a
leaf cloned before the call, as a network's outputs are.  Per case ``<name>/``:
  stats       the seven float32 stats in STATS order (0 for a term the gates leave out)
  none        (6,) bool: the head maps whose ``.grad`` the reference leaves None
  grad_out    the gradient fed to ``loss.backward``
  <head>_idx, <head>_val   the gradient at flat indices: for hm and hm_hp every element of small maps, else a seeded
              sample with every positive and clamp-edge element; for the regression maps every non-zero element
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "train_loss.npz")
HEADS = ("hm", "wh", "hps", "reg", "hm_hp", "hp_offset")
FULL = 4096             # focal maps up to this many elements are stored whole
SAMPLE = 3000


def focal_index(gt, x, seed):
    n = gt.size
    if n <= FULL:
        return np.arange(n, dtype=np.int64)
    rng = np.random.default_rng(seed)
    s = 1 / (1 + np.exp(-np.asarray(x, np.float64).reshape(-1)))
    pick = np.union1d(rng.choice(n, SAMPLE, replace=False), np.flatnonzero(gt.reshape(-1) == 1))
    return np.union1d(pick, np.flatnonzero((np.abs(s - 1e-4) < 1e-7) | (np.abs(s - 0.9999) < 1e-7)))


def reference_grads(ref_tr, cfg, batch, heads, grad_out):
    leaves = [torch.from_numpy(np.ascontiguousarray(h)).requires_grad_(True) for h in heads]
    crit = ref_tr.MultiPoseLoss(cfg, 0)
    loss, st = crit([h.clone() for h in leaves], {k: torch.from_numpy(v) for k, v in batch.items()})
    loss.backward(torch.tensor(grad_out, dtype=torch.float32))
    stats = np.array([float(st[k]) for k in ("loss", "hm_loss", "hp_loss", "hm_hp_loss", "hp_offset_loss",
                                             "wh_loss", "off_loss")], np.float32)
    return stats, [None if h.grad is None else h.grad.numpy() for h in leaves]


def restated_grads(cfg, batch, heads, grad_out):
    from oracle import train_loss_ref
    leaves = [torch.from_numpy(np.ascontiguousarray(h)).requires_grad_(True) for h in heads]
    loss, st = train_loss_ref.loss_torch(leaves, {k: torch.from_numpy(v) for k, v in batch.items()}, cfg.LOSS)
    loss.backward(torch.tensor(grad_out, dtype=torch.float32))
    stats = np.array([float(st[k]) for k in train_loss_ref.STATS], np.float32)
    return stats, [None if h.grad is None else h.grad.numpy() for h in leaves]


def main():
    from oracle import train_loss_ref
    from oracle.make_golden_train import ref_cfg
    from oracle.make_golden_val import _reference
    from tests import train_loss_cases
    _, ref_tr, _ = _reference()
    out = {}
    for n, name in enumerate(train_loss_cases.NAMES):
        cfg, batch, heads, grad_out = train_loss_cases.case(name, ref_cfg())
        want, wg = reference_grads(ref_tr, cfg, batch, heads, grad_out)
        got, gg = restated_grads(cfg, batch, heads, grad_out)
        assert np.array_equal(got, want), (name, got, want)
        for h, a, b in zip(HEADS, wg, gg):
            assert (a is None) == (b is None), (name, h)
            assert a is None or np.array_equal(a, b), (name, h, np.abs(a - b).max())
        s64 = train_loss_ref.stats64(heads, batch, cfg.LOSS)
        assert np.all(np.abs(s64 - want) <= 1e-5 * np.abs(want)), (name, s64, want)
        key = name + "/"
        out[key + "stats"] = want
        out[key + "none"] = np.array([g is None for g in wg])
        out[key + "grad_out"] = np.float32(grad_out)
        for h, g, x in zip(HEADS, wg, heads):
            if g is None:
                continue
            if h in ("hm", "hm_hp"):
                tg = batch[h]
                idx = focal_index(tg, x, n)
                c = cfg.LOSS
                w = c.HM_WEIGHT if h == "hm" else c.HM_HP_WEIGHT
                v, bound, edge = train_loss_ref.focal_grad64(x, tg, grad_out, w, float((tg == 1).sum()))
                ok = (np.abs(g - v) <= bound) | edge
                assert ok.all(), (name, h, int((~ok).sum()))
            else:
                idx = np.flatnonzero(g.reshape(-1))
            out[key + h + "_idx"] = idx.astype(np.int32)
            out[key + h + "_val"] = g.reshape(-1)[idx]
        print(name, "stats", want.tolist())
    np.savez_compressed(OUT, **out)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    sys.path.insert(0, ROOT)
    main()
