"""Cases of the trainer's loss (``centerpose_b200.train_loss``), shared by ``oracle/make_golden_train_loss.py`` and the
tests.  A case is a LOSS override, a batch (numpy, with the batch dimension, the keys the gates keep), the six seeded
head maps and the gradient fed to ``backward``.

* ``train/<name>``: the training batches of ``tests/train_cases.CASES`` (the numpy restatement of the reference's
  ``__getitem__``, pinned against it) with seeded logits.
* constructed batches at R = 8: no positive at all, a ``rot != 0`` image (hm 0.9999 everywhere, masks 0) next to
  normal ones, two and three objects on one centre and joints of several people on one pixel, predictions equal to
  their targets, logits at and just beyond both clamp edges, and every gate combination of the LOSS settings."""
from __future__ import annotations

import numpy as np
import torch

from tests.train_cases import CASES, case_cfg, dataset

J, M = 17, 32
HEAD_CHANNELS = (1, 2, 2 * J, 2, J, 2)
KEYS = ["hm", "hm_hp", "wh", "reg", "ind", "reg_mask", "hps", "hps_mask", "hp_offset", "hp_ind", "hp_mask"]
LO, HI = np.float32(1e-4), np.float32(1 - 1e-4)

# name, LOSS overrides
GATES = [("gate_no_hm_hp", {"HM_HP": False}), ("gate_hm_hp_weight_0", {"HM_HP_WEIGHT": 0.}),
         ("gate_wh_weight_0", {"WH_WEIGHT": 0.}), ("gate_no_reg_offset", {"REG_OFFSET": False}),
         ("gate_no_hp_offset", {"REG_HP_OFFSET": False}), ("gate_off_weight_0", {"OFF_WEIGHT": 0.}),
         ("gate_all_off", {"HM_HP": False, "WH_WEIGHT": 0., "REG_OFFSET": False, "REG_HP_OFFSET": False})]
CONSTRUCTED = ["no_pos", "rot_image", "shared_pixels", "exact", "clamp_edges"]
NAMES = ["train/" + c[0] for c in CASES] + CONSTRUCTED + [g[0] for g in GATES]
GRAD_OUT = {"exact": 3.5, "shared_pixels": -0.75}


def logits(seed, B, R):
    """Six seeded (B, C, R, R) float32 head maps: hm and hm_hp logits around -3 (their logistic spans both clamp
    bounds), regression maps of the targets' scale."""
    rng = np.random.RandomState(seed)
    out = []
    for n, c in enumerate(HEAD_CHANNELS):
        if n in (0, 4):
            out.append((rng.standard_normal((B, c, R, R)) * 3 - 3).astype(np.float32))
        else:
            out.append((rng.standard_normal((B, c, R, R)) * (10 if n in (1, 2) else 0.5)).astype(np.float32))
    return out


def gate_keys(loss):
    return [k for k in KEYS if not ((k == "reg" and not loss["REG_OFFSET"]) or (k == "hm_hp" and not loss["HM_HP"])
                                    or (k.startswith("hp_") and not loss["REG_HP_OFFSET"]))]


def clamp_edge_logits():
    """float32 logits whose float32 logistic is the lower clamp bound, just below it, the upper bound and just above
    it, as torch computes the logistic."""
    out = []
    for bound, sign in ((LO, -1), (HI, 1)):
        x = np.float32(np.log(bound / (1 - np.float64(bound))))
        for _ in range(400):
            s = torch.sigmoid(torch.tensor(x)).numpy()
            if s == bound:
                break
            x = np.nextafter(x, np.float32(np.inf) if s < bound else np.float32(-np.inf))
        assert torch.sigmoid(torch.tensor(x)).numpy() == bound
        beyond = x
        while torch.sigmoid(torch.tensor(beyond)).numpy() == bound:
            beyond = np.nextafter(beyond, np.float32(sign * np.inf))
        out += [x, beyond]
    return np.array(out, np.float32)


def _synthetic(seed, B=3, R=8, n=4):
    """A batch of B images with n objects each at distinct centres, their joints partly visible."""
    rng = np.random.default_rng(seed)
    f = np.float32
    b = {"hm": (rng.uniform(0, 0.95, (B, 1, R, R)) * (rng.random((B, 1, R, R)) < 0.6)).astype(f),
         "hm_hp": (rng.uniform(0, 0.95, (B, J, R, R)) * (rng.random((B, J, R, R)) < 0.3)).astype(f),
         "wh": np.zeros((B, M, 2), f), "reg": np.zeros((B, M, 2), f), "ind": np.zeros((B, M), np.int64),
         "reg_mask": np.zeros((B, M), np.uint8), "hps": np.zeros((B, M, 2 * J), f),
         "hps_mask": np.zeros((B, M, 2 * J), np.uint8), "hp_offset": np.zeros((B, M * J, 2), f),
         "hp_ind": np.zeros((B, M * J), np.int64), "hp_mask": np.zeros((B, M * J), np.int64)}
    for i in range(B):
        ct = rng.choice(R * R, n, replace=False)
        b["ind"][i, :n] = ct
        b["reg_mask"][i, :n] = 1
        b["hm"][i, 0].reshape(-1)[ct] = 1
        b["wh"][i, :n] = rng.uniform(1, 30, (n, 2))
        b["reg"][i, :n] = rng.uniform(0, 1, (n, 2))
        for k in range(n):
            vis = rng.random(J) < 0.7
            b["hps"][i, k] = np.where(np.repeat(vis, 2), rng.uniform(-20, 20, 2 * J), 0)
            b["hps_mask"][i, k] = np.repeat(vis, 2)
            pix = rng.integers(0, R * R, J)
            b["hp_ind"][i, k * J:(k + 1) * J] = np.where(vis, pix, 0)
            b["hp_mask"][i, k * J:(k + 1) * J] = vis
            b["hp_offset"][i, k * J:(k + 1) * J] = np.where(vis[:, None], rng.uniform(0, 1, (J, 2)), 0)
            for j in np.flatnonzero(vis):
                b["hm_hp"][i, j].reshape(-1)[pix[j]] = 1
    return b


def constructed(name):
    """``(batch, heads)`` of a constructed case."""
    seed = 50 + (CONSTRUCTED.index(name) if name in CONSTRUCTED else 10 + [g[0] for g in GATES].index(name))
    b = _synthetic(seed)
    B, R = b["hm"].shape[0], b["hm"].shape[-1]
    heads = logits(seed, B, R)
    if name == "no_pos":
        for k in ("hm", "hm_hp"):
            b[k][b[k] == 1] = np.float32(0.96)
    elif name == "rot_image":
        b["hm"][1] = np.float32(0.9999)
        b["reg_mask"][1] = 0
        b["hps_mask"][1] = 0
    elif name == "shared_pixels":
        b["ind"][0, 1] = b["ind"][0, 0]                         # two objects on one centre
        b["ind"][1, 1] = b["ind"][1, 2] = b["ind"][1, 0]        # three
        for k in range(4):                                       # joint 3 of every person on one pixel, with joint 5
            b["hp_ind"][0, k * J + 3] = b["hp_ind"][0, 5]        # of person 0 and joint 7 of person 2
            b["hp_mask"][0, k * J + 3] = 1
        b["hp_ind"][0, 2 * J + 7] = b["hp_ind"][0, 5]
        b["hp_mask"][0, 2 * J + 7] = 1
        b["hps_mask"][:, :3] = 1
    elif name == "exact":
        # every second entry's prediction equals its target: sign(0) = 0
        _, wh, hps, reg, _, hp_offset = heads
        for i in range(B):
            for k in range(0, M, 2):
                for c in range(2):
                    wh[i, c].reshape(-1)[b["ind"][i, k]] = b["wh"][i, k, c]
                    reg[i, c].reshape(-1)[b["ind"][i, k]] = b["reg"][i, k, c]
                for c in range(2 * J):
                    hps[i, c].reshape(-1)[b["ind"][i, k]] = b["hps"][i, k, c]
            for e in range(0, M * J, 2):
                for c in range(2):
                    hp_offset[i, c].reshape(-1)[b["hp_ind"][i, e]] = b["hp_offset"][i, e, c]
    elif name == "clamp_edges":
        x = clamp_edge_logits()
        hm, hm_hp = heads[0], heads[4]
        for i in range(B):
            hm[i, 0, i, :4] = x
            hm[i, 0, i + 3, :4] = x
            b["hm"][i, 0, i + 3, :4] = 1                         # the same logits on positives
            for j in range(0, J, 4):
                hm_hp[i, j, 2, 2:6] = x
                b["hm_hp"][i, j, 2, 2:4] = 1
    return b, heads


def case(name, base_cfg):
    """``(cfg, batch, heads, grad_out)`` of case ``name``; ``base_cfg`` is the package's default config (the golden
    generator passes the reference's view of it)."""
    import copy
    if name.startswith("train/"):
        from oracle.make_golden_train import pixels, restated
        ci = [c[0] for c in CASES].index(name[6:])
        _, settings, res, np_seed, py_seed = CASES[ci]
        cfg = case_cfg(base_cfg, settings, res)
        ds = dataset(name[6:])
        items = restated(ds, pixels(ci, ds), cfg, np_seed, py_seed)
        batch = {k: np.stack([np.asarray(tg[k]) for tg, _ in items]) for k in KEYS}
        heads = logits(900 + ci, len(items), cfg.MODEL.OUTPUT_RES)
    else:
        cfg = copy.deepcopy(base_cfg)
        for g, over in GATES:
            if g == name:
                cfg.LOSS.update(over)
        batch, heads = constructed(name)
        cfg.MODEL.OUTPUT_RES = batch["hm"].shape[-1]
        cfg.MODEL.INPUT_RES = cfg.MODEL.INPUT_H = cfg.MODEL.INPUT_W = 4 * cfg.MODEL.OUTPUT_RES
        cfg.MODEL.DOWN_RATIO = 4
    batch = {k: batch[k] for k in gate_keys(cfg.LOSS)}
    return cfg, batch, heads, GRAD_OUT.get(name, 1.0)
