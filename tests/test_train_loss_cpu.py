"""CPU tests of the trainer's loss: the torch restatement (oracle/train_loss_ref.py) and the float64 gradient bounds
against the reference's MultiPoseLoss and backward (tests/golden/train_loss.npz), the settings and inputs
``train_loss.MultiPoseLoss`` refuses, and the C-ABI structs the new entry points take."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from centerpose_b200 import train_loss
from centerpose_b200.config import default_cfg
from oracle import train_loss_ref
from tests import train_loss_cases as tc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "train_loss.npz")
HEADS = train_loss_ref.HEADS


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLD))


def restated(cfg, batch, heads, grad_out):
    leaves = [torch.from_numpy(np.ascontiguousarray(h)).requires_grad_(True) for h in heads]
    loss, st = train_loss_ref.loss_torch(leaves, {k: torch.from_numpy(v) for k, v in batch.items()}, cfg.LOSS)
    loss.backward(torch.tensor(grad_out))
    return np.array([float(st[k].detach()) for k in train_loss_ref.STATS], np.float32), \
        [None if h.grad is None else h.grad.numpy() for h in leaves]


@pytest.mark.parametrize("name", tc.NAMES)
def test_restatement_matches_golden(gold, name):
    cfg, batch, heads, grad_out = tc.case(name, default_cfg("dla_34"))
    key = name + "/"
    assert float(gold[key + "grad_out"]) == grad_out
    stats, grads = restated(cfg, batch, heads, grad_out)
    want = gold[key + "stats"]
    assert np.all(np.abs(stats - want) <= 1e-6 * np.abs(want)), (stats, want)
    s64 = train_loss_ref.stats64(heads, batch, cfg.LOSS)
    assert np.all(np.abs(s64 - want) <= 1e-5 * np.abs(want)), (s64, want)
    assert [g is None for g in grads] == gold[key + "none"].tolist()
    assert [g is None for g in grads] == [not on for on in train_loss.head_gates(cfg)]
    for h, g, x in zip(HEADS, grads, heads):
        if g is None:
            continue
        idx, val = gold[key + h + "_idx"], gold[key + h + "_val"]
        if h in ("hm", "hm_hp"):
            c = cfg.LOSS
            v, bound, edge = train_loss_ref.focal_grad64(x, batch[h], grad_out,
                                                         c.HM_WEIGHT if h == "hm" else c.HM_HP_WEIGHT,
                                                         float((batch[h] == 1).sum()))
            for got in (g.reshape(-1)[idx], val):
                ok = np.abs(got - v.reshape(-1)[idx]) <= bound.reshape(-1)[idx]
                assert (ok | edge.reshape(-1)[idx]).all()
            e = edge.reshape(-1)[idx]
            assert np.array_equal(g.reshape(-1)[idx][e] == 0, val[e] == 0)
        else:
            # the reference's scatter_add on the CPU sums in slot order: the restatement is the same op
            assert np.array_equal(np.flatnonzero(g.reshape(-1)), idx) and np.array_equal(g.reshape(-1)[idx], val)


def test_cases_reach_what_they_claim(gold):
    cfg, batch, heads, _ = tc.case("no_pos", default_cfg("dla_34"))
    assert not (batch["hm"] == 1).any() and not (batch["hm_hp"] == 1).any()
    _, batch, _, _ = tc.case("rot_image", default_cfg("dla_34"))
    assert (batch["hm"][1] == np.float32(0.9999)).all() and (batch["hm"][0] == 1).any()
    _, batch, _, _ = tc.case("shared_pixels", default_cfg("dla_34"))
    assert len(set(batch["ind"][1, :3].tolist())) == 1
    hp = batch["hp_ind"][0][batch["hp_mask"][0] == 1]
    assert np.bincount(hp).max() >= 5
    x = tc.clamp_edge_logits()
    s = torch.sigmoid(torch.from_numpy(x)).numpy()
    assert s[0] == tc.LO and s[1] < tc.LO and s[2] == tc.HI and s[3] > tc.HI
    # every gate combination leaves the heads the reference leaves without a gradient
    nones = {tuple(gold[n + "/none"].tolist()) for n in tc.NAMES}
    assert len(nones) >= 5
    # the exact case has gathered entries whose prediction equals the target
    cfg, batch, heads, _ = tc.case("exact", default_cfg("dla_34"))
    wh = heads[1][0].reshape(2, -1)[:, batch["ind"][0]].T
    assert (wh == batch["wh"][0]).all(axis=1).sum() >= 4


@pytest.mark.parametrize("key, value", [("MSE_LOSS", True), ("DENSE_HP", True), ("REG_LOSS", "sl1")])
def test_refuses_what_val_refuses(key, value):
    cfg = default_cfg("dla_34")
    cfg.LOSS[key] = value
    with pytest.raises(NotImplementedError):
        train_loss.MultiPoseLoss(cfg)


def test_refuses_stacks_and_oracles():
    cfg = default_cfg("dla_34")
    cfg.MODEL.NUM_STACKS = 2
    with pytest.raises(NotImplementedError):
        train_loss.MultiPoseLoss(cfg, 0)
    cfg = default_cfg("dla_34")
    cfg.TEST.EVAL_ORACLE_HM = True
    with pytest.raises(NotImplementedError):
        train_loss.MultiPoseLoss(cfg, 0)


def test_refuses_bad_inputs():
    cfg, batch, heads, _ = tc.case("rot_image", default_cfg("dla_34"))
    crit = train_loss.MultiPoseLoss(cfg)
    assert list(crit.parameters()) == []
    tb = {k: torch.from_numpy(v) for k, v in batch.items()}
    th = [torch.from_numpy(h) for h in heads]
    with pytest.raises(ValueError, match="CUDA float32"):
        crit(th, tb)                                              # CPU heads
    with pytest.raises(ValueError, match="six head maps"):
        crit(th[:5], tb)


def _struct_fields(hdr, name):
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (name, name), hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = []
    for decl in body.split(";"):
        decl = re.sub(r"\bconst\b", "", decl).strip()
        if decl:
            fields += [re.sub(r"[\s*]", "", f) for f in decl.split(None, 1)[1].replace("*", " ").split(",")]
    return fields


def test_c_abi_structs_and_signatures():
    from centerpose_b200 import _lib
    hdr = open(os.path.join(ROOT, "include", "centerpose_b200.h")).read()
    for cls, name in ((_lib.Heads, "cpb200_multi_pose_heads"), (_lib.Targets, "cpb200_multi_pose_targets"),
                      (_lib.LossCfg, "cpb200_multi_pose_loss_cfg")):
        assert [f for f, _ in cls._fields_] == _struct_fields(hdr, name), name
    assert ctypes.sizeof(_lib.Heads) == 6 * 8 and ctypes.sizeof(_lib.Targets) == 11 * 8
    assert ctypes.sizeof(_lib.LossCfg) == 8 * 4
    for fn, n in (("cpb200_multi_pose_loss_train_batch", 9), ("cpb200_multi_pose_loss_train_backward", 9),
                  ("cpb200_multi_pose_loss_train_workspace_bytes", 1)):
        decl = re.search(r"\b%s\((.*?)\);" % fn, hdr, re.S).group(1)
        assert len(decl.split(",")) == n, fn
    if os.path.exists(_lib.LIBPATH):
        L = _lib.lib()
        assert len(L.cpb200_multi_pose_loss_train_batch.argtypes) == 9
        assert len(L.cpb200_multi_pose_loss_train_backward.argtypes) == 9
        assert L.cpb200_multi_pose_loss_train_workspace_bytes(32) == 8 * 3 * 18 * 32 + 4 * 6
