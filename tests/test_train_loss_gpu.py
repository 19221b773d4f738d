"""GPU tests of the trainer's loss (train_loss.MultiPoseLoss: cpb200_multi_pose_loss_train_batch / _backward) against
the reference's MultiPoseLoss and backward (tests/golden/train_loss.npz), and against the torch restatement's autograd
on the device (oracle/train_loss_ref.py) on TrainData batches of seeded JPEG files.

Bounds:
* stats: 1e-5 relative to the reference, and 2 float32 ulp of the float64 restatement (``val.loss``'s bounds);
* regression gradients: every entry adds +c, -c or 0 to its pixel, and the kernel writes count * c rounded once.
  Torch's first two additions are exact (c + c, c - c, c + 0), so wherever at most three entries meet at a pixel its
  sum is the same single rounding of count * c: bit-equal.  Where k > 3 meet, each later partial sum is rounded by at
  most half an ulp of k * |c|, so the two differ by at most (k - 1) / 2 ulp of k * |c|;
* focal gradients: |device - float64 chain| within ``train_loss_ref.focal_grad64``'s per-element bound, which
  propagates every float32 rounding and CUDA's stated 2 ulp ``expf`` / 1 ulp ``logf`` errors through the chain.
  Where the logistic is within its error of a clamp bound the device must take the reference's side: 0 or not.
"""
import copy
import os

import numpy as np
import pytest
import torch

from centerpose_b200 import train_loss
from centerpose_b200.config import default_cfg
from oracle import train_loss_ref
from tests import train_loss_cases as tc
from tests.train_cases import seeded_jpeg_batch

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_loss.npz")
HEADS = train_loss_ref.HEADS
DEV = torch.device("cuda:0")


def _ulp2(got, want):
    got, want = np.float32(got), np.float32(want)
    return np.abs(got.astype(np.float64) - want) <= 2 * np.spacing(np.abs(want)).astype(np.float64)


def meet_counts(batch, h):
    """Per element of regression map ``h`` (flat (B, C, R, R)), how many gathered entries with m != 0 reach it."""
    B, R = batch["hm"].shape[0], batch["hm"].shape[-1]
    ind, mask, C = {"wh": ("ind", "reg_mask", 2), "reg": ("ind", "reg_mask", 2), "hps": ("ind", "hps_mask", 2 * tc.J),
                    "hp_offset": ("hp_ind", "hp_mask", 2)}[h]
    ind, mask = np.asarray(batch[ind]), np.asarray(batch[mask])
    n = ind.shape[1]
    m = mask if mask.ndim == 3 else np.repeat(mask[:, :, None], C, axis=2)
    b, k, c = np.meshgrid(np.arange(B), np.arange(n), np.arange(C), indexing="ij")
    flat = ((b * C + c) * R * R + ind[b, k]).reshape(-1)
    counts = np.zeros(B * C * R * R, np.int64)
    np.add.at(counts, flat[(m != 0).reshape(-1)], 1)
    return counts


def term_c(batch, h, cfg, grad_out):
    """c = (grad_out * weight) / (sum(m) + 1e-4) of regression term ``h``, in float32 as torch computes it."""
    c = cfg.LOSS
    w = {"wh": c.WH_WEIGHT, "reg": c.OFF_WEIGHT, "hps": c.HP_WEIGHT, "hp_offset": c.OFF_WEIGHT}[h]
    den = np.float32(np.float32(meet_counts(batch, h).sum()) + np.float32(1e-4))
    return np.float32(np.float32(np.float32(grad_out) * np.float32(w)) / den)


def check_regression(got, want, counts, c, what):
    got, want = got.reshape(-1), want.reshape(-1)
    few = counts <= 3
    assert np.array_equal(got[few], want[few]), (what, int((got[few] != want[few]).sum()))
    k = counts[~few]
    tol = (k - 1) / 2 * np.spacing(np.float32(k * abs(float(c)))).astype(np.float64)
    assert (np.abs(got[~few].astype(np.float64) - want[~few]) <= tol).all(), what


def check_focal(got, x, gt, grad_out, weight, npos, ref, what):
    """``got`` within the float64 chain's bound; on clamp edges the same side (0 or not) as ``ref``."""
    v, bound, edge = train_loss_ref.focal_grad64(x, gt, grad_out, weight, npos)
    ok = (np.abs(got.astype(np.float64) - v) <= bound) | edge
    assert ok.all(), (what, int((~ok).sum()))
    if ref is not None:
        assert np.array_equal(got[edge] == 0, ref[edge] == 0), what
    return np.max(np.abs(got - v)[~edge] / np.maximum(np.spacing(np.abs(v[~edge]).astype(np.float32)), 1e-45),
                  initial=0)


def run_device(cfg, batch, heads, grad_out):
    leaves = [h.detach().clone().requires_grad_(True) for h in heads]
    loss, st = train_loss.MultiPoseLoss(cfg, 0)(leaves, batch)
    assert loss.dim() == 0 and loss.grad_fn is not None
    assert set(st) == set(train_loss_ref.STATS) and all(v.dim() == 0 and v.is_cuda for v in st.values())
    (grad_out * loss).backward() if grad_out != 1 else loss.backward()
    stats = np.array([st[k].item() for k in train_loss_ref.STATS], np.float32)
    return loss, stats, leaves


def run_restated(cfg, batch, heads, grad_out):
    leaves = [h.detach().clone().requires_grad_(True) for h in heads]
    loss, st = train_loss_ref.loss_torch(leaves, batch, cfg.LOSS)
    loss.backward(torch.tensor(grad_out, device=loss.device))
    return np.array([float(st[k].detach()) for k in train_loss_ref.STATS], np.float32), leaves


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLD))


@pytest.mark.parametrize("name", tc.NAMES)
def test_matches_golden(gold, name):
    cfg, batch, heads, grad_out = tc.case(name, default_cfg("dla_34"))
    key = name + "/"
    db = {k: torch.from_numpy(v).to(DEV) for k, v in batch.items()}
    dh = [torch.from_numpy(h).to(DEV) for h in heads]
    _, stats, leaves = run_device(cfg, db, dh, grad_out)
    want = gold[key + "stats"]
    assert np.all(np.abs(stats - want) <= 1e-5 * np.abs(want)), (stats, want)
    assert _ulp2(stats, train_loss_ref.stats64(heads, batch, cfg.LOSS)).all()
    assert [x.grad is None for x in leaves] == gold[key + "none"].tolist()
    for h, x, leaf in zip(HEADS, heads, leaves):
        assert np.array_equal(leaf.detach().cpu().numpy(), x), h               # the maps are left as they are
        if leaf.grad is None:
            continue
        g = leaf.grad.cpu().numpy()
        idx, val = gold[key + h + "_idx"], gold[key + h + "_val"]
        if h in ("hm", "hm_hp"):
            c = cfg.LOSS
            ref = np.zeros(g.size, np.float32)
            ref[idx] = val
            sel = np.zeros(g.size, bool)
            sel[idx] = True
            check_focal(g.reshape(-1)[sel], x.reshape(-1)[sel], batch[h].reshape(-1)[sel], grad_out,
                        c.HM_WEIGHT if h == "hm" else c.HM_HP_WEIGHT, float((batch[h] == 1).sum()), ref[sel],
                        (name, h))
        else:
            ref = np.zeros(g.size, np.float32)
            ref[idx] = val
            check_regression(g, ref, meet_counts(batch, h), term_c(batch, h, cfg, grad_out), (name, h))


def test_clamp_edges_reach_both_sides(gold):
    """The clamp-edge logits: the positives and negatives at the bounds pass a gradient, those beyond get exactly 0."""
    cfg, batch, heads, grad_out = tc.case("clamp_edges", default_cfg("dla_34"))
    db = {k: torch.from_numpy(v).to(DEV) for k, v in batch.items()}
    _, _, leaves = run_device(cfg, db, [torch.from_numpy(h).to(DEV) for h in heads], grad_out)
    g = leaves[0].grad.cpu().numpy()
    for i in range(3):
        for row in (i, i + 3):
            assert g[i, 0, row, 0] != 0 and g[i, 0, row, 1] == 0 and g[i, 0, row, 2] != 0 and g[i, 0, row, 3] == 0


@pytest.fixture(scope="module")
def jpeg_batch(tmp_path_factory):
    return seeded_jpeg_batch(tmp_path_factory.mktemp("train_loss"))


def test_train_batches_match_restatement(jpeg_batch):
    cfg, batch = jpeg_batch
    B, R = batch["hm"].shape[0], batch["hm"].shape[-1]
    assert (B, R) == (32, 128)
    heads_np = tc.logits(31, B, R)
    heads = [torch.from_numpy(h).to(DEV) for h in heads_np]
    _, stats, leaves = run_device(cfg, batch, heads, 1.0)
    want, ref = run_restated(cfg, batch, heads, 1.0)
    assert np.all(np.abs(stats - want) <= 1e-5 * np.abs(want)), (stats, want)
    bnp = {k: v.cpu().numpy() for k, v in batch.items() if k != "input"}
    assert _ulp2(stats, train_loss_ref.stats64(heads_np, bnp, cfg.LOSS)).all()
    worst = {}
    for h, x, leaf, r in zip(HEADS, heads_np, leaves, ref):
        assert np.array_equal(leaf.detach().cpu().numpy(), x), h
        g, rg = leaf.grad.cpu().numpy(), r.grad.cpu().numpy()
        if h in ("hm", "hm_hp"):
            npos = float((bnp[h] == 1).sum())
            w = cfg.LOSS.HM_WEIGHT if h == "hm" else cfg.LOSS.HM_HP_WEIGHT
            for b in range(B):                     # image by image: the float64 chain holds ~60 temporaries
                worst[h] = max(worst.get(h, 0), check_focal(g[b], x[b], bnp[h][b], 1.0, w, npos, rg[b], (h, b)))
                check_focal(rg[b], x[b], bnp[h][b], 1.0, w, npos, None, ("torch", h, b))
        else:
            check_regression(g, rg, meet_counts(bnp, h), term_c(bnp, h, cfg, 1.0), h)
    print("worst focal gradient error against the float64 chain, in ulp:", worst)


def test_deterministic_and_grad_output(jpeg_batch):
    cfg, batch = jpeg_batch
    B, R = batch["hm"].shape[0], batch["hm"].shape[-1]
    heads = [torch.from_numpy(h).to(DEV) for h in tc.logits(32, B, R)]
    _, _, a = run_device(cfg, batch, heads, 1.0)
    _, _, b = run_device(cfg, batch, heads, 1.0)
    for x, y in zip(a, b):
        assert torch.equal(x.grad.view(torch.int32), y.grad.view(torch.int32))
    # grad_output != 1 against the restatement's autograd
    _, _, s = run_device(cfg, batch, heads, 3.5)
    _, ref = run_restated(cfg, batch, heads, 3.5)
    bnp = {k: v.cpu().numpy() for k, v in batch.items() if k != "input"}
    for h, x, r in zip(HEADS, s, ref):
        if h not in ("hm", "hm_hp"):
            check_regression(x.grad.cpu().numpy(), r.grad.cpu().numpy(), meet_counts(bnp, h), term_c(bnp, h, cfg, 3.5),
                             h)
    # a loss summed with another term, and retain_graph: two backwards accumulate twice the gradient
    leaves = [h.detach().clone().requires_grad_(True) for h in heads]
    loss, _ = train_loss.MultiPoseLoss(cfg, 0)(leaves, batch)
    total = loss + leaves[1].sum() * 0
    total.backward(retain_graph=True)
    once = [x.grad.clone() for x in leaves]
    total.backward()
    for x, o, y in zip(leaves, once, a):
        assert torch.equal(o, y.grad) and torch.equal(x.grad, 2 * o)


def test_gates_and_refusals(jpeg_batch):
    cfg, batch = jpeg_batch
    B, R = batch["hm"].shape[0], batch["hm"].shape[-1]
    heads = [torch.from_numpy(h).to(DEV) for h in tc.logits(33, B, R)]
    for _, over in tc.GATES:
        c = copy.deepcopy(cfg)
        c.LOSS.update(over)
        keys = tc.gate_keys(c.LOSS)
        _, _, leaves = run_device(c, {k: batch[k] for k in keys}, heads, 1.0)
        assert [x.grad is None for x in leaves] == [not on for on in train_loss.head_gates(c)], over
    crit = train_loss.MultiPoseLoss(cfg, 0)
    short = {k: v for k, v in batch.items() if k != "hp_mask"}
    with pytest.raises(ValueError, match="no target 'hp_mask'"):
        crit(heads, short)
    with pytest.raises(ValueError, match="CUDA float32"):
        crit([h.half() for h in heads], batch)
    bad = dict(batch)
    bad["ind"] = batch["ind"].int()
    with pytest.raises(ValueError, match="target 'ind'"):
        crit(heads, bad)


class Tiny(torch.nn.Module):
    """batch['input'] (B, 3, S, S) -> the six heads at S / 4."""

    def __init__(self):
        super().__init__()
        torch.manual_seed(5)
        self.pool = torch.nn.AvgPool2d(4)
        self.conv = torch.nn.Conv2d(3, 16, 3, padding=1)
        self.head = torch.nn.Conv2d(16, sum(tc.HEAD_CHANNELS), 1)
        with torch.no_grad():
            self.head.bias[0] = -2.19
            self.head.bias[39:56] = -2.19

    def forward(self, x):
        y = self.head(torch.relu(self.conv(self.pool(x))))
        return list(torch.split(y, list(tc.HEAD_CHANNELS), dim=1))


def test_short_training_loop(tmp_path):
    """Five Adam steps on the same five TrainData batches, with the device loss and with the restatement: the
    parameters agree within 1e-4 (1 % of one step at lr 1e-2), and the loss on the first batch falls in both."""
    batches = [seeded_jpeg_batch(tmp_path, B=8, res=128, seed=s) for s in range(5)]
    cfg = batches[0][0]
    runs = []
    for use_device in (True, False):
        model = Tiny().to(DEV)
        opt = torch.optim.Adam(model.parameters(), lr=1e-2)
        crit = train_loss.MultiPoseLoss(cfg, 0)
        loss_fn = (lambda o, b: crit(o, b)) if use_device else (lambda o, b: train_loss_ref.loss_torch(o, b, cfg.LOSS))
        losses = []
        for _, batch in batches:
            loss, _ = loss_fn(model(batch["input"]), batch)
            opt.zero_grad()
            loss.backward()
            opt.step()
            losses.append(loss.item())
        with torch.no_grad():
            losses.append(loss_fn(model(batches[0][1]["input"]), batches[0][1])[0].item())
        runs.append(([p.detach().clone() for p in model.parameters()], losses))
    (pa, la), (pb, lb) = runs
    assert la[-1] < la[0] and lb[-1] < lb[0], (la, lb)
    assert np.allclose(la, lb, rtol=1e-4), (la, lb)
    for x, y in zip(pa, pb):
        assert (x - y).abs().max().item() <= 1e-4
