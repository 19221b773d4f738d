"""CPU tests of the training DCNv2: the backward restatements against each other, torchvision and the golden fixture;
the module structure against the reference's dcn_v2.py (where the reference tree is mounted); ``install_ext``; the
refusals of ``centerpose_b200.dcn``; and the C ABI's symbols in the built library."""
import os
import sys

import numpy as np
import pytest
import torch

from centerpose_b200 import dcn
from oracle import make_golden_dcn_train as mg

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dcn_train.npz")
CFG = (3, 3, 1, 1, 1, 1, 1, 1, 1)
INPUTS = ("input", "weight", "bias", "offset", "mask", "grad_out")


def _case(name):
    z = np.load(GOLD)
    return {k: z[name + "/" + k] for k in INPUTS}, {k: z[name + "/" + k] for k in ("out",) + mg.GRADS}


@pytest.mark.parametrize("name", mg.NAMES)
def test_restatements_agree_with_golden(name):
    """Literal loops == golden; vectorised float64 autograd and torchvision's float64 backward within rounding."""
    c, gold = _case(name)
    mg.check_close(name + " literal", mg.literal(c), gold, rtol=0.0)
    mg.check_close(name + " vectorised", mg.vectorised(c), gold)
    mg.check_close(name + " torchvision", mg.torchvision_f64(c), gold, skip={"grad_offset": mg.on_minus_one(c)})


@pytest.mark.parametrize("name", mg.NAMES)
def test_golden_inputs_are_the_constructed_cases(name):
    c, _ = _case(name)
    made = mg.make_case(name)
    for k in INPUTS:
        assert np.array_equal(made[k], c[k]), k


def test_edges_case_reaches_every_sampling_case():
    c, _ = _case("edges")
    B, _, H, W = c["input"].shape
    hb, wb = mg._base(H, W)
    h = hb + c["offset"][:, 0::2].astype(np.float64)
    for v in (-1.0, H - 1, H):
        assert (h == v).any(), v
    assert ((h > -1) & (h < 0)).any() and ((h > H - 1) & (h < H)).any() and (h > H + 1).any() and (h < -2).any()
    assert ((h < 0) & (np.trunc(h) != np.floor(h)) & (h > -1)).any()
    assert (c["mask"] == 0).any()


def test_pile_case_piles_samples():
    c, _ = _case("pile")
    B, _, H, W = c["input"].shape
    hb, wb = mg._base(H, W)
    pos = {(float(a), float(b)) for a, b in zip((hb + c["offset"][:, 0::2]).ravel(),
                                                 (wb + c["offset"][:, 1::2]).ravel())}
    assert len(pos) <= 4


def test_reference_module_structure():
    from oracle import ref_harness
    if not ref_harness.reference_available():
        pytest.skip("reference tree not mounted")
    mg.check_reference_module()


def test_install_ext_registers_module():
    old = sys.modules.get("_ext")
    try:
        ext = dcn.install_ext()
        assert sys.modules["_ext"] is ext
        for n in ("dcn_v2_forward", "dcn_v2_backward", "dcn_v2_psroi_pooling_forward",
                  "dcn_v2_psroi_pooling_backward"):
            assert callable(getattr(ext, n)), n
        with pytest.raises(NotImplementedError):
            ext.dcn_v2_psroi_pooling_forward(None)
        with pytest.raises(ValueError):
            dcn.install_ext("fp16")
    finally:
        if old is None:
            sys.modules.pop("_ext", None)
        else:
            sys.modules["_ext"] = old


def _tensors(device="cpu", dtype=torch.float32, C=4, Co=3, H=5, W=6, k=3):
    return (torch.zeros(2, C, H, W, dtype=dtype, device=device), torch.zeros(Co, C, k, k, dtype=dtype, device=device),
            torch.zeros(Co, dtype=dtype, device=device), torch.zeros(2, 2 * k * k, H, W, dtype=dtype, device=device),
            torch.zeros(2, k * k, H, W, dtype=dtype, device=device))


def test_refuses_cpu_tensors():
    with pytest.raises(RuntimeError, match="CUDA"):
        dcn.dcn_v2_forward(*_tensors(), *CFG)
    x = _tensors()
    with pytest.raises(RuntimeError, match="CUDA"):
        dcn.dcn_v2_backward(*x, torch.zeros(2, 3, 5, 6), *CFG)


def test_refuses_other_dtypes(monkeypatch):
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    for dt in (torch.float16, torch.float64):
        with pytest.raises(ValueError, match="float32"):
            dcn.dcn_v2_forward(*_tensors(device="meta", dtype=dt), *CFG)


def test_refusals_before_the_device(monkeypatch):
    """The shape and configuration checks, on tensors that claim to be CUDA tensors (no device needed)."""
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    x = _tensors(device="meta")
    with pytest.raises(RuntimeError, match=r"kernel shape wont match: \(5 x 5 vs 3 x 3\)"):
        dcn.dcn_v2_forward(*x, 5, 5, 1, 1, 1, 1, 1, 1, 1)
    bad = list(x); bad[1] = torch.zeros(3, 5, 3, 3, device="meta")
    with pytest.raises(RuntimeError, match=r"kernel channels wont match: \(4 vs 5\)"):
        dcn.dcn_v2_forward(*bad, *CFG)
    for i, name in ((2, "stride"), (4, "padding"), (6, "dilation"), (8, "deformable_groups")):
        cfg = list(CFG); cfg[i] = 2
        with pytest.raises(NotImplementedError, match=name):
            dcn.dcn_v2_forward(*x, *cfg)
    k5 = _tensors(device="meta", k=5)
    with pytest.raises(NotImplementedError, match="kernel_size"):
        dcn.dcn_v2_forward(*k5, 5, 5, 1, 1, 1, 1, 1, 1, 1)
    with pytest.raises(ValueError, match="precision"):
        dcn.dcn_v2_forward(*x, *CFG, precision="bf16")


def test_split_rule_matches_library_and_cases_reach_every_regime():
    """The weight gradient's split K restated in tests/dcn_train_cases.py gives the library's split count (its
    workspace holds one Co x C*9 fp32 partial per split) on every accuracy case, and the cases reach every regime of
    the rule, from one K step per split to single splits of several steps and splits of hundreds of steps."""
    from centerpose_b200 import _lib
    from tests import dcn_train_cases as dc
    L = _lib.lib()
    reached = set()
    for B, C, Co, H, W in dc.ACCURACY:
        splits, steps = dc.wgrad_split(B, C, H, W, Co)
        assert L.cpb200_dcn_train_workspace_bytes(B, C, H, W, Co) == splits * Co * C * 9 * 4, (B, C, Co, H, W)
        assert (splits - 1) * steps < -(-B * H * W // dc.BK) <= splits * steps, (B, C, Co, H, W)
        reached |= dc.split_regimes(B, C, H, W, Co)
    assert reached == set(dc.REGIMES), set(dc.REGIMES) - reached
    assert dc.split_regimes(32, 64, 128, 128, 64) >= {"over 400 steps per split", "short last split",
                                                      "split boundary inside an image"}
    assert dc.wgrad_split(32, 64, 128, 128, 64) == (53, 619)


def test_modules_match_reference_layout():
    torch.manual_seed(3)
    m = dcn.DCN(40, 24, kernel_size=(3, 3), stride=1, padding=1, dilation=1, deformable_groups=1)
    sd = m.state_dict()
    assert list(sd) == ["weight", "bias", "conv_offset_mask.weight", "conv_offset_mask.bias"]
    assert sd["weight"].shape == (24, 40, 3, 3) and sd["conv_offset_mask.weight"].shape == (27, 40, 3, 3)
    bound = 1 / np.sqrt(40 * 9)
    assert sd["weight"].abs().max() <= bound and sd["weight"].abs().max() > 0.9 * bound
    assert not sd["bias"].any() and not sd["conv_offset_mask.weight"].any() and not sd["conv_offset_mask.bias"].any()
