"""CPU tests of the training keypoint heads (centerpose_b200.heads_train): the module against the reference's
KeypointHead (tests/golden/heads_train_init.npz), the C ABI's prototypes, the backward's workspace rule and the
refusals before any library call."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from centerpose_b200 import heads_train
from tests import heads_train_cases as hc_cases

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "heads_train_init.npz")


def test_module_matches_reference_init():
    """Same state_dict keys in order, named_parameters() order, shapes and, from the same seed, the same values."""
    z = np.load(GOLD)
    torch.manual_seed(int(z["seed"]))
    m = heads_train.KeypointHead(int(z["C"]), int(z["hc"]))
    sd = m.state_dict()
    assert list(sd) == list(z["keys"])
    assert [n for n, _ in m.named_parameters()] == list(z["params"])
    for k, v in sd.items():
        want = z["value/" + k]
        assert tuple(v.shape) == want.shape, k
        assert np.array_equal(v.numpy(), want), k
    assert [id(p) for p in m.head_parameters()] == [id(p) for p in m.parameters()]


def _heads_header():
    from centerpose_b200 import _lib
    with open(_lib.HEADS_TRAIN_HEADER) as f:
        return f.read()


def test_prototypes_bind():
    """The three prototypes of include/centerpose_b200_heads_train.h parse, are exported and are bound as declared."""
    from centerpose_b200 import _lib
    text = _heads_header()
    sigs = _lib.signatures(text)
    code = re.sub(r"/\*.*?\*/|//[^\n]*", " ", text, flags=re.S)
    assert set(sigs) == set(re.findall(r"\b(cpb200_[a-z0-9_]+)\s*\(", code))
    assert set(sigs) == {"cpb200_heads_train_" + n for n in ("workspace_bytes", "forward", "backward")}
    assert not set(sigs) & set(_lib.signatures()), "declared in both public headers"
    I, P = ctypes.c_int, ctypes.c_void_p
    assert sigs["cpb200_heads_train_workspace_bytes"] == (ctypes.c_size_t, [I] * 5)
    assert sigs["cpb200_heads_train_forward"] == (I, [P] * 5 + [_lib.Heads] + [I] * 6 + [P])
    assert sigs["cpb200_heads_train_backward"] == (I, [P] * 4 + [_lib.Heads] + [P] * 5 + [I] * 6 +
                                                   [P, ctypes.c_size_t, P])
    L = _lib.lib()
    for n, (restype, argtypes) in sigs.items():
        fn = getattr(L, n)
        assert fn.restype is restype and list(fn.argtypes) == argtypes, n


def test_every_stream_entry_point_has_a_stream_case():
    """Every entry point of the heads header that takes a stream is held on a side stream by a case of
    tests/test_heads_train_streams_gpu.py, and the stream is its last parameter, as _lib.launch appends it."""
    from centerpose_b200 import _lib
    from tests.stream_cases import stream_entry_points
    declared = stream_entry_points(_heads_header())
    covered = {e for entries in hc_cases.STREAM_CASES.values() for e in entries}
    assert declared == covered, (sorted(declared), sorted(covered))
    sigs = _lib.signatures(_heads_header())
    for name in declared:
        assert sigs["cpb200_" + name][1][-1] is ctypes.c_void_p, name


def test_workspace_rule_matches_library():
    from centerpose_b200 import _lib
    L = _lib.lib()
    shapes = sorted(set(hc_cases.ALL_SHAPES))      # every shape tests/test_heads_train_gpu.py runs
    regimes = set()
    for B, C, H, W, hc in shapes:
        assert L.cpb200_heads_train_workspace_bytes(B, C, H, W, hc) == hc_cases.workspace_bytes(B, C, H, W, hc), \
            (B, C, H, W, hc)
        n = hc_cases.chunk_images(B, H, W, hc)
        if n == 1 and B > 1:
            regimes.add("one image per chunk")
        if 1 < n < B:
            regimes.add("several images per chunk")
        if n < B and B % n:
            regimes.add("short last chunk")
        if n == B:
            regimes.add("single chunk")
    assert regimes == {"one image per chunk", "several images per chunk", "short last chunk", "single chunk"}, regimes
    assert hc_cases.chunk_images(18, 128, 128, 256) == 2
    assert L.cpb200_heads_train_workspace_bytes(0, 8, 8, 8, 8) == 0


def _params(C=8, hc=16, device="cpu", dtype=torch.float32):
    torch.manual_seed(0)
    m = heads_train.KeypointHead(C, hc).to(device=device, dtype=dtype)
    return m.head_parameters()


def test_refuses_cpu_tensors():
    with pytest.raises(RuntimeError, match="CUDA"):
        heads_train.heads_forward(torch.zeros(1, 8, 4, 4), _params())
    m = heads_train.KeypointHead(8, 16)
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros(1, 8, 4, 4))


def test_refusals_before_the_device(monkeypatch):
    """Dtype, channel and precision checks on tensors that claim to be CUDA tensors (no device needed)."""
    monkeypatch.setattr(torch.Tensor, "is_cuda", property(lambda self: True))
    ps = _params(device="meta")
    for dt in (torch.float16, torch.float64):
        with pytest.raises(ValueError, match="float32"):
            heads_train.heads_forward(torch.zeros(1, 8, 4, 4, device="meta", dtype=dt), ps)
    with pytest.raises(RuntimeError, match="channels"):
        heads_train.heads_forward(torch.zeros(1, 5, 4, 4, device="meta"), ps)
    with pytest.raises(RuntimeError, match="channels"):
        heads_train.heads_backward(torch.zeros(1, 5, 4, 4, device="meta"), ps, [None] * 6)
    with pytest.raises(ValueError, match="precision"):
        heads_train.heads_forward(torch.zeros(1, 8, 4, 4, device="meta"), ps, precision="bf16")
    with pytest.raises(ValueError, match="precision"):
        heads_train.KeypointHead(8, 16, precision="tf32")
    gos = [torch.zeros(1, c, 4, 4, device="meta") for c in heads_train.OUTPUTS]
    gos[2] = torch.zeros(1, 3, 4, 4, device="meta")
    with pytest.raises(ValueError, match="grad_output hps"):
        heads_train.heads_backward(torch.zeros(1, 8, 4, 4, device="meta"), ps, gos)


def test_state_dict_round_trips_with_reference():
    """A state_dict of either module loads into the other (reference tree mounted)."""
    from oracle import ref_harness
    if not ref_harness.reference_available():
        pytest.skip("reference tree not mounted")
    from oracle import make_golden_heads_train as mg
    ref = mg.reference_module()
    torch.manual_seed(mg.SEED)
    mine = heads_train.KeypointHead(mg.C, mg.HC)
    ref.load_state_dict(mine.state_dict())
    mine.load_state_dict(ref.state_dict())
