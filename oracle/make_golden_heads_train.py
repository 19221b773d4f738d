"""Generate ``tests/golden/heads_train_init.npz``: the reference's ``KeypointHead`` (lib/models/heads/keypoint.py) as
constructed under a fixed seed, for ``centerpose_b200.heads_train.KeypointHead`` to match.

Run:  python -m oracle.make_golden_heads_train      (from the repo root, with the reference tree mounted)

The unmodified reference module is built at C = 8, hc = 16 after ``torch.manual_seed(SEED)``; the fixture holds its
state_dict keys in order (``keys``), its ``named_parameters()`` names in order (``params``) and every tensor's value
under its key (shapes travel with the values).  Before anything is written, the float64 restatement the tests use
(``heads_f64``: ``oracle.dla_ref.keypoint_head``, torch ``F.conv2d``) is checked against the reference module's own
autograd on the CPU: outputs and the gradients of x and of every parameter, for seeded x and grad_output.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from oracle import dla_ref

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "heads_train_init.npz")
C, HC, SEED = 8, 16, 2024


def heads_f64(params, x, prefix="head_model"):
    """The six maps of ``x`` through ``oracle.dla_ref.keypoint_head`` for ``params`` ({"hm.0.weight": ...})."""
    return dla_ref.keypoint_head({prefix + "." + k: v for k, v in params.items()}, x, prefix)


def reference_module():
    from oracle import ref_harness
    ref_harness.load_reference()
    from models.heads.keypoint import KeypointHead
    torch.manual_seed(SEED)
    return KeypointHead(C, HC)


def check_restatement(ref):
    """heads_f64 against the reference module's autograd, float64 on the CPU."""
    m = ref.double()
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, C, 7, 9, generator=g, dtype=torch.float64, requires_grad=True)
    outs = m(x)
    gos = [torch.randn(o.shape, generator=g, dtype=torch.float64) for o in outs]
    torch.autograd.backward(outs, gos)
    want = [o.detach() for o in outs] + [x.grad] + [p.grad for p in m.parameters()]
    names = [n for n, _ in m.named_parameters()]
    leaves = {n: p.detach().clone().requires_grad_(True) for n, p in m.named_parameters()}
    x2 = x.detach().clone().requires_grad_(True)
    got_outs = heads_f64(leaves, x2)
    torch.autograd.backward(got_outs, gos)
    got = [o.detach() for o in got_outs] + [x2.grad] + [leaves[n].grad for n in names]
    for i, (a, b) in enumerate(zip(got, want)):
        err = (a - b).abs().max().item()
        assert err <= 1e-12 * max(1.0, b.abs().max().item()), (i, err)
    print("float64 restatement == reference KeypointHead autograd: 6 outputs, grad x and %d parameter grads"
          % len(names))


def main():
    ref = reference_module()
    sd = ref.state_dict()
    arrays = {"keys": np.array(list(sd)), "params": np.array([n for n, _ in ref.named_parameters()]),
              "C": np.int64(C), "hc": np.int64(HC), "seed": np.int64(SEED)}
    for k, v in sd.items():
        arrays["value/" + k] = v.numpy().copy()
    check_restatement(ref)
    np.savez_compressed(OUT, **arrays)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
