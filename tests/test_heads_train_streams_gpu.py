"""The training heads' entry points (include/centerpose_b200_heads_train.h) put all their work on the caller's stream:
each case of tests/heads_train_cases.STREAM_CASES runs through tests/test_streams_gpu.py's held-stream harness, with
its own stream held behind a spin kernel and again with the default stream held, and must give the default-stream
result bit for bit with every output overwritten in full."""
import pytest
import torch

from tests.heads_train_cases import STREAM_CASES
from tests.test_streams_gpu import DEV, Case, check_held

pytestmark = pytest.mark.gpu


def _heads_train_case(dev, precision):
    from centerpose_b200 import heads_train
    from tests.heads_train_cases import make_inputs
    x, params, gos = make_inputs(2, 24, 9, 11, 40, seed=6)

    def call(ins, alloc):
        leaves = [t.requires_grad_(True) for t in ins[:25]]
        outs = heads_train._Heads.apply(precision, *leaves)
        torch.autograd.backward(outs, ins[25:])
        return [o.detach() for o in outs] + [t.grad for t in leaves]
    return Case([t.to(dev) for t in [x] + params + gos], call)


BUILD = {"heads_train_default": lambda dev: _heads_train_case(dev, "default"),
         "heads_train_fp32": lambda dev: _heads_train_case(dev, "fp32")}


def test_every_case_has_a_builder():
    assert set(BUILD) == set(STREAM_CASES)


@pytest.mark.parametrize("name", sorted(BUILD))
def test_entry_point_on_held_stream(name):
    check_held(BUILD[name](DEV), DEV)
