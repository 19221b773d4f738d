"""The video path's drawing-plan entry points (include/centerpose_b200_video.h) put all their work on the caller's
stream: each case of tests/video_cases.STREAM_CASES runs through tests/test_streams_gpu.py's held-stream harness, with
its own stream held behind a spin kernel and again with the default stream held, and must give the default-stream
result bit for bit.  Both write their tables only in part by design (a polygon's points, the persons an image draws),
so their outputs are zero-filled in every leg."""
import numpy as np
import pytest
import torch

from tests.test_streams_gpu import DEV, KEEP, Case, check_held
from tests.video_cases import STREAM_CASES

pytestmark = pytest.mark.gpu


def _ellipse_case(dev):
    from centerpose_b200 import _lib
    rng = np.random.default_rng(4)
    n = 300
    params = np.stack([rng.integers(-50, 400, n), rng.integers(-50, 300, n), rng.integers(0, 400, n),
                       rng.integers(-180, 181, n)], 1).astype(np.int32)

    def call(ins, alloc):
        verts = alloc((n, 361, 2), torch.int32, poison=False)
        counts = alloc((n,), torch.int32)
        _lib.launch("ellipse_poly_batch", DEV, ins[0], n, verts, counts)
        return [verts, counts]
    return Case([torch.from_numpy(params).to(dev)], call, decoys=[KEEP])


def _plan_case(dev):
    from centerpose_b200 import _lib, render
    from tests import render_cases as rc
    h, w, B, N = 120, 160, 3, 12
    rows = np.stack([np.concatenate([rc.rows(h, w, N - 8, 60 + b, off=0.3), rc.edge_rows(h, w)]) for b in range(B)])
    labels = torch.from_numpy(render.label_table(render.LABELS).view(np.uint8)).to(dev)
    sizes = [B * 40, B * N * 224, B * N * 18 * 24, B * 4096 * 8, B * N * 24, B * 16]

    def call(ins, alloc):
        out = [alloc((s,), torch.uint8, poison=False) for s in sizes]
        _lib.launch("render_plan_batch", DEV, ins[0], B, N, h, w, 0.3, 0x8080FF, ins[1], render.LABELS, 4096,
                    1 << 16, *out)
        return out
    return Case([torch.from_numpy(rows).to(dev), labels], call, decoys=[None, KEEP])


BUILD = {"ellipse_poly": _ellipse_case, "render_plan": _plan_case}


def test_every_case_has_a_builder():
    assert set(BUILD) == set(STREAM_CASES)


@pytest.mark.parametrize("name", sorted(BUILD))
def test_entry_point_on_held_stream(name):
    check_held(BUILD[name](DEV), DEV)
