"""The fused decode kernel on the constructed cases of tests/decode_cases.py: every case's (B, K, 5+3J) rows equal the
oracle's bit for bit (the kernel follows the oracle's fp32 operation order, so no tolerance is needed), the fused
back-projection stays within the 2e-3 px of test_decode_fused_post_process, and the fused logistic gives the same rows
whichever scan path reads the logits."""
import numpy as np
import pytest
import torch

from oracle import decode_ref
from tests.decode_cases import CASE, Inputs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _dev(a, misaligned):
    a = np.ascontiguousarray(a)
    if not misaligned:
        return torch.from_numpy(a).to(DEV)
    flat = torch.empty(a.size + 1, dtype=torch.float32, device=DEV)
    t = flat[1:].view(a.shape)                  # contiguous, 4 bytes past a 16-byte boundary
    t.copy_(torch.from_numpy(a))
    assert t.data_ptr() % 16 == 4
    return t


def _run(inp: Inputs, apply_sigmoid=False, affine=None):
    from centerpose_b200 import multi_pose_decode
    t = {k: _dev(v, inp.misaligned) for k, v in inp.maps.items()}
    out = multi_pose_decode(t["heat"], t["wh"], t["kps"], reg=t["reg"] if inp.use_reg else None, hm_hp=t["hm_hp"],
                            hp_offset=t["hp_offset"] if inp.use_off else None, K=inp.K, apply_sigmoid=apply_sigmoid,
                            affine=affine)
    torch.cuda.synchronize()
    return out.cpu().numpy()


def _oracle(inp: Inputs, b=None):
    d = {k: (v if b is None else v[b:b + 1]) for k, v in inp.maps.items()}
    return decode_ref.multi_pose_decode(d["heat"], d["wh"], d["kps"], d["reg"] if inp.use_reg else None, d["hm_hp"],
                                        d["hp_offset"] if inp.use_off else None, K=inp.K)


def _assert_bit_exact(got, want, what=""):
    assert got.shape == want.shape, (got.shape, want.shape)
    if np.array_equal(got, want):
        return
    bad = np.argwhere(got != want)
    b, r, c = bad[0]
    raise AssertionError(f"{what}{len(bad)} values differ; first at image {b} row {r} column {c}: kernel "
                         f"{got[b, r, c]!r}, oracle {want[b, r, c]!r}; kernel row {got[b, r].tolist()}, "
                         f"oracle row {want[b, r].tolist()}")


@pytest.mark.parametrize("name", list(CASE))
def test_case_matches_oracle_bit_exact(name):
    inp = CASE[name].build()
    got = _run(inp)
    for b in range(got.shape[0]):             # each image against the oracle run on that image alone
        _assert_bit_exact(got[b:b + 1], _oracle(inp, b), f"image {b}: ")


def test_workspace_returns_to_zero_between_batches():
    """B = 48 (864 CTAs), then B = 3, then B = 48 again on the same stream: the per-image sync words of the reused
    workspace must be back at zero, or the second B = 48 call's joint CTAs would group against stale centre rows"""
    inp = CASE["batch_48"].build()
    first = _run(inp)
    small = Inputs({k: v[:3].copy() for k, v in inp.maps.items()}, inp.K)
    _assert_bit_exact(_run(small), first[:3])
    _assert_bit_exact(_run(inp), first)


@pytest.mark.parametrize("name", ["sqrttie", "box_and_distance_edges", "tie_across_halves", "fill_few_9x13",
                                  "segment_overflow"])
def test_case_affine_matches_post_process(name):
    from centerpose_b200.decode import affine_for_meta
    from oracle import post_process_ref
    inp = CASE[name].build()
    B = inp.shape[0]
    sizes = [(480, 640), (1080, 1920), (333, 500)]
    metas = [post_process_ref.make_meta(*sizes[b % 3], 1.0, True) for b in range(B)]
    got = _run(inp, affine=affine_for_meta(metas).to(DEV))
    ref = _oracle(inp)
    for b in range(B):
        want = post_process_ref.multi_pose_post_process(ref[b:b + 1].copy(), [metas[b]["c"]], [metas[b]["s"]],
                                                        metas[b]["out_height"], metas[b]["out_width"])[0][1]
        assert np.abs(got[b] - want).max() <= 2e-3, np.abs(got[b] - want).max()


def _logits(kind):
    """16x128 logits: 'peaks' uniform in [-3, 3) (every cell > 0 after the logistic, ~1/9 of them peaks: more than K
    centre peaks, so no zero fill); 'ties' one constant logit (every cell ties: select_slow)"""
    d = decode_ref.synth_decode_inputs(1, 16, 128, seed=91, kind="smooth")
    rng = np.random.RandomState(92)
    for k, C in (("heat", 1), ("hm_hp", 17)):
        d[k] = (rng.uniform(-3, 3, size=(1, C, 16, 128)) if kind == "peaks" else np.full((1, C, 16, 128), 0.7)
                ).astype(np.float32)
    return d


@pytest.mark.parametrize("kind", ["peaks", "ties"])
def test_fused_sigmoid_same_rows_on_every_scan_path(kind):
    """apply_sigmoid=True cannot match the oracle bit for bit (the kernel's logistic uses __expf), but every scan path
    applies the same logistic: scan_w128<true> on 16x128, scan_vec on the same map with a 17th row of -1e30 logits
    (logistic 0: no peak, and no flat index moves), scan_scalar on a misaligned view.  'ties' runs select_slow."""
    d = _logits(kind)
    K = 100
    base = _run(Inputs(d, K), apply_sigmoid=True)
    tall = {k: np.concatenate([v, np.zeros_like(v[:, :, :1])], axis=2) for k, v in d.items()}
    tall["heat"][:, :, 16] = -1e30
    tall["hm_hp"][:, :, 16] = -1e30
    _assert_bit_exact(_run(Inputs(tall, K), apply_sigmoid=True), base, "17-row scan_vec vs scan_w128: ")
    _assert_bit_exact(_run(Inputs(d, K, misaligned=True), apply_sigmoid=True), base, "scan_scalar vs scan_w128: ")
    if kind == "peaks":
        assert (base[0, :, 4] > 0).all()
