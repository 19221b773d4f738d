"""The pre-process warp, flip merge and soft-NMS kernels of csrc/post.cu on the constructed cases of
tests/post_cases.py, each held to its reference exactly:

  * cpb200_pre_process and cpb200_pre_process_batch equal the integer warp model plus the float64 normalisation
    (torch.equal), write nothing outside their output, and mirror the copy exactly;
  * cpb200_flip_merge equals the torch restatement of the reference's flip merge, and refuses bad arguments without
    launching;
  * cpb200_soft_nms_39 and _batch leave each image's whole (N, 56) array and keep count equal to the host port, dead
    rows included, and agree with the reference's compiled Cython on the golden fixture.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

from tests import post_cases as pc

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
GOLD = os.path.join(os.path.dirname(__file__), "golden", "soft_nms_cases.npz")
CANARY = 1.5e38            # any kernel write into the guard bands replaces it


def _mean_std():
    return (ctypes.c_float * 3)(*pc.MEAN), (ctypes.c_float * 3)(*pc.STD)


def _guarded(n_out, guard=4096):
    buf = torch.full((guard + n_out + guard,), CANARY, dtype=torch.float32, device=DEV)
    return buf, buf[guard:guard + n_out]


def _check_guards(buf, n_out, guard=4096):
    assert bool((buf[:guard] == CANARY).all()) and bool((buf[guard + n_out:] == CANARY).all()), \
        "the kernel wrote outside its output"


def _pre_single(img, t, OH, OW, flip):
    from centerpose_b200 import _lib
    src = torch.from_numpy(np.ascontiguousarray(img)).to(DEV)
    n = (2 if flip else 1) * 3 * OH * OW
    buf, out = _guarded(n)
    M = (ctypes.c_double * 6)(*np.asarray(t, np.float64).reshape(6))
    mean, std = _mean_std()
    st = _lib.lib().cpb200_pre_process(src.data_ptr(), img.shape[0], img.shape[1], M, out.data_ptr(), OH, OW, mean, std,
                                       1 if flip else 0, torch.cuda.current_stream().cuda_stream)
    _lib.check(st, "pre_process")
    torch.cuda.synchronize()
    _check_guards(buf, n)
    return out.view(-1, 3, OH, OW).cpu()


def _pre_batch(images, trans, OH, OW, flip):
    from centerpose_b200 import _lib
    from centerpose_b200.detector import _PRE_IMAGE
    table = np.zeros(len(images), _PRE_IMAGE)
    pos = 0
    for n, (im, t) in enumerate(zip(images, trans)):
        table[n] = (pos, im.shape[0], im.shape[1], np.asarray(t, np.float64).reshape(6))
        pos += im.nbytes
    pix = torch.from_numpy(np.concatenate([im.reshape(-1) for im in images])).to(DEV)
    tab = torch.from_numpy(table.view(np.uint8).copy()).to(DEV)
    n = (2 if flip else 1) * len(images) * 3 * OH * OW
    buf, out = _guarded(n)
    mean, std = _mean_std()
    st = _lib.lib().cpb200_pre_process_batch(pix.data_ptr(), tab.data_ptr(), len(images), out.data_ptr(), OH, OW, mean,
                                             std, 1 if flip else 0, torch.cuda.current_stream().cuda_stream)
    _lib.check(st, "pre_process_batch")
    torch.cuda.synchronize()
    _check_guards(buf, n)
    return out.view(-1, 3, OH, OW).cpu()


def _first_diff(got, want):
    bad = (got != want).nonzero()
    i = tuple(bad[0].tolist())
    return f"{len(bad)} values differ; first at {i}: kernel {got[i].item()!r}, model {want[i].item()!r}"


@pytest.mark.parametrize("label", list(pc.WARP_CASE))
def test_pre_process_equals_warp_model(label):
    case = pc.WARP_CASE[label]
    images, trans = case.build()
    want = [torch.from_numpy(pc.pre_process_model(im, t, case.OH, case.OW, case.flip)) for im, t in zip(images, trans)]
    for n, (im, t) in enumerate(zip(images, trans)):
        got = _pre_single(im, t, case.OH, case.OW, case.flip)
        assert torch.equal(got, want[n]), f"cpb200_pre_process, image {n}: " + _first_diff(got, want[n])
        if case.flip:      # the mirrored copy is the first image reversed along x, exactly
            assert torch.equal(got[1], got[0].flip(-1))
    got = _pre_batch(images, trans, case.OH, case.OW, case.flip)
    want = torch.cat(want)
    assert torch.equal(got, want), "cpb200_pre_process_batch: " + _first_diff(got, want)


@pytest.mark.parametrize("label", list(pc.FLIP_CASE))
def test_flip_merge_equals_restatement(label):
    from centerpose_b200 import _lib
    case = pc.FLIP_CASE[label]
    maps = [torch.from_numpy(a) if a is not None else None for a in case.build()]
    want = pc.flip_merge_ref(*maps, case.perm)
    dev = [m.to(DEV) if m is not None else None for m in maps]
    P = case.P
    outs = [torch.full((P,) + tuple(m.shape[1:]), CANARY, device=DEV) if m is not None else None for m in dev]
    perm = (ctypes.c_int * case.J)(*case.perm)
    st = _lib.lib().cpb200_flip_merge(*[m.data_ptr() if m is not None else None for m in dev],
                                      *[o.data_ptr() if o is not None else None for o in outs],
                                      P, case.H, case.W, case.J, case.CH, perm, torch.cuda.current_stream().cuda_stream)
    _lib.check(st, "flip_merge")
    for name, g, w in zip(("hm", "wh", "hps", "hm_hp"), outs, want):
        assert (g is None) == (w is None)
        if g is not None:
            g = g.cpu()
            assert torch.equal(g, w), f"{name}: " + _first_diff(g, w)


def test_flip_merge_refuses_bad_arguments_without_launching():
    from centerpose_b200 import _lib
    L = _lib.lib()
    t = torch.zeros(2, 1, 4, 4, device=DEV)
    wh = torch.zeros(2, 2, 4, 4, device=DEV)
    hps = torch.zeros(2, 130, 4, 4, device=DEV)
    hp = torch.zeros(2, 65, 4, 4, device=DEV)
    o = torch.full((1, 130, 4, 4), CANARY, device=DEV)
    s = torch.cuda.current_stream().cuda_stream

    def call(hm, J, perm, hm_hp=hp.data_ptr(), o_hp=o.data_ptr()):
        return L.cpb200_flip_merge(hm, wh.data_ptr(), hps.data_ptr(), hm_hp, o.data_ptr(), o.data_ptr(), o.data_ptr(),
                                   o_hp, 1, 4, 4, J, 1, perm, s)

    ok = (ctypes.c_int * 64)(*range(64))
    bad_hi = (ctypes.c_int * 17)(*([0] * 16 + [17]))
    bad_lo = (ctypes.c_int * 17)(*([-1] + [0] * 16))
    before = L.cpb200_launch_count()
    assert call(None, 17, ok) == 1                                     # hm null
    assert call(t.data_ptr(), 17, None) == 1                           # flip_perm null
    assert call(t.data_ptr(), 17, ok, o_hp=None) == 1                  # hm_hp without its output
    assert call(t.data_ptr(), 65, (ctypes.c_int * 65)(*range(65))) == 1
    assert call(t.data_ptr(), 0, ok) == 1
    assert call(t.data_ptr(), 17, bad_hi) == 1
    assert call(t.data_ptr(), 17, bad_lo) == 1
    torch.cuda.synchronize()
    assert L.cpb200_launch_count() == before
    assert bool((o == CANARY).all())
    assert call(t.data_ptr(), 64, ok, hm_hp=None, o_hp=None) == 0      # J = 64, the largest accepted
    torch.cuda.synchronize()
    assert L.cpb200_launch_count() == before + 1


def _assert_rows_equal(got, want, keep_got, keep_want, what):
    assert keep_got == keep_want, f"{what}: keep {keep_got} != {keep_want}"
    if np.array_equal(got, want):
        return
    bad = np.argwhere(got != want)
    r, c = bad[0]
    raise AssertionError(f"{what}: {len(bad)} values differ; first at row {r} column {c}: kernel {got[r, c]!r}, "
                         f"port {want[r, c]!r}")


def _port(rows, case):
    from centerpose_b200.soft_nms import soft_nms_39
    out = rows.copy()
    return out, len(soft_nms_39(out, **case.params()))


@pytest.mark.parametrize("label", list(pc.NMS_CASE))
def test_soft_nms_equals_port(label):
    from centerpose_b200.soft_nms import soft_nms_39_cuda, soft_nms_39_cuda_batch
    case = pc.NMS_CASE[label]
    rows = case.build()
    want, keep = _port(rows, case)
    dev = torch.from_numpy(rows.copy()).to(DEV)
    k = soft_nms_39_cuda(dev, **case.params())
    _assert_rows_equal(dev.cpu().numpy(), want, k, keep, "cpb200_soft_nms_39")
    # the same image three times in one batched launch
    dev = torch.from_numpy(np.stack([rows] * 3)).to(DEV)
    ks = soft_nms_39_cuda_batch(dev, **case.params()).cpu().tolist()
    for b in range(3):
        _assert_rows_equal(dev[b].cpu().numpy(), want, ks[b], keep, f"cpb200_soft_nms_39_batch image {b}")


def test_soft_nms_batch_of_300_images():
    from centerpose_b200.soft_nms import soft_nms_39_cuda_batch
    case = pc.NMS_BATCH
    rows = case.build()
    dev = torch.from_numpy(rows.copy()).to(DEV)
    ks = soft_nms_39_cuda_batch(dev, **case.params()).cpu().tolist()
    got = dev.cpu().numpy()
    for b in range(rows.shape[0]):
        want, keep = _port(rows[b], case)
        _assert_rows_equal(got[b], want, ks[b], keep, f"image {b}")


def test_soft_nms_matches_compiled_reference_golden():
    """tests/golden/soft_nms_cases.npz: the reference's own Cython soft_nms_39 on the constructed cases.  Keep counts
    and every moved or unmoved column equal; scores within 1 ulp (Cython 3 rounds one product differently)."""
    from centerpose_b200.soft_nms import soft_nms_39_cuda
    from tests.test_post_cases_cpu import assert_matches_cython
    g = np.load(GOLD)
    for case in pc.NMS_CASES:
        rows = case.build()
        dev = torch.from_numpy(rows.copy()).to(DEV)
        k = soft_nms_39_cuda(dev, **case.params())
        assert_matches_cython(dev.cpu().numpy(), k, g, case)
