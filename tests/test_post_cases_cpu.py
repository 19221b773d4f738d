"""CPU checks of tests/post_cases.py, the cases and references the pre-process warp, flip merge and soft-NMS kernels
are held to on the GPU (tests/test_post_cases_gpu.py):

  * the integer warp model equals cv2.warpAffine and the numpy normalisation byte for byte on every warp case, the tie
    cases included, and the normalisation is exhaustive over all 256 values of each channel;
  * each case reaches the branches it claims, and together the cases reach every warp, flip and soft-NMS class
    (printed per kernel with the cases that reach each);
  * the torch flip restatement equals the reference's flip helpers, and the host soft_nms_39 port equals a literal
    restatement of nms.pyx:172-275, the kernel-plan trace, and the reference's compiled Cython (golden fixture);
  * restated bugs (wrong tail restore, ``>=`` arg-max, a walk that ignores or drops the hit flag, a sign flip on
    ``wh``, ``floor`` for ``llrint`` ...) give results that differ from the references on the cases.
"""
import os

import cv2
import numpy as np
import pytest
import torch

from tests import post_cases as pc

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def assert_matches_cython(got, keep, g, case):
    """``got`` (N, 56) and ``keep`` against the Cython golden of ``case``: keep count and every column but the score
    exactly, scores within 1 ulp (Cython 3 evaluates one float product of nms.pyx in double)."""
    assert str(g[f"sha_{case.label}"]) == pc.digest(case.build()), f"{case.label}: input changed since the golden"
    want = np.asarray(g[f"out_{case.label}"])
    assert keep == int(g[f"keep_{case.label}"]), (case.label, keep, int(g[f"keep_{case.label}"]))
    cols = np.r_[0:4, 5:56]
    assert np.array_equal(got[:, cols], want[:, cols]), f"{case.label}: rows moved differently"
    ulp = np.spacing(np.maximum(np.abs(got[:, 4]), np.abs(want[:, 4])).astype(np.float32))
    assert (np.abs(got[:, 4] - want[:, 4]) <= ulp).all(), f"{case.label}: scores beyond 1 ulp"


def _coverage(kernel, classes, reached):
    lines = [f"{kernel}: {len(classes)} classes"]
    for c in classes:
        lines.append(f"  {c:28s} {', '.join(reached.get(c, [])) or 'NOT REACHED'}")
    print("\n".join(lines))
    missing = [c for c in classes if not reached.get(c)]
    assert not missing, f"{kernel}: no case reaches {missing}"


# ---------------------------------------------------------------------------------------------------------- warp
_WARP = {}


def _warp_built(label):
    if label not in _WARP:
        _WARP[label] = pc.WARP_CASE[label].build()
    return _WARP[label]


@pytest.mark.parametrize("label", list(pc.WARP_CASE))
def test_warp_model_equals_cv2_and_numpy(label):
    case = pc.WARP_CASE[label]
    for im, t in zip(*_warp_built(label)):
        inp = cv2.warpAffine(im, t, (case.OW, case.OH), flags=cv2.INTER_LINEAR)
        assert np.array_equal(pc.warp_u8(im, t, case.OH, case.OW), inp)
        # base_detector.py:45-50
        ref = ((inp / 255. - pc.MEAN.reshape(1, 1, 3)) / pc.STD.reshape(1, 1, 3)).astype(np.float32)
        ref = ref.transpose(2, 0, 1)[None]
        if case.flip:
            ref = np.concatenate((ref, ref[:, :, :, ::-1]), axis=0)
        assert np.array_equal(pc.pre_process_model(im, t, case.OH, case.OW, case.flip), ref)


def test_normalisation_is_exhaustive():
    u = np.arange(256, dtype=np.uint8)
    inp = np.stack([u, u, u], -1)[None]                                        # every value in every channel
    ref = ((inp / 255. - pc.MEAN.reshape(1, 1, 3)) / pc.STD.reshape(1, 1, 3)).astype(np.float32)[0].T
    assert np.array_equal(pc.normalise_lut(), ref)
    # and the all-values case feeds each of the 256 values through each channel of the kernel
    im, = _warp_built("all_values_identity")[0]
    for c in range(3):
        assert set(np.unique(im[..., c]).tolist()) == set(range(256))


@pytest.mark.parametrize("label", list(pc.WARP_CASE))
def test_warp_case_reaches_its_claims(label):
    case = pc.WARP_CASE[label]
    got = pc.warp_case_classes(case, *_warp_built(label))
    assert set(case.claims) <= got, f"{label} misses {sorted(set(case.claims) - got)}"
    assert set(case.claims) <= set(pc.WARP_CLASSES)


def test_warp_cases_cover_every_class():
    reached = {}
    for case in pc.WARP_CASES:
        for c in case.claims:
            reached.setdefault(c, []).append(case.label)
    _coverage("pre_process_kernel", pc.WARP_CLASSES, reached)


def test_tie_cases_separate_rounding_from_fma():
    """On the tie row the separately rounded term is exactly k + 1/2 and llrint takes the even neighbour; the fused
    term is off the tie and rounds the other way, which moves at least one output byte."""
    for label, key in (("tie_x_row", "X0"), ("tie_y_row", "Y0")):
        case = pc.WARP_CASE[label]
        (im,), (t,) = _warp_built(label)
        c = pc.warp_coords(t, case.OH, case.OW)
        f = pc.warp_coords(t, case.OH, case.OW, fused=True)
        rows = np.flatnonzero(c.ties[key] & (getattr(c, key) != getattr(f, key)))
        assert len(rows) >= 1, label
        assert not np.array_equal(pc.warp_u8(im, t, case.OH, case.OW), pc.warp_u8(im, t, case.OH, case.OW, fused=True))


def test_warp_bugs_are_visible():
    """``floor`` for ``llrint`` and the fused row term each change the output of some case."""
    for kw in (dict(rnd=np.floor), dict(fused=True)):
        assert any(not np.array_equal(pc.warp_u8(im, t, c.OH, c.OW), pc.warp_u8(im, t, c.OH, c.OW, **kw))
                   for c in pc.WARP_CASES for im, t in zip(*_warp_built(c.label))), kw


# ---------------------------------------------------------------------------------------------------------- flip
def _flip_lr_np(x, flip_idx):          # lib/models/utils.py:30-36
    tmp = x[..., ::-1].copy()
    for e in flip_idx:
        tmp[:, e[0], ...], tmp[:, e[1], ...] = tmp[:, e[1], ...].copy(), tmp[:, e[0], ...].copy()
    return tmp


def _flip_lr_off_np(x, flip_idx):      # lib/models/utils.py:38-47
    tmp = x[..., ::-1].copy()
    shape = tmp.shape
    tmp = tmp.reshape(tmp.shape[0], 17, 2, tmp.shape[2], tmp.shape[3])
    tmp[:, :, 0, :, :] *= -1
    for e in flip_idx:
        tmp[:, e[0], ...], tmp[:, e[1], ...] = tmp[:, e[1], ...].copy(), tmp[:, e[0], ...].copy()
    return tmp.reshape(shape)


def test_flip_restatement_equals_reference_helpers():
    """flip_merge_ref with the COCO pairs == multi_pose.py:45-53 with the reference's helpers, on the coded maps and on
    the golden outputs of the reference's own flip_lr / flip_lr_off (tests/golden/flip.npz)."""
    case = pc.FLIP_CASE["coco_7x12"]
    hm, wh, hps, hp = case.build()
    o = pc.flip_merge_ref(*[torch.from_numpy(a) for a in (hm, wh, hps, hp)], case.perm)
    want = [(hm[0:1] + hm[1:2, ..., ::-1]) / 2, (wh[0:1] + wh[1:2, ..., ::-1]) / 2,
            (hps[0:1] + _flip_lr_off_np(hps[1:2], pc.COCO_FLIP_IDX)) / 2,
            (hp[0:1] + _flip_lr_np(hp[1:2], pc.COCO_FLIP_IDX)) / 2]
    for g, w in zip(o, want):
        assert np.array_equal(g.numpy(), w.astype(np.float32))
    g = np.load(os.path.join(GOLD, "flip.npz"))
    z_hp, z_hps = np.zeros_like(g["hm_hp"]), np.zeros_like(g["hps"])
    z_hm = np.zeros((2, 1) + g["hm_hp"].shape[2:], np.float32)
    o = pc.flip_merge_ref(torch.from_numpy(z_hm), torch.from_numpy(np.zeros((2, 2) + z_hm.shape[2:], np.float32)),
                          torch.from_numpy(np.concatenate([z_hps, g["hps"]])),
                          torch.from_numpy(np.concatenate([z_hp, g["hm_hp"]])), pc.COCO_PERM)
    assert np.array_equal(o[2].numpy() * 2, g["flip_lr_off"]) and np.array_equal(o[3].numpy() * 2, g["flip_lr"])


@pytest.mark.parametrize("label", list(pc.FLIP_CASE))
def test_flip_case_reaches_its_claims_and_values_are_exact(label):
    case = pc.FLIP_CASE[label]
    got = pc.flip_case_classes(case)
    assert set(case.claims) <= got, f"{label} misses {sorted(set(case.claims) - got)}"
    maps = [a for a in case.build() if a is not None]
    vals = np.concatenate([a.reshape(-1) for a in maps])
    assert (np.abs(vals) <= 2 ** 22).all() and (vals == np.round(vals)).all()
    assert len(np.unique(vals)) == len(vals)                   # every element has its own value
    assert sorted(case.perm) == list(range(case.J))


def test_flip_cases_cover_every_class():
    reached = {}
    for case in pc.FLIP_CASES:
        for c in case.claims:
            reached.setdefault(c, []).append(case.label)
    _coverage("flip_merge_kernel", pc.FLIP_CLASSES, reached)


def _flip_bug(name, hm, wh, hps, hp, perm):
    a = lambda t: t[0::2]
    f = lambda t: torch.flip(t[1::2], [3])
    o = list(pc.flip_merge_ref(hm, wh, hps, hp, perm))
    if name == "hps sign dropped":
        P, C2, H, W = a(hps).shape
        o[2] = (a(hps) + f(hps).reshape(P, C2 // 2, 2, H, W)[:, list(perm)].reshape(P, C2, H, W)) / 2
    elif name == "wh x negated":
        w = f(wh).clone(); w[:, 0] *= -1; o[1] = (a(wh) + w) / 2
    elif name == "perm applied to wh":
        p = [perm[c] % 2 if c < len(perm) else c for c in range(2)]
        o[1] = (a(wh) + f(wh)[:, p]) / 2
    elif name == "no mirror":
        o[0] = (a(hm) + hm[1::2]) / 2
    elif name == "perm ignored":
        if hp is not None:
            o[3] = (a(hp) + f(hp)) / 2
        else:
            P, C2, H, W = a(hps).shape
            b = f(hps).reshape(P, C2 // 2, 2, H, W).clone(); b[:, :, 0] *= -1
            o[2] = (a(hps) + b.reshape(P, C2, H, W)) / 2
    return o


FLIP_BUGS = ("hps sign dropped", "wh x negated", "perm applied to wh", "no mirror", "perm ignored")


def test_flip_bugs_are_visible():
    caught = {b: [] for b in FLIP_BUGS}
    for case in pc.FLIP_CASES:
        maps = [torch.from_numpy(a) if a is not None else None for a in case.build()]
        ref = pc.flip_merge_ref(*maps, case.perm)
        for b in FLIP_BUGS:
            got = _flip_bug(b, *maps, case.perm)
            if any(g is not None and not torch.equal(g, r) for g, r in zip(got, ref)):
                caught[b].append(case.label)
        if case.W > 1:
            assert case.label in caught["no mirror"]
        assert case.label in caught["hps sign dropped"] and case.label in caught["wh x negated"]
    assert all(caught.values()), caught


# ---------------------------------------------------------------------------------------------------------- soft-NMS
def _nms_images(case):
    rows = case.build()
    return rows if rows.ndim == 3 else rows[None]


@pytest.mark.parametrize("label", list(pc.NMS_CASE) + [pc.NMS_BATCH.label])
def test_soft_nms_port_equals_literal_and_trace(label):
    """centerpose_b200.soft_nms.soft_nms_39 == the literal nms.pyx restatement == the kernel-plan trace, whole arrays."""
    from centerpose_b200.soft_nms import soft_nms_39
    case = pc.NMS_CASE.get(label, pc.NMS_BATCH)
    for rows in _nms_images(case):
        assert np.isfinite(rows).all()                                     # the NaN-free premise
        a, b, c = rows.copy(), rows.copy(), rows.copy()
        ka = len(soft_nms_39(a, **case.params()))
        kb = pc.soft_nms_literal(b, **case.params())
        kc, _ = pc.soft_nms_trace(c, **case.params())
        assert ka == kb == kc
        assert np.array_equal(a, b) and np.array_equal(a, c)


@pytest.mark.parametrize("label", list(pc.NMS_CASE) + [pc.NMS_BATCH.label])
def test_soft_nms_case_reaches_its_claims(label):
    case = pc.NMS_CASE.get(label, pc.NMS_BATCH)
    imgs = _nms_images(case)
    got = {f"N{imgs.shape[1]}"} | ({"batch"} if len(imgs) > 1 else set())
    for rows in imgs:
        got |= pc.soft_nms_trace(rows.copy(), **case.params())[1]
    assert set(case.claims) <= got, f"{label} misses {sorted(set(case.claims) - got)}"
    assert set(case.claims) <= set(pc.NMS_CLASSES)


def test_soft_nms_cases_cover_every_class():
    reached = {}
    for case in pc.NMS_CASES + [pc.NMS_BATCH]:
        for c in case.claims:
            reached.setdefault(c, []).append(case.label)
    _coverage("soft_nms_kernel", pc.NMS_CLASSES, reached)


def test_soft_nms_bugs_are_visible():
    """Each restated kernel bug changes the array or keep count of at least one case that claims the branch."""
    needs = {"no tail restore": "tail_restore", "argmax >=": "tie_thread", "walk ignores s_hit": "low_score_not_hit",
             "s_hit not carried": "moved_in_not_hit_low"}
    for bug, branch in needs.items():
        caught = []
        for case in pc.NMS_CASES:
            if branch not in case.claims:
                continue
            rows = case.build()
            a, b = rows.copy(), rows.copy()
            ka, _ = pc.soft_nms_trace(a, **case.params())
            kb, _ = pc.soft_nms_trace(b, **case.params(), bug=bug)
            if ka != kb or not np.array_equal(a, b):
                caught.append(case.label)
        assert caught, f"no case tells '{bug}' from the reference"


def test_soft_nms_port_matches_compiled_reference_golden():
    g = np.load(os.path.join(GOLD, "soft_nms_cases.npz"))
    for case in pc.NMS_CASES:
        rows = case.build()
        k = pc.soft_nms_literal(rows, **case.params())
        assert_matches_cython(rows, k, g, case)
