"""Plain references and constructed cases for the three numeric kernels of csrc/post.cu:

  * ``pre_process_kernel`` (cpb200_pre_process, _batch): cv2.warpAffine (INTER_LINEAR, constant-0 border) of an 8-bit
    image, ``(u/255. - mean)/std`` in float64 rounded to float32, HWC->CHW and the mirrored copy.  ``warp_coords`` is
    an integer model of cv2's fixed-point warp (imgwarp.cpp: double inverse, AB_SCALE = 1024, round_delta = 16,
    ``saturate_cast<short>`` of the tap, 5-bit weights); ``pre_process_model`` adds the normalisation.
  * ``flip_merge_kernel`` (cpb200_flip_merge): ``flip_merge_ref`` restates multi_pose.py:45-53 for any class count,
    joint count and joint permutation, in torch fp32.
  * ``soft_nms_kernel`` (cpb200_soft_nms_39, _batch): ``soft_nms_literal`` restates nms.pyx:172-275 line by line;
    ``soft_nms_trace`` follows the kernel's plan (parallel decay, then the swap-with-last walk over the rows that
    touched box i) and records which branches each step reaches.

Every case has a label, the branches it claims, and a builder; tests/test_post_cases_cpu.py proves the claims and the
references, tests/test_post_cases_gpu.py holds the kernels to the references exactly.

Scores are NaN-free by premise: the reference's strict ``<`` scan, ``np.argmax`` and the kernel's reduction treat a NaN
score differently, and the detector's scores (sigmoids of finite logits) are never NaN.  The CPU test checks the
premise on every case.
"""
from __future__ import annotations

import hashlib
import math
from dataclasses import dataclass
from fractions import Fraction
from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np
import torch

from centerpose_b200.image import get_affine_transform

F32 = np.float32
# cfg.DATASET.MEAN / STD of the COCO pose models (centerpose_b200/config.py)
MEAN = np.array([0.408, 0.447, 0.47], np.float32)
STD = np.array([0.289, 0.274, 0.278], np.float32)
AB_SCALE, ROUND_DELTA, INTER_BITS = 1024, 16, 5
SHORT_MIN, SHORT_MAX = -32768, 32767


def digest(*arrays) -> str:
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


# =====================================================================================================================
# warp model
# =====================================================================================================================
def invert(t) -> Tuple[float, ...]:
    """cv2.warpAffine's inverse of the forward 2x3 matrix (imgwarp.cpp, invertAffineTransform order): every product
    and difference rounded to double on its own (Python floats)."""
    t = [float(v) for v in np.asarray(t, np.float64).reshape(6)]
    D = t[0] * t[4] - t[1] * t[3]
    D = 1.0 / D if D != 0 else 0.0
    m0, m4, m1, m3 = t[4] * D, t[0] * D, t[1] * -D, t[3] * -D
    m2 = -m0 * t[2] - m1 * t[5]
    m5 = -m3 * t[2] - m4 * t[5]
    return m0, m1, m2, m3, m4, m5


def row_term(a: float, b: float, y: int, fused: bool = False) -> float:
    """``(a*y + b) * 1024`` as cv2 evaluates it (two roundings), or with ``a*y + b`` rounded once (an FMA)."""
    s = float(Fraction(a) * y + Fraction(b)) if fused else a * float(y) + b
    return s * 1024.0


def _is_tie(v: np.ndarray) -> np.ndarray:
    return (v - np.floor(v)) == 0.5


@dataclass
class Coords:
    X0: np.ndarray          # (OH,) int64: llrint(row term) + round_delta
    Y0: np.ndarray
    adelta: np.ndarray      # (OW,) int64: llrint(m0 * x * 1024)
    bdelta: np.ndarray
    X: np.ndarray           # (OH, OW) int64: (X0 + adelta) >> 5, source x in 1/32 px
    Y: np.ndarray
    sx_raw: np.ndarray      # X >> 5 before saturate_cast<short>
    sy_raw: np.ndarray
    sx: np.ndarray
    sy: np.ndarray
    fx: np.ndarray
    fy: np.ndarray
    ties: dict              # "X0" / "Y0" / "adelta" / "bdelta" -> bool array: the term was exactly k + 1/2


def warp_coords(t, OH: int, OW: int, fused: bool = False, rnd: Callable = np.rint) -> Coords:
    """The per-pixel source coordinates of cv2.warpAffine(INTER_LINEAR) as integers.  ``fused`` evaluates the row terms
    with one rounding (what an FMA-contracted kernel computes); ``rnd`` replaces llrint (round half to even)."""
    m0, m1, m2, m3, m4, m5 = invert(t)
    x = np.arange(OW, dtype=np.float64)
    ad_v, bd_v = m0 * x * 1024.0, m3 * x * 1024.0
    x0_v = np.array([row_term(m1, m2, y, fused) for y in range(OH)])
    y0_v = np.array([row_term(m4, m5, y, fused) for y in range(OH)])
    adelta, bdelta = rnd(ad_v).astype(np.int64), rnd(bd_v).astype(np.int64)
    X0 = rnd(x0_v).astype(np.int64) + ROUND_DELTA
    Y0 = rnd(y0_v).astype(np.int64) + ROUND_DELTA
    X = (X0[:, None] + adelta[None, :]) >> (10 - INTER_BITS)
    Y = (Y0[:, None] + bdelta[None, :]) >> (10 - INTER_BITS)
    sx_raw, sy_raw = X >> INTER_BITS, Y >> INTER_BITS
    return Coords(X0, Y0, adelta, bdelta, X, Y, sx_raw, sy_raw, np.clip(sx_raw, SHORT_MIN, SHORT_MAX),
                  np.clip(sy_raw, SHORT_MIN, SHORT_MAX), X & 31, Y & 31,
                  {"X0": _is_tie(x0_v), "Y0": _is_tie(y0_v), "adelta": _is_tie(ad_v), "bdelta": _is_tie(bd_v)})


def _taps(c: Coords, h: int, w: int):
    """[(valid (OH,OW), row, col, weight)] of the four bilinear taps; weights are the integers that sum to 2^15."""
    fx, fy = c.fx, c.fy
    out = []
    for dy, dx, wgt in ((0, 0, (32 - fx) * (32 - fy) * 32), (0, 1, fx * (32 - fy) * 32),
                        (1, 0, (32 - fx) * fy * 32), (1, 1, fx * fy * 32)):
        yy, xx = c.sy + dy, c.sx + dx
        out.append(((yy >= 0) & (yy < h) & (xx >= 0) & (xx < w), yy, xx, wgt))
    return out


def warp_u8(img: np.ndarray, t, OH: int, OW: int, **kw) -> np.ndarray:
    """cv2.warpAffine(img, t, (OW, OH), flags=INTER_LINEAR) with the constant-0 border, on the integer model."""
    h, w = img.shape[:2]
    c = warp_coords(t, OH, OW, **kw)
    acc = np.zeros((OH, OW, 3), np.int64)
    for ok, yy, xx, wgt in _taps(c, h, w):
        v = img[np.clip(yy, 0, h - 1), np.clip(xx, 0, w - 1)].astype(np.int64)
        acc += v * (ok * wgt)[..., None]
    return np.clip((acc + (1 << 14)) >> 15, 0, 255).astype(np.uint8)


def normalise_lut(mean=MEAN, std=STD) -> np.ndarray:
    """(3, 256) float32: ``(u/255. - mean[c]) / std[c]`` in double, rounded to float (the numpy expression of
    base_detector.py:45 with float32 mean / std promoted to float64)."""
    lut = np.empty((3, 256), np.float32)
    for c in range(3):
        for u in range(256):
            lut[c, u] = F32((u / 255.0 - float(mean[c])) / float(std[c]))
    return lut


def pre_process_model(img: np.ndarray, t, OH: int, OW: int, flip: bool, mean=MEAN, std=STD, **kw) -> np.ndarray:
    """(1 or 2, 3, OH, OW) float32: what cpb200_pre_process writes for one image."""
    u = warp_u8(img, t, OH, OW, **kw)
    lut = normalise_lut(mean, std)
    chw = np.stack([lut[c][u[..., c]] for c in range(3)])
    return np.stack([chw, chw[:, :, ::-1]]) if flip else chw[None]


def _non_dyadic(t) -> bool:
    """The exact inverse of the matrix's linear part is not representable, so the double inverse is rounded."""
    a = [Fraction(float(v)) for v in np.asarray(t, np.float64).reshape(6)]
    D = a[0] * a[4] - a[1] * a[3]
    if D == 0:
        return False
    return any(float(v) != v for v in (a[4] / D, a[1] / D, a[3] / D, a[0] / D))


def warp_classes(img, t, OH: int, OW: int) -> set:
    """The warp branches one (image, matrix) reaches, named as in WARP_CLASSES."""
    h, w = img.shape[:2]
    c = warp_coords(t, OH, OW)
    f = warp_coords(t, OH, OW, fused=True)
    a = np.asarray(t, np.float64).reshape(2, 3)
    det = a[0, 0] * a[1, 1] - a[0, 1] * a[1, 0]
    got = set()
    for k, v in c.ties.items():
        if v.any():
            got.add("tie_" + k)
    if (c.X0 != f.X0).any():
        got.add("fused_X0_differs")
    if (c.Y0 != f.Y0).any():
        got.add("fused_Y0_differs")
    if "fused_X0_differs" in got or "fused_Y0_differs" in got:
        if (warp_u8(img, t, OH, OW) != warp_u8(img, t, OH, OW, fused=True)).any():
            got.add("fused_changes_output")
    for nm, raw in (("x", c.sx_raw), ("y", c.sy_raw)):
        if (raw < SHORT_MIN).any():
            got.add(f"clamp_{nm}_lo")
        if (raw > SHORT_MAX).any():
            got.add(f"clamp_{nm}_hi")
    ok = np.stack([tp[0] for tp in _taps(c, h, w)])
    n_in = ok.sum(0)
    if (n_in == 4).any():
        got.add("taps_all_in")
    if ((n_in > 0) & (n_in < 4)).any():
        got.add("taps_partial")
    if (n_in == 0).any():
        got.add("taps_all_out")
    for nm, cond in (("left", c.sx == -1), ("right", c.sx == w - 1), ("top", c.sy == -1), ("bottom", c.sy == h - 1)):
        if cond.any():
            got.add("edge_" + nm)
    if ((c.fx == 0) & (c.fy == 0)).any():
        got.add("integer_sample")
    if det == 0:
        got.add("singular")
    elif det < 0:
        got.add("reflection")
    if a[0, 1] != 0 or a[1, 0] != 0:
        got.add("off_diagonal")
    if _non_dyadic(t):
        got.add("non_dyadic")
    if h == 1 or w == 1:
        got.add("sub_tap_source")
    if OH * OW > h * w:
        got.add("upscale")
    return got


WARP_CLASSES = ("tie_X0", "tie_Y0", "tie_adelta", "tie_bdelta", "fused_X0_differs", "fused_Y0_differs",
                "fused_changes_output",
                "clamp_x_lo", "clamp_x_hi", "clamp_y_lo", "clamp_y_hi", "taps_all_in", "taps_partial", "taps_all_out",
                "edge_left", "edge_right", "edge_top", "edge_bottom", "integer_sample", "singular", "reflection",
                "off_diagonal", "non_dyadic", "sub_tap_source", "upscale", "batch_mixed_sizes", "flip", "no_flip")


def tie_matrix(axis: str, abcd=(1.1, 2.3, 0.2, 0.9), y: int = 45, near: float = 12.0) -> np.ndarray:
    """A forward matrix whose row term for output row ``y`` lands exactly on a rounding tie ``(k + 1/2) / 1024`` of the
    separately rounded evaluation, while the fused (FMA) evaluation rounds to the other integer.  The row term
    ``m1*y`` (axis "x") or ``m4*y`` (axis "y") is large next to the tie value, so the rounding error of the product is
    many ulps of the tie value and the fused sum cannot round back onto the tie.  The translation is stepped one ulp at
    a time until ``m2`` (or ``m5``) makes the sum exact."""
    a, b, c, d = abcd
    for k in range(int(near * 1024), int(near * 1024) + 4096):
        tie = (k + 0.5) / 1024
        for sgn in (1.0, -1.0):
            t = np.array([[a, b, 0.0], [c, d, 0.0]])
            m0, m1, _, m3, m4, _ = invert(t)
            p = (m1 if axis == "x" else m4) * float(y)
            if Fraction(p) == Fraction(m1 if axis == "x" else m4) * y:
                raise ValueError("the row product is exact: pick a non-dyadic matrix")
            want = Fraction(tie) - Fraction(p)
            if float(want) != want:
                continue
            want = float(want)
            # axis x: m2 = (-m0) * t2 - m1 * 0;  axis y: m5 = (-m3) * 0 - m4 * t5
            v = -want / m0 if axis == "x" else -want / m4
            for _ in range(256):
                t[0 if axis == "x" else 1, 2] = v
                got = invert(t)[2 if axis == "x" else 5]
                if got == want:
                    break
                v = np.nextafter(v, sgn * np.inf)
            else:
                continue
            mm = invert(t)
            ma, mb = (mm[1], mm[2]) if axis == "x" else (mm[4], mm[5])
            sep, fus = row_term(ma, mb, y), row_term(ma, mb, y, fused=True)
            if sep - math.floor(sep) == 0.5 and int(np.rint(sep)) != int(np.rint(fus)):
                return t
    raise ValueError("no tie found")


@dataclass
class WarpCase:
    label: str
    claims: Tuple[str, ...]
    build: Callable[[], Tuple[List[np.ndarray], List[np.ndarray]]]    # -> (images, forward matrices)
    OH: int
    OW: int
    flip: bool


def _img(h, w, seed, kind="random"):
    rng = np.random.RandomState(seed)
    if kind in ("stripes_x", "stripes_y"):    # 0 / 255 stripes: a 1/32 px step of the sample moves the byte by ~8
        ramp = np.arange(w)[None, :] if kind == "stripes_x" else np.arange(h)[:, None]
        v = (ramp % 2) * 255 + np.zeros((h, w), np.int64)
        return np.repeat(v[..., None], 3, 2).astype(np.uint8)
    if kind == "all_values":     # every byte value in every channel
        v = (np.arange(h * w * 3) % 256).reshape(h, w, 3)
        return np.ascontiguousarray(np.stack([v[..., 0], (v[..., 1] + 85) % 256, (v[..., 2] + 170) % 256], -1)
                                    ).astype(np.uint8)
    return rng.randint(0, 256, (h, w, 3)).astype(np.uint8)


def geometry(h: int, w: int, fix_res: bool, inp=(512, 512), pad=31):
    """(trans_input, inp_h, inp_w) of MultiPoseDetector._pre_process_geometry at scale 1 (base_detector.py:33-47)."""
    if fix_res:
        inp_h, inp_w = inp
        c = np.array([w / 2., h / 2.], dtype=np.float32)
        s = max(h, w) * 1.0
    else:
        inp_h, inp_w = (h | pad) + 1, (w | pad) + 1
        c = np.array([w // 2, h // 2], dtype=np.float32)
        s = np.array([inp_w, inp_h], dtype=np.float32)
    return get_affine_transform(c, s, 0, [inp_w, inp_h]), inp_h, inp_w


def _rot(scale, deg, tx, ty, shear=0.0, flip_x=False):
    r = math.radians(deg)
    a = np.array([[math.cos(r), -math.sin(r) + shear], [math.sin(r), math.cos(r)]]) * scale
    if flip_x:
        a[:, 0] *= -1
    return np.concatenate([a, [[tx], [ty]]], 1)


def _single(h, w, seed, t, kind="random"):
    return lambda: ([_img(h, w, seed, kind)], [np.asarray(t, np.float64)])


def _geo_case(label, shapes, fix_res, flip, claims):
    def build():
        ims = [_img(h, w, 50 + n) for n, (h, w) in enumerate(shapes)]
        return ims, [geometry(h, w, fix_res)[0] for h, w in shapes]
    _, OH, OW = geometry(*shapes[0], fix_res)
    return WarpCase(label, claims, build, OH, OW, flip)


WARP_CASES: List[WarpCase] = [
    _geo_case("fix_res_480x640", [(480, 640)], True, True, ("taps_all_in", "taps_all_out", "flip")),
    _geo_case("padded_427x640", [(427, 640)], False, False, ("integer_sample", "no_flip")),
    _geo_case("fix_res_batch_mixed", [(480, 640), (100, 37), (1, 1), (333, 500)], True, True,
              ("batch_mixed_sizes", "sub_tap_source", "upscale", "flip")),
    _geo_case("padded_batch_mixed", [(200, 300), (193, 290), (170, 290)], False, False,
              ("batch_mixed_sizes", "no_flip")),
    WarpCase("non_dyadic_scale", ("non_dyadic", "edge_right", "edge_bottom", "upscale"),
             _single(23, 31, 1, _rot(1.7, 0, -3.3, -2.1)), 48, 64, False),
    # D == 1 exactly and m0 = 1 + 2^-11, m3 = -2^-11: every odd column puts adelta and bdelta on a rounding tie
    WarpCase("column_ties", ("tie_adelta", "tie_bdelta", "edge_left", "edge_top", "off_diagonal"),
             _single(30, 30, 11, [[1.0, 1.0, -10.0], [2.0 ** -11, 1.0 + 2.0 ** -11, 3.0]]), 40, 40, False),
    WarpCase("rotation", ("off_diagonal", "non_dyadic", "taps_partial", "taps_all_out"),
             _single(40, 50, 2, _rot(0.9, 33, 12.25, -8.5)), 56, 72, True),
    WarpCase("shear", ("off_diagonal",), _single(40, 50, 3, _rot(1.3, 0, -5.0, 1.5, shear=0.37)), 48, 60, False),
    WarpCase("reflection", ("reflection", "non_dyadic"), _single(30, 44, 4, _rot(1.15, 10, 60.0, 3.0, flip_x=True)),
             40, 64, True),
    WarpCase("singular", ("singular",), _single(9, 13, 5, [[1.5, 3.0, 2.0], [0.5, 1.0, -1.0]]), 8, 16, False),
    WarpCase("far_translation", ("clamp_x_lo", "clamp_y_hi"), _single(16, 16, 6, _rot(1.0, 0, 40000.25, -50000.5)),
             8, 8, False),
    WarpCase("far_translation_neg", ("clamp_x_hi", "clamp_y_lo"), _single(16, 16, 7, _rot(0.75, 0, -33000.0, 70000.0)),
             8, 8, True),
    WarpCase("source_1x1", ("sub_tap_source", "upscale", "edge_left", "edge_right"),
             _single(1, 1, 8, _rot(7.3, 0, 1.4, 2.2)), 16, 16, True),
    WarpCase("all_values_identity", ("integer_sample",), _single(16, 16, 0, np.eye(2, 3), "all_values"), 16, 16, False),
    WarpCase("tie_x_row", ("tie_X0", "fused_X0_differs", "fused_changes_output", "off_diagonal", "non_dyadic"),
             lambda: ([_img(64, 48, 9, "stripes_x")], [tie_matrix("x")]), 48, 64, False),
    WarpCase("tie_y_row", ("tie_Y0", "fused_Y0_differs", "fused_changes_output", "off_diagonal", "non_dyadic"),
             lambda: ([_img(48, 40, 10, "stripes_y")], [tie_matrix("y", abcd=(1.9, 0.3, 0.7, 1.2), y=200, near=20.0)]),
             208, 48, True),
]
WARP_CASE = {c.label: c for c in WARP_CASES}


def warp_case_classes(case: WarpCase, images=None, trans=None) -> set:
    if images is None:
        images, trans = case.build()
    got = set()
    for im, t in zip(images, trans):
        got |= warp_classes(im, t, case.OH, case.OW)
    if len({im.shape for im in images}) > 1:
        got.add("batch_mixed_sizes")
    got.add("flip" if case.flip else "no_flip")
    return got


# =====================================================================================================================
# flip merge
# =====================================================================================================================
def flip_merge_ref(hm, wh, hps, hm_hp, perm: Sequence[int]):
    """multi_pose.py:45-53 (flip_tensor / flip_lr / flip_lr_off of lib/models/utils.py:27-47) on 2P images, written for
    any joint permutation: joint j of the merged map averages joint perm[j] of the mirrored image, whose keypoint x
    offsets change sign.  torch fp32, so the sum and the halving round as the reference's do."""
    def pair(a):
        return a[0::2], torch.flip(a[1::2], [3])
    perm = torch.as_tensor(list(perm), dtype=torch.long)
    a, b = pair(hm); o_hm = (a + b) / 2
    a, b = pair(wh); o_wh = (a + b) / 2
    a, b = pair(hps)
    P, C2, H, W = b.shape
    b = b.reshape(P, C2 // 2, 2, H, W).clone()
    b[:, :, 0] *= -1
    o_hps = (a + b[:, perm].reshape(P, C2, H, W)) / 2
    o_hp = None
    if hm_hp is not None:
        a, b = pair(hm_hp); o_hp = (a + b[:, perm]) / 2
    return o_hm, o_wh, o_hps, o_hp


COCO_FLIP_IDX = [[1, 2], [3, 4], [5, 6], [7, 8], [9, 10], [11, 12], [13, 14], [15, 16]]
GRID_THREADS = 132 * 16 * 256          # flip_merge_kernel's largest grid: beyond this the grid-stride loop runs


def pairs_perm(idx, J):
    perm = list(range(J))
    for a, b in idx:
        perm[a], perm[b] = perm[b], perm[a]
    return perm


@dataclass
class FlipCase:
    label: str
    claims: Tuple[str, ...]
    P: int
    H: int
    W: int
    CH: int
    J: int
    perm: Tuple[int, ...]
    hm_hp: bool = True

    def channels(self):
        return self.CH + 2 + 2 * self.J + (self.J if self.hm_hp else 0)

    def build(self):
        """fp32 maps whose every value is an exact integer in [-2^22, 2^22) that identifies (map, image, channel, y,
        x): a bijective multiplicative hash of the element's position in the concatenated inputs, so a wrong
        source shows up as a wrong number, and a sum of two values is (almost surely) the sum of no other two."""
        shapes = [(2 * self.P, self.CH), (2 * self.P, 2), (2 * self.P, 2 * self.J)] + \
            ([(2 * self.P, self.J)] if self.hm_hp else [])
        out, base = [], 0
        for n, c in shapes:
            size = n * c * self.H * self.W
            assert base + size < 1 << 23
            code = ((np.arange(base, base + size, dtype=np.int64) * 2654435761) % (1 << 23)) - (1 << 22)
            out.append(code.astype(np.float32).reshape(n, c, self.H, self.W))
            base += size
        return tuple(out) + ((None,) if not self.hm_hp else ())


def flip_case_classes(c: FlipCase) -> set:
    got = {f"J{c.J}", f"classes{c.CH}", "hm_hp" if c.hm_hp else "hm_hp_null"}
    got.add("W1" if c.W == 1 else ("W_odd" if c.W % 2 else "W_even"))
    if c.H == 1:
        got.add("H1")
    if list(c.perm) != pairs_perm(COCO_FLIP_IDX, 17):
        got.add("perm_not_coco")
    if c.P * c.channels() * c.H * c.W > GRID_THREADS:
        got.add("grid_stride")
    if c.P > 1:
        got.add("pairs>1")
    return got


FLIP_CLASSES = ("W1", "W_odd", "W_even", "H1", "classes1", "classes3", "J1", "J17", "J64", "perm_not_coco", "hm_hp",
                "hm_hp_null", "grid_stride", "pairs>1")
COCO_PERM = tuple(pairs_perm(COCO_FLIP_IDX, 17))
FLIP_CASES = [
    FlipCase("coco_7x12", ("J17", "classes1", "hm_hp", "W_even"), 1, 7, 12, 1, 17, COCO_PERM),
    FlipCase("coco_w1_null", ("W1", "hm_hp_null", "pairs>1"), 2, 9, 1, 1, 17, COCO_PERM, hm_hp=False),
    FlipCase("h1_odd_3classes", ("H1", "W_odd", "classes3", "perm_not_coco"), 3, 1, 13, 3, 17,
             tuple((j * 5 + 3) % 17 for j in range(17))),
    FlipCase("j1", ("J1", "W_odd"), 1, 5, 9, 1, 1, (0,)),
    FlipCase("j64_cycle", ("J64", "classes3", "perm_not_coco"), 1, 6, 10, 3, 64, tuple((j + 1) % 64 for j in range(64))),
    FlipCase("j64_null", ("J64", "hm_hp_null"), 2, 3, 7, 1, 64, tuple(63 - j for j in range(64)), hm_hp=False),
    FlipCase("grid_stride_128", ("grid_stride", "pairs>1", "hm_hp", "J17"), 2, 128, 128, 1, 17, COCO_PERM),
]
FLIP_CASE = {c.label: c for c in FLIP_CASES}


# =====================================================================================================================
# soft-NMS
# =====================================================================================================================
NMS_T = 128          # soft_nms_kernel's block size: position pos is scanned by thread (pos - i) % 128 in step i


def soft_nms_literal(boxes: np.ndarray, sigma=0.5, Nt=0.3, threshold=0.001, method=0) -> int:
    """nms.pyx:172-275 restated line by line in float32 (the Cython ``cdef float`` locals).  ``N`` is captured by
    ``range`` once, as the C loop Cython emits.  ``ua`` is a double there; ``iw*ih / ua`` rounded to float equals the
    float division, since a double holds the float quotient to more than twice float's precision.  Returns the
    number of kept rows; ``boxes`` is changed in place."""
    sigma, Nt, threshold, one = F32(sigma), F32(Nt), F32(threshold), F32(1)
    N = boxes.shape[0]
    for i in range(N):
        maxscore = boxes[i, 4]
        maxpos = i
        tx1, ty1, tx2, ty2, ts = boxes[i, 0], boxes[i, 1], boxes[i, 2], boxes[i, 3], boxes[i, 4]
        pos = i + 1
        while pos < N:
            if maxscore < boxes[pos, 4]:
                maxscore = boxes[pos, 4]
                maxpos = pos
            pos = pos + 1
        boxes[i, 0:5] = boxes[maxpos, 0:5]
        boxes[maxpos, 0], boxes[maxpos, 1], boxes[maxpos, 2], boxes[maxpos, 3], boxes[maxpos, 4] = tx1, ty1, tx2, ty2, ts
        for j in range(5, 39):
            tmp = boxes[i, j]; boxes[i, j] = boxes[maxpos, j]; boxes[maxpos, j] = tmp
        tx1, ty1, tx2, ty2 = boxes[i, 0], boxes[i, 1], boxes[i, 2], boxes[i, 3]
        pos = i + 1
        while pos < N:
            x1, y1, x2, y2 = boxes[pos, 0], boxes[pos, 1], boxes[pos, 2], boxes[pos, 3]
            area = (x2 - x1 + one) * (y2 - y1 + one)
            iw = (min(tx2, x2) - max(tx1, x1) + one)
            if iw > 0:
                ih = (min(ty2, y2) - max(ty1, y1) + one)
                if ih > 0:
                    ua = F32((tx2 - tx1 + one) * (ty2 - ty1 + one) + area - iw * ih)
                    ov = iw * ih / ua
                    if method == 1:
                        weight = one - ov if ov > Nt else one
                    elif method == 2:
                        weight = F32(np.exp(float(-(ov * ov) / sigma)))
                    else:
                        weight = F32(0) if ov > Nt else one
                    boxes[pos, 4] = weight * boxes[pos, 4]
                    if boxes[pos, 4] < threshold:
                        boxes[pos, 0:5] = boxes[N - 1, 0:5]
                        for j in range(5, 39):
                            tmp = boxes[pos, j]; boxes[pos, j] = boxes[N - 1, j]; boxes[N - 1, j] = tmp
                        N = N - 1
                        pos = pos - 1
            pos = pos + 1
    return N


def _decay(r, t, sigma, Nt, method):
    """(hit, iw, ih, ov, new score) of row r against box t: the arithmetic of nms.pyx:236-253 in float32."""
    one = F32(1)
    x1, y1, x2, y2 = r[0], r[1], r[2], r[3]
    area = (x2 - x1 + one) * (y2 - y1 + one)
    iw = min(t[2], x2) - max(t[0], x1) + one
    if not iw > 0:
        return False, iw, None, None, r[4]
    ih = min(t[3], y2) - max(t[1], y1) + one
    if not ih > 0:
        return False, iw, ih, None, r[4]
    ua = (t[2] - t[0] + one) * (t[3] - t[1] + one) + area - iw * ih
    ov = iw * ih / ua
    if method == 1:
        weight = one - ov if ov > Nt else one
    elif method == 2:
        weight = F32(np.exp(np.float64(-(ov * ov) / sigma)))
    else:
        weight = F32(0) if ov > Nt else one
    return True, iw, ih, ov, weight * r[4]


def soft_nms_trace(boxes: np.ndarray, sigma=0.5, Nt=0.3, threshold=0.001, method=0, bug: Optional[str] = None):
    """soft_nms_39 on the kernel's plan: (1) the first arg-max of [i, N) as 128 threads and a reduction find it,
    (2) swap columns 0..38, (3) decay every row in (i, N) against box i, (4) the swap-with-last walk over the rows
    that touched box i, restoring the pre-decay score of the copy left at the tail.  Returns (keep, events): the
    branches reached.  ``bug`` restates one plausible kernel bug (SOFT_NMS_BUGS) instead."""
    sigma, Nt, threshold = F32(sigma), F32(Nt), F32(threshold)
    N0 = boxes.shape[0]
    N = N0
    ev = set()
    for i in range(N0):
        if i >= N:
            ev.add("outer_loop_ends_early")
            break
        s = boxes[i:N, 4]
        m = s.max()
        tied = np.flatnonzero(s == m)
        if len(tied) > 1:
            t0 = tied[0]
            for q in tied[1:]:
                ev.add("tie_thread" if t0 % NMS_T == q % NMS_T else
                       ("tie_lanes" if (t0 % NMS_T) // 32 == (q % NMS_T) // 32 else "tie_warps"))
        if bug == "argmax >=":        # each thread keeps the LAST maximum of its stride, the reduction the lowest index
            cand = [tid + NMS_T * int(np.flatnonzero(s[tid::NMS_T] == s[tid::NMS_T].max())[-1])
                    for tid in range(min(NMS_T, len(s)))]
            maxpos = i + min((c for c in cand if s[c] == m))
        else:
            maxpos = i + int(tied[0])
        if maxpos != i:
            ev.add("maxpos_swap")
            tmp = boxes[i, :39].copy(); boxes[i, :39] = boxes[maxpos, :39]; boxes[maxpos, :39] = tmp
        t = boxes[i, :4].copy()
        s_orig = boxes[:, 4].copy()
        hit = np.zeros(N0, bool)
        for pos in range(i + 1, N):
            h, iw, ih, ov, new = _decay(boxes[pos], t, sigma, Nt, method)
            if iw == 0:
                ev.add("touch_iw0")
            elif ih is not None and ih == 0:
                ev.add("touch_ih0")
            if h:
                if ov == Nt:
                    ev.add(f"ov_eq_Nt_m{method}")
                if new == threshold:
                    ev.add("score_eq_threshold")
                boxes[pos, 4] = new
                hit[pos] = True
        for pos in range(i + 1, N):
            if not hit[pos] and boxes[pos, 4] < threshold:
                ev.add("low_score_not_hit")
        n, pos, removed, last_removed_at = N, i + 1, 0, -1
        while pos < n:
            gate = hit[pos] if bug != "walk ignores s_hit" else True
            if gate and boxes[pos, 4] < threshold:
                ev.add("remove")
                if last_removed_at == pos:
                    ev.add("remove_moved_in")
                if pos == n - 1:
                    ev.add("remove_last")
                elif hit[n - 1] and boxes[n - 1, 4] != s_orig[n - 1]:
                    ev.add("tail_restore")
                if pos != n - 1 and not hit[n - 1] and boxes[n - 1, 4] < threshold:
                    ev.add("moved_in_not_hit_low")
                boxes[pos, :5] = boxes[n - 1, :5]
                tmp = boxes[pos, 5:39].copy(); boxes[pos, 5:39] = boxes[n - 1, 5:39]; boxes[n - 1, 5:39] = tmp
                if pos != n - 1 and bug != "no tail restore":
                    boxes[n - 1, 4] = s_orig[n - 1]
                if bug != "s_hit not carried":
                    hit[pos] = hit[n - 1]
                n -= 1
                removed += 1
                last_removed_at = pos
            else:
                pos += 1
        if removed >= 2 and n == i + 1:
            ev.add("removal_chain_empties_tail")
        N = n
    return N, ev


SOFT_NMS_BUGS = ("no tail restore", "argmax >=", "walk ignores s_hit", "s_hit not carried")
NMS_CLASSES = ("maxpos_swap", "tie_thread", "tie_lanes", "tie_warps", "ov_eq_Nt_m0", "ov_eq_Nt_m1", "ov_eq_Nt_m2",
               "score_eq_threshold", "touch_iw0", "touch_ih0", "low_score_not_hit", "remove", "remove_moved_in",
               "remove_last", "tail_restore", "moved_in_not_hit_low", "removal_chain_empties_tail",
               "outer_loop_ends_early", "N1", "N127", "N128", "N129", "N256", "N257", "N882", "batch")


def _rows(spec, seed=0):
    """(N, 56) float32 rows from [(x1, y1, x2, y2, score)]; columns 5..55 hold values unique to the row and column, so
    every move of columns 0..38 (and every non-move of 39..55) is visible."""
    r = np.zeros((len(spec), 56), np.float32)
    r[:, :5] = np.asarray(spec, np.float32)
    r[:, 5:] = (seed * 100000 + np.arange(len(spec))[:, None] * 64 + np.arange(5, 56)[None, :] + 0.5).astype(np.float32)
    return r


@dataclass
class NmsCase:
    label: str
    claims: Tuple[str, ...]
    build: Callable[[], np.ndarray]       # (N, 56), or (B, N, 56) for a batch
    method: int
    Nt: float
    threshold: float
    sigma: float = 0.5

    def params(self):
        return dict(sigma=self.sigma, Nt=self.Nt, threshold=self.threshold, method=self.method)


A = (0, 0, 9, 9)          # box i of the constructed steps: 10 x 10 px (the +1 of the reference's areas)


def _chain():
    # box 0 is second in line; row 1 wins step 0, and every other row overlaps it with IoU > 0.3: the walk removes
    # row 2, re-examines each row moved in from the tail and removes it too, until the last removal is the tail itself
    return _rows([(1, 0, 10, 9, 0.8), A + (0.9,), (0, 1, 9, 10, 0.7), (1, 1, 10, 10, 0.6), (0, 0, 8, 9, 0.5),
                  (0, 0, 9, 8, 0.4)])


def _gating():
    # step 0 (box A, score 0.9), method 1, Nt 0.3, threshold 0.25:
    #   row 1: IoU 0.5 -> weight 0.5, 0.4 -> 0.2 < 0.25: removed; the tail row (far away, score 0.1, never touched)
    #          moves in and must stay;
    #   row 2: IoU 0.5, 0.5 -> 0.25 == threshold: kept;   row 3: IoU 0.3 == Nt: weight 1;
    #   rows 4, 5: touch A with iw == 0 and ih == 0, score 0.125 < threshold: not hit, kept
    return _rows([A + (0.9,), (0, 0, 4, 9, 0.4), (5, 0, 9, 9, 0.5), (3, 0, 5, 9, 0.6), (10, 0, 19, 9, 0.125),
                  (0, 10, 9, 19, 0.125), (100, 100, 109, 109, 0.1)])


def _ov_eq_nt(frac):
    # IoU exactly frac (in tenths): a k x 10 box inside A has IoU k*10 / 100, and fl(k/10) == fl(Nt) for Nt = k/10;
    # a (k+1) x 10 box decays / goes, so the step still removes something
    k = int(round(frac * 10))
    return _rows([A + (0.9,), (0, 0, k - 1, 9, 0.8), (0, 0, k, 9, 0.7), (50, 50, 59, 59, 0.6), (1, 0, k, 9, 0.5)])


def _random(N, seed, plant_ties=True, score_den=64):
    """Dyadic rows: integer corners on a 256 px field, scores k / score_den (ties), the top score planted at rows 3, 4,
    40 and 131 so step 0 ties inside one thread's stride, across lanes and across warps."""
    rng = np.random.RandomState(seed)
    x1 = rng.randint(0, 240, N); y1 = rng.randint(0, 240, N)
    w = rng.randint(3, 60, N); h = rng.randint(3, 60, N)
    s = rng.randint(1, score_den, N) / score_den
    spec = np.stack([x1, y1, x1 + w, y1 + h, s], 1)
    if plant_ties:
        for n, r in enumerate((3, 4, 40, 131)):
            if r < N:
                spec[r] = (300 + 20 * n, 300, 310 + 20 * n, 310, 1.0)
    return _rows(spec.tolist(), seed)


NMS_CASES: List[NmsCase] = [
    NmsCase("chain_hard", ("maxpos_swap", "remove", "remove_moved_in", "remove_last", "tail_restore",
                           "removal_chain_empties_tail", "outer_loop_ends_early"), _chain, 0, 0.3, 0.001),
    NmsCase("chain_linear", ("remove_moved_in", "remove_last", "tail_restore", "removal_chain_empties_tail"),
            _chain, 1, 0.3, 0.5),
    NmsCase("chain_gaussian", ("remove_moved_in", "remove_last", "tail_restore"), _chain, 2, 0.3, 0.6),
    NmsCase("gating_linear", ("score_eq_threshold", "ov_eq_Nt_m1", "touch_iw0", "touch_ih0", "low_score_not_hit",
                              "moved_in_not_hit_low", "remove"), _gating, 1, 0.3, 0.25),
    NmsCase("gating_hard", ("touch_iw0", "touch_ih0", "low_score_not_hit", "moved_in_not_hit_low", "remove"),
            _gating, 0, 0.45, 0.25),
    NmsCase("ov_eq_nt_hard_0.3", ("ov_eq_Nt_m0",), lambda: _ov_eq_nt(0.3), 0, 0.3, 0.001),
    NmsCase("ov_eq_nt_linear_0.5", ("ov_eq_Nt_m1",), lambda: _ov_eq_nt(0.5), 1, 0.5, 0.3),
    NmsCase("ov_eq_nt_gauss_0.7", ("ov_eq_Nt_m2",), lambda: _ov_eq_nt(0.7), 2, 0.7, 0.5),
    NmsCase("n1", ("N1",), lambda: _rows([(5, 5, 20, 20, 0.5)]), 2, 0.3, 0.001),
    NmsCase("n127", ("N127", "tie_lanes", "tie_warps"), lambda: _random(127, 127), 0, 0.3, 0.001),
    NmsCase("n128", ("N128", "tie_lanes", "tie_warps"), lambda: _random(128, 128), 1, 0.3, 0.1),
    NmsCase("n129", ("N129", "tie_lanes", "tie_warps"), lambda: _random(129, 129), 2, 0.3, 0.3),
    NmsCase("n256", ("N256", "tie_thread", "tie_lanes", "tie_warps"), lambda: _random(256, 256), 0, 0.3, 0.001),
    NmsCase("n257", ("N257", "tie_thread", "remove_last"), lambda: _random(257, 257), 1, 0.5, 0.2),
    NmsCase("n882", ("N882", "tie_thread", "tie_lanes", "tie_warps", "remove_moved_in", "tail_restore"),
            lambda: _random(882, 882), 2, 0.3, 0.4),
]
NMS_CASE = {c.label: c for c in NMS_CASES}
# a few hundred images in one cpb200_soft_nms_39_batch launch (not in the golden fixture: each image is checked
# against the port)
NMS_BATCH = NmsCase("batch_300x48", ("batch",), lambda: np.stack([_random(48, 1000 + b, plant_ties=b % 2 == 0,
                                                                          score_den=16) for b in range(300)]),
                    1, 0.3, 0.3)
