"""Plain-numpy model of ``cv2.ellipse2Poly(center, (half_len, 2), angle, 0, 360, 1)``, the limb polygon the pose
drawing fills, for the tests of ``cpb200_ellipse_poly_batch`` and ``cpb200_render_plan_batch`` (csrc/render_plan.cu).

cv2 does not document it; these are its rules, pinned equal to cv2 by ``test_video_cpu.py`` over every integer angle
in [-180, 180], every half-length a limb of a 4096 x 4096 frame can have and centres of both parities:
  * the angle is brought into [0, 360] by whole turns, and its cosine and sine, like the 361 arc points', come from a
    float table of sin(i degrees) to seven decimals (``SIN``), widened to double;
  * point i is (cx + x * cos - y * sin, cy + x * sin + y * cos) in double, left to right, with x = half_len *
    SIN[450 - i] and y = 2 * SIN[i], each coordinate rounded half to even (where cx + offset lands on .5, the
    centre's parity decides);
  * a point equal to the one before it is dropped (the last point, equal to the first, stays); a polygon of one point
    becomes the centre twice.
"""
from __future__ import annotations

import numpy as np

SIN = np.float32(np.round(np.sin(np.deg2rad(np.arange(451, dtype=np.float64))), 7))
MAX_POINTS = 361
# the longest limb of a 4096 x 4096 frame joins opposite corners: int(sqrt(2 * 4095 ** 2) / 2)
MAX_HALF_LEN = int((2 * 4095 ** 2) ** 0.5 / 2)


def _norm(angle):
    while angle < 0:
        angle += 360
    while angle > 360:
        angle -= 360
    return angle


def ellipse_polys(cx, cy, half_len, angle):
    """The polygons of arrays ``cx``, ``cy``, ``half_len`` (M,) at one integer ``angle``: ``(points, counts)``, the
    (sum(counts), 2) int64 points of every polygon back to back and the (M,) point counts."""
    a = _norm(int(angle))
    alpha, beta = np.float64(SIN[450 - a]), np.float64(SIN[a])
    i = np.arange(MAX_POINTS)
    x = np.asarray(half_len, np.float64)[:, None] * SIN[450 - i].astype(np.float64)[None]
    y = 2.0 * SIN[i].astype(np.float64)[None]
    cx = np.asarray(cx, np.float64)[:, None]
    cy = np.asarray(cy, np.float64)[:, None]
    px = np.rint((cx + x * alpha) - y * beta).astype(np.int64)
    py = np.rint((cy + x * beta) + y * alpha).astype(np.int64)
    keep = np.ones(px.shape, bool)
    keep[:, 1:] = (px[:, 1:] != px[:, :-1]) | (py[:, 1:] != py[:, :-1])
    counts = keep.sum(1)
    pts = np.stack([px[keep], py[keep]], 1)
    single = np.flatnonzero(counts == 1)
    if len(single):                          # never with a half-width of 2, stated for completeness
        out, k = [], 0
        for m, c in enumerate(counts):
            out.append(np.array([[cx[m, 0], cy[m, 0]]] * 2, np.int64) if c == 1 else pts[k:k + c])
            k += c
        pts, counts = np.concatenate(out), np.maximum(counts, 2)
    return pts, counts


def ellipse_poly(cx, cy, half_len, angle):
    """One polygon: the (n, 2) int64 points of ``cv2.ellipse2Poly((cx, cy), (half_len, 2), angle, 0, 360, 1)``."""
    return ellipse_polys([cx], [cy], [half_len], angle)[0]


def domain():
    """The exhaustive domain: per angle in [-180, 180] the (cx, cy, half_len) of every half-length up to
    ``MAX_HALF_LEN`` at two centres, (even, odd) and (odd, even)."""
    L = np.arange(MAX_HALF_LEN + 1)
    cx = np.concatenate([np.full(len(L), 2048), np.full(len(L), 2049)])
    cy = np.concatenate([np.full(len(L), 2049), np.full(len(L), 2048)])
    return cx, cy, np.concatenate([L, L])
